// vkr_tile_launch.cuh -- how the host launches a tile kernel: one CTA per 16x8 tile with shade_tile() (vkr_shading_tile.cuh) as its body.
//
// Included by the four kernel translation units (vkr_shading_kernel.cu, vkr_textured_light_kernel.cu, vkr_related_work_kernel.cu,
// vkr_textured_related_work_kernel.cu); each of them is compiled once per bound of the light vertex count and exports one entry point per bound.
// Everything here has internal linkage: every unit is compiled with its own VKR_MAXV_TU.
#pragma once
#include "vkr_shading_tile.cuh"

// One object per bound of the light vertex count, MAX_POLYGONAL_LIGHT_VERTEX_COUNT = 3 .. 7 (__graft_entry__.py); its entry point is
// VKR_TILE_LAUNCHER(<family>_v), e.g. vkr_launch_shading_kernel_v4 for quad lights.
#ifndef VKR_MAXV_TU
#error "compile with -DVKR_MAXV_TU=<3..7>"
#endif
#define VKR_CONCAT2(a, b) a##b
#define VKR_CONCAT(a, b) VKR_CONCAT2(a, b)
#define VKR_TILE_LAUNCHER(prefix) VKR_CONCAT(prefix, VKR_MAXV_TU)

#ifndef VKR_TRACED_CTAS_PER_SM
#define VKR_TRACED_CTAS_PER_SM 2   // CTAs per SM the register allocation of the kernels with shadow rays is made for (with kShadeRegs / kTraceRegs, vkr_shading_tile.cuh)
#endif
// __launch_bounds__ of every tile kernel: the shading warps, plus the trace warps when it traces shadow rays
#define VKR_TILE_LAUNCH_BOUNDS(TRACE) __launch_bounds__((TRACE) ? kShadeThreads + kTraceThreads : kShadeThreads, (TRACE) ? VKR_TRACED_CTAS_PER_SM : 3)

namespace vkr {

static bool traces_shadow_rays(const shading_kernel_params& p) { return p.trace_shadow_rays != 0 && p.tri_count != 0; }

// What every tile kernel that shades radiance needs; light_textures: the kernel reads the light textures.
static bool tile_launch_valid(const shading_kernel_params& p, bool light_textures) {
	if (p.stack_depth < 2 || p.stack_depth > kMaxStackDepth) return false;
	return !light_textures || (p.light_texture_texels && p.light_texture_dims && p.light_texture_offsets && p.light_texture_count != 0);
}

// Dynamic shared memory of a tile in the layout shade_tile() carves it
template <bool OPTIMAL, bool TRACE>
static size_t tile_smem_bytes(const shading_kernel_params& p) {
	return p.constants_smem_bytes + (TRACE ? tile_streams_bytes(OPTIMAL) + sizeof(int) * (size_t) p.stack_depth * kTraceThreads : 0);
}

typedef void tile_kernel_t(const shading_kernel_params);

template <bool OPTIMAL, bool TRACE>
static cudaError_t launch_tile_kernel(tile_kernel_t* kernel, const shading_kernel_params& p, cudaStream_t stream) {
	if (p.tile_count <= 0) return cudaSuccess;
	const int threads = TRACE ? kShadeThreads + kTraceThreads : kShadeThreads;
	const size_t smem = tile_smem_bytes<OPTIMAL, TRACE>(p);
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
	if (err != cudaSuccess) return err;
	// Shared memory for exactly the CTAs the register file admits; the rest of the 228 KB stays L1 for BVH nodes
	int ctas = 0;
	err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kernel, threads, smem);
	if (err != cudaSuccess) return err;
	const int carveout = (int) ((100 * ((smem + 1024) * (size_t) (ctas > 0 ? ctas : 1)) + 228 * 1024 - 1) / (228 * 1024));
	err = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout > 100 ? 100 : carveout);
	if (err != cudaSuccess) return err;
	kernel<<<p.tile_count, threads, smem, stream>>>(p);
	return cudaGetLastError();
}

// The frame's tiles with the kernel that traces shadow rays if the frame has any, else with the one that does not
template <bool OPTIMAL>
static cudaError_t launch_tile_kernel(tile_kernel_t* traced, tile_kernel_t* untraced, const shading_kernel_params& p, cudaStream_t stream) {
	return traces_shadow_rays(p) ? launch_tile_kernel<OPTIMAL, true>(traced, p, stream) : launch_tile_kernel<OPTIMAL, false>(untraced, p, stream);
}

} // namespace vkr
