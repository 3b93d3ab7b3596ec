// vkr_textured_light_kernel.cu -- the shading megakernel for frames with textured polygonal lights (sm_90a).
//
// get_polygon_radiance() of the reference (src/shaders/shading_pass.frag.glsl:151-185) multiplies the light's radiance by a texture when its
// texturing technique is not "none": an area texture in the light's plane, a light probe seen through the polygon (portal) or an IES profile,
// each read with textureLod(..., 0) through a sampler that repeats in u and clamps in v (src/main.c:613-623). The kernels of
// vkr_shading_kernel.cu are built without that branch (LIGHT_TEXTURES = false: what every configuration of the benchmark runs); this
// translation unit instantiates the same tile body (vkr_shading_tile.cuh) and the same per-light code (vkr_shade_light.cuh) with
// LIGHT_TEXTURES = true, so the texture fetch sits exactly where the shader has it: after the visibility pre-test, before the BRDF product,
// and in the light display of the tile prologue. vkr_api.cu sends a frame here when at least one light of the constant block is textured.
// The biased variant of the sampler is a run-time choice inside the kernel (half as many kernels to compile; the choice is uniform).
// Compile with -fmad=false (see vkr_device_math.cuh).
#include "vkr_shading_tile.cuh"
#include "vkr_shade_light.cuh"

namespace vkr {

template <int STRATEGY, int MAXP, bool OPTIMAL, bool TRACE>
struct textured_light_shader {
	VKR_DEV void operator()(bool on, const shading_point& sp, const ltc_state& l, const unsigned char* light, noise_stream& ns,
		const shading_kernel_params& p, const unsigned char* cb, uint32_t px, uint32_t py, ray_producer& q, pixel_sum& result, int lane) const
	{
		if (p.biased_sampling) shade_light<STRATEGY, MAXP, true, OPTIMAL, TRACE, true>(on, sp, l, light, ns, p, cb, px, py, q, result, lane);
		else shade_light<STRATEGY, MAXP, false, OPTIMAL, TRACE, true>(on, sp, l, light, ns, p, cb, px, py, q, result, lane);
	}
};

template <int STRATEGY, int MAXP, bool OPTIMAL, bool TRACE>
__global__ void __launch_bounds__(TRACE ? kShadeThreads + kTraceThreads : kShadeThreads, TRACE ? 2 : 3)
textured_light_kernel(const shading_kernel_params p) {
	shade_tile<MAXP, OPTIMAL, TRACE, true>(p, textured_light_shader<STRATEGY, MAXP, OPTIMAL, TRACE>());
}

} // namespace vkr

using namespace vkr;

template <int STRATEGY, int MAXP, bool OPTIMAL, bool TRACE>
static cudaError_t launch_traced(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.tile_count <= 0) return cudaSuccess;
	const int threads = TRACE ? kShadeThreads + kTraceThreads : kShadeThreads;
	constexpr size_t stream_floats = stream_floats_per_warp(OPTIMAL);
	const size_t smem = p.constants_smem_bytes + (TRACE ? sizeof(float) * stream_floats * kShadeWarps + sizeof(int) * (size_t) p.stack_depth * kTraceThreads : 0);
	auto kernel = textured_light_kernel<STRATEGY, MAXP, OPTIMAL, TRACE>;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
	if (err != cudaSuccess) return err;
	int ctas = 0;
	err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kernel, threads, smem);
	if (err != cudaSuccess) return err;
	const int carveout = (int) ((100 * ((smem + 1024) * (size_t) (ctas > 0 ? ctas : 1)) + 228 * 1024 - 1) / (228 * 1024));
	err = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout > 100 ? 100 : carveout);
	if (err != cudaSuccess) return err;
	kernel<<<p.tile_count, threads, smem, stream>>>(p);
	return cudaGetLastError();
}

template <int STRATEGY, int MAXP, bool OPTIMAL>
static cudaError_t launch_variant(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.trace_shadow_rays != 0 && p.tri_count != 0) return launch_traced<STRATEGY, MAXP, OPTIMAL, true>(p, stream);
	return launch_traced<STRATEGY, MAXP, OPTIMAL, false>(p, stream);
}

// One translation unit per vertex bound (built with -DVKR_MAXP_TU=4 .. 8, __graft_entry__.py): MAXP = light vertices + 1.
#ifndef VKR_MAXP_TU
#error "compile with -DVKR_MAXP_TU=<4..8>"
#endif
#define VKR_CONCAT2(a, b) a##b
#define VKR_CONCAT(a, b) VKR_CONCAT2(a, b)
cudaError_t VKR_CONCAT(vkr_launch_textured_light_kernel_maxp, VKR_MAXP_TU)(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.stack_depth < 2 || p.stack_depth > kMaxStackDepth) return cudaErrorInvalidValue;
	if (p.trace_shadow_rays != 0 && p.tri_count != 0 && p.bvh_width != VKR_BVH_WIDTH) return cudaErrorInvalidValue;
	if (!p.light_texture_texels || !p.light_texture_dims || !p.light_texture_offsets || p.light_texture_count == 0) return cudaErrorInvalidValue;
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY: return launch_variant<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXP_TU, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS: return launch_variant<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXP_TU, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY: return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY, VKR_MAXP_TU, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_MIS:
		if (p.mis_heuristic == VKR_MIS_OPTIMAL) return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, VKR_MAXP_TU, true>(p, stream);
		return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, VKR_MAXP_TU, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM: return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM, VKR_MAXP_TU, false>(p, stream);
	default: return cudaErrorInvalidValue;
	}
}
