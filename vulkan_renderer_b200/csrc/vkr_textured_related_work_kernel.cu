// vkr_textured_related_work_kernel.cu -- the related-work sampling techniques for frames with textured polygonal lights (sm_90a).
//
// related_work_kernel (vkr_related_work_kernel.cu) with LIGHT_TEXTURES = true: the texture fetch of get_polygon_radiance()
// (src/shaders/shading_pass.frag.glsl:151-185) where the shader has it, in the per-light code (vkr_related_work_light.cuh) and in the light
// display of the tile prologue (vkr_shading_tile.cuh). vkr_api.cu sends a frame here when a light of the constant block is textured and the
// sampling technique is one of sample_polygon_technique_t 0..10. Compile with -fmad=false (see vkr_device_math.cuh).
#include "vkr_shading_tile.cuh"
#include "vkr_related_work_light.cuh"

namespace vkr {

template <int STRATEGY, int MAXV, bool TRACE>
__global__ void __launch_bounds__(TRACE ? kShadeThreads + kTraceThreads : kShadeThreads, TRACE ? 2 : 3)
textured_related_work_kernel(const shading_kernel_params p) {
	shade_tile<MAXV + 1, false, TRACE, true>(p, related_work_light_shader<STRATEGY, MAXV, TRACE, true>());
}

} // namespace vkr

using namespace vkr;

static constexpr size_t kStreamFloats = stream_floats_per_warp(false);

template <int STRATEGY, int MAXV, bool TRACE>
static cudaError_t launch(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.tile_count <= 0) return cudaSuccess;
	const int threads = TRACE ? kShadeThreads + kTraceThreads : kShadeThreads;
	const size_t smem = p.constants_smem_bytes + (TRACE ? sizeof(float) * kStreamFloats * kShadeWarps + sizeof(int) * (size_t) p.stack_depth * kTraceThreads : 0);
	auto kernel = textured_related_work_kernel<STRATEGY, MAXV, TRACE>;
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

template <int STRATEGY, int MAXV>
static cudaError_t launch_traced(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.trace_shadow_rays != 0 && p.tri_count != 0) return launch<STRATEGY, MAXV, true>(p, stream);
	return launch<STRATEGY, MAXV, false>(p, stream);
}

// One translation unit per light vertex bound (built with -DVKR_MAXV_TU=3 .. 7, __graft_entry__.py)
#ifndef VKR_MAXV_TU
#error "compile with -DVKR_MAXV_TU=<3..7>"
#endif
#define VKR_CONCAT2(a, b) a##b
#define VKR_CONCAT(a, b) VKR_CONCAT2(a, b)
cudaError_t VKR_CONCAT(vkr_launch_textured_related_work_kernel_maxv, VKR_MAXV_TU)(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.error_display != 0) return cudaErrorInvalidValue;
	if (p.stack_depth < 2 || p.stack_depth > kMaxStackDepth) return cudaErrorInvalidValue;
	if (p.trace_shadow_rays != 0 && p.tri_count != 0 && p.bvh_width != VKR_BVH_WIDTH) return cudaErrorInvalidValue;
	if (p.polygon_sampling_technique < VKR_TECHNIQUE_BASELINE || p.polygon_sampling_technique > VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) return cudaErrorInvalidValue;
	if (!p.light_texture_texels || !p.light_texture_dims || !p.light_texture_offsets || p.light_texture_count == 0) return cudaErrorInvalidValue;
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY: return launch_traced<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXV_TU>(p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS: return launch_traced<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXV_TU>(p, stream);
	default: return cudaErrorInvalidValue;
	}
}
