// vkr_textured_related_work_kernel.cu -- the related-work sampling techniques for frames with textured polygonal lights (sm_90a).
//
// related_work_kernel (vkr_related_work_kernel.cu) with LIGHT_TEXTURES = true: the texture fetch of get_polygon_radiance()
// (src/shaders/shading_pass.frag.glsl:151-185) where the shader has it, in the per-light code (vkr_related_work_light.cuh) and in the light
// display of the tile prologue (vkr_shading_tile.cuh). vkr_api.cu sends a frame here when a light of the constant block is textured and the
// sampling technique is one of sample_polygon_technique_t 0..10. Compile with -fmad=false (see vkr_device_math.cuh).
#include "vkr_tile_launch.cuh"
#include "vkr_related_work_light.cuh"

namespace vkr {

template <int STRATEGY, int MAXV, bool TRACE>
__global__ void VKR_TILE_LAUNCH_BOUNDS(TRACE)
textured_related_work_kernel(const shading_kernel_params p) {
	shade_tile<MAXV + 1, false, TRACE, true>(p, related_work_light_shader<STRATEGY, MAXV, TRACE, true>());
}

} // namespace vkr

using namespace vkr;

cudaError_t VKR_TILE_LAUNCHER(vkr_launch_textured_related_work_kernel_v)(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.error_display != 0) return cudaErrorInvalidValue;
	if (!tile_launch_valid(p, true)) return cudaErrorInvalidValue;
	if (p.polygon_sampling_technique < VKR_TECHNIQUE_BASELINE || p.polygon_sampling_technique > VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) return cudaErrorInvalidValue;
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY:
		return launch_tile_kernel<false>(textured_related_work_kernel<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXV_TU, true>, textured_related_work_kernel<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXV_TU, false>, p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS:
		return launch_tile_kernel<false>(textured_related_work_kernel<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXV_TU, true>, textured_related_work_kernel<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXV_TU, false>, p, stream);
	default: return cudaErrorInvalidValue;
	}
}
