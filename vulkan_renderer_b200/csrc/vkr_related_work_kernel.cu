// vkr_related_work_kernel.cu -- the shading megakernel with the related-work polygon sampling techniques (sm_90a).
//
// SURVEY 8 row f4: the samplers the reference compares projected solid angle sampling against (shading_pass.frag.glsl:332-481,
// polygon_sampling_related_work.glsl): baseline, Turk, Urena, Arvo (solid angle / projected solid angle), solid angle with and
// without clipping, Hart et al.'s bilinear and biquadratic cosine warps. The tile body, the warp-specialised ray streams and the
// output stage are those of the main kernel (vkr_shading_tile.cuh); only the light shader differs. Same launch shape, same
// arithmetic contract (-fmad=false), results bit-identical to the reference shader fixtures ("_q<technique>").
// The error display modes of the shader (colour-coded error of the sampling procedure) live here too: error_display_kernel.
// The technique is a warp-uniform run-time switch inside one kernel per (strategy, vertex bound, shadow rays): these are
// comparison baselines, not the benchmarked path, so code size matters more than the last register.
#include "vkr_tile_launch.cuh"
#include "vkr_related_work_light.cuh"
#include "vkr_error_display.cuh"

namespace vkr {

// Light shader of the error display modes (vkr_error_display.cuh)
template <int MAXV>
struct error_display_light_shader {
	VKR_DEV void operator()(bool on, const shading_point& sp, const ltc_state& l, const unsigned char* light, noise_stream& ns,
		const shading_kernel_params& p, const unsigned char* cb, uint32_t px, uint32_t py, ray_producer&, pixel_sum& result, int) const
	{
		if (!on) return; // no warp-level operations below: lanes are independent
		f3 color;
		if (error_display_of_light<MAXV>(&color, sp, l, light, ns, p, cb, px, py)) result.color = result.color + color;
	}
};

template <int MAXV>
__global__ void VKR_TILE_LAUNCH_BOUNDS(false)
error_display_kernel(const shading_kernel_params p) {
	shade_tile<MAXV + 1, false, false>(p, error_display_light_shader<MAXV>());
}

template <int STRATEGY, int MAXV, bool TRACE>
__global__ void VKR_TILE_LAUNCH_BOUNDS(TRACE)
related_work_kernel(const shading_kernel_params p) {
	shade_tile<MAXV + 1, false, TRACE>(p, related_work_light_shader<STRATEGY, MAXV, TRACE>());
}

} // namespace vkr

using namespace vkr;

cudaError_t VKR_TILE_LAUNCHER(vkr_launch_related_work_kernel_v)(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.error_display != 0) { // the error display modes of projected solid angle sampling (techniques 10, 11, 12)
		if (p.error_display < 1 || p.error_display > 6 || p.polygon_sampling_technique < VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) return cudaErrorInvalidValue;
		return launch_tile_kernel<false, false>(error_display_kernel<VKR_MAXV_TU>, p, stream);
	}
	if (!tile_launch_valid(p, false)) return cudaErrorInvalidValue;
	if (p.polygon_sampling_technique < VKR_TECHNIQUE_BASELINE || p.polygon_sampling_technique > VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) return cudaErrorInvalidValue;
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY:
		return launch_tile_kernel<false>(related_work_kernel<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXV_TU, true>, related_work_kernel<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXV_TU, false>, p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS:
		return launch_tile_kernel<false>(related_work_kernel<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXV_TU, true>, related_work_kernel<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXV_TU, false>, p, stream);
	default: return cudaErrorInvalidValue;
	}
}
