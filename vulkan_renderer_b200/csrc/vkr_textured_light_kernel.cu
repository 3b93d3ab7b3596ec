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
#include "vkr_tile_launch.cuh"
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
__global__ void VKR_TILE_LAUNCH_BOUNDS(TRACE)
textured_light_kernel(const shading_kernel_params p) {
	shade_tile<MAXP, OPTIMAL, TRACE, true>(p, textured_light_shader<STRATEGY, MAXP, OPTIMAL, TRACE>());
}

} // namespace vkr

using namespace vkr;

constexpr int kMaxP = VKR_MAXV_TU + 1;   // MAXP: vertices of a light after clipping to the horizon

// the kernels of one strategy, with and without shadow rays
template <int STRATEGY, bool OPTIMAL = false>
static cudaError_t launch(const shading_kernel_params& p, cudaStream_t stream) {
	return launch_tile_kernel<OPTIMAL>(textured_light_kernel<STRATEGY, kMaxP, OPTIMAL, true>, textured_light_kernel<STRATEGY, kMaxP, OPTIMAL, false>, p, stream);
}

cudaError_t VKR_TILE_LAUNCHER(vkr_launch_textured_light_kernel_v)(const shading_kernel_params& p, cudaStream_t stream) {
	if (!tile_launch_valid(p, true)) return cudaErrorInvalidValue;
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY: return launch<VKR_STRATEGY_DIFFUSE_ONLY>(p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS: return launch<VKR_STRATEGY_DIFFUSE_GGX_MIS>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY: return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_MIS:
		if (p.mis_heuristic == VKR_MIS_OPTIMAL) return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, true>(p, stream);
		return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM: return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM>(p, stream);
	default: return cudaErrorInvalidValue;
	}
}
