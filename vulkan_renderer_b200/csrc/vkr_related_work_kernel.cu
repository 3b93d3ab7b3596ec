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

// Sampling probe (vkr_sample_related_work_batch): one thread per sample runs the prepare() and sample() of the tile kernel's light shader for one
// (light, shading point) pair. frame = rows x, y, z of world_to_shading_space, then its translation. Thread 0 writes the GGX density factor and
// whether the light is lit; a culled light leaves the directions and densities as they were.
template <int TECHNIQUE, int MAXV>
__global__ void __launch_bounds__(128)
related_work_probe_kernel(const unsigned char* light_block, const float* position_frame, uint32_t n, const float* rnd, float* out_dirs, float* out_densities, float* out_ggx_lit) {
	rw_light<MAXV> light;
	rw_load_light<MAXV>(light, light_block);
	const float* fr = position_frame + 3;
	rw_frame frame;
	frame.rx = make3(fr[0], fr[1], fr[2]); frame.ry = make3(fr[3], fr[4], fr[5]); frame.rz = make3(fr[6], fr[7], fr[8]); frame.t = make3(fr[9], fr[10], fr[11]);
	rw_sampler<TECHNIQUE, MAXV> sampler;
	const bool lit = sampler.prepare(light, make3(position_frame[0], position_frame[1], position_frame[2]), frame);
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i == 0) { out_ggx_lit[0] = lit ? sampler.ggx_density_factor() : 0.0f; out_ggx_lit[1] = lit ? 1.0f : 0.0f; }
	if (i >= n || !lit) return;
	float density;
	const f3 d = sampler.sample(make2(rnd[2 * i], rnd[2 * i + 1]), &density);
	out_dirs[3 * i] = d.x; out_dirs[3 * i + 1] = d.y; out_dirs[3 * i + 2] = d.z;
	out_densities[i] = density;
}

} // namespace vkr

using namespace vkr;

cudaError_t VKR_TILE_LAUNCHER(vkr_launch_related_work_probe_v)(uint32_t technique, const unsigned char* light_block, const float* position_frame, uint32_t n, const float* random_numbers,
	float* out_dirs, float* out_densities, float* out_ggx_lit, cudaStream_t stream)
{
	const unsigned blocks = (n + 127) / 128 > 0 ? (n + 127) / 128 : 1;
	switch (technique) {
#define VKR_PROBE(T) case T: related_work_probe_kernel<T, VKR_MAXV_TU><<<blocks, 128, 0, stream>>>(light_block, position_frame, n, random_numbers, out_dirs, out_densities, out_ggx_lit); break;
	VKR_PROBE(0) VKR_PROBE(1) VKR_PROBE(2) VKR_PROBE(3) VKR_PROBE(4) VKR_PROBE(5) VKR_PROBE(6) VKR_PROBE(7) VKR_PROBE(8) VKR_PROBE(9) VKR_PROBE(10)
#undef VKR_PROBE
	default: return cudaErrorInvalidValue;
	}
	return cudaGetLastError();
}

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
