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
#include "vkr_shading_tile.cuh"
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
__global__ void __launch_bounds__(kShadeThreads, 3)
error_display_kernel(const shading_kernel_params p) {
	shade_tile<MAXV + 1, false, false>(p, error_display_light_shader<MAXV>());
}

template <int STRATEGY, int MAXV, bool TRACE>
__global__ void __launch_bounds__(TRACE ? kShadeThreads + kTraceThreads : kShadeThreads, TRACE ? 2 : 3)
related_work_kernel(const shading_kernel_params p) {
	shade_tile<MAXV + 1, false, TRACE>(p, related_work_light_shader<STRATEGY, MAXV, TRACE>());
}

} // namespace vkr

using namespace vkr;

static constexpr size_t kStreamFloats = stream_floats_per_warp(false);

template <int STRATEGY, int MAXV, bool TRACE>
static cudaError_t launch_related_work(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.tile_count <= 0) return cudaSuccess;
	const int threads = TRACE ? kShadeThreads + kTraceThreads : kShadeThreads;
	const size_t smem = p.constants_smem_bytes + (TRACE ? sizeof(float) * kStreamFloats * kShadeWarps + sizeof(int) * (size_t) p.stack_depth * kTraceThreads : 0);
	auto kernel = related_work_kernel<STRATEGY, MAXV, TRACE>;
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

template <int MAXV>
static cudaError_t launch_error_display(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.tile_count <= 0) return cudaSuccess;
	auto kernel = error_display_kernel<MAXV>;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) p.constants_smem_bytes);
	if (err != cudaSuccess) return err;
	kernel<<<p.tile_count, kShadeThreads, p.constants_smem_bytes, stream>>>(p);
	return cudaGetLastError();
}

template <int STRATEGY, int MAXV>
static cudaError_t launch_related_work_traced(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.trace_shadow_rays != 0 && p.tri_count != 0) return launch_related_work<STRATEGY, MAXV, true>(p, stream);
	return launch_related_work<STRATEGY, MAXV, false>(p, stream);
}

// One translation unit per light vertex bound (built with -DVKR_MAXV_TU=3 .. 7, __graft_entry__.py)
#ifndef VKR_MAXV_TU
#error "compile with -DVKR_MAXV_TU=<3..7>"
#endif
#define VKR_CONCAT2(a, b) a##b
#define VKR_CONCAT(a, b) VKR_CONCAT2(a, b)
cudaError_t VKR_CONCAT(vkr_launch_related_work_kernel_maxv, VKR_MAXV_TU)(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.error_display != 0) { // the error display modes of projected solid angle sampling (techniques 10, 11, 12)
		if (p.error_display < 1 || p.error_display > 6 || p.polygon_sampling_technique < VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) return cudaErrorInvalidValue;
		return launch_error_display<VKR_MAXV_TU>(p, stream);
	}
	if (p.stack_depth < 2 || p.stack_depth > kMaxStackDepth) return cudaErrorInvalidValue;
	if (p.trace_shadow_rays != 0 && p.tri_count != 0 && p.bvh_width != VKR_BVH_WIDTH) return cudaErrorInvalidValue;
	if (p.polygon_sampling_technique < VKR_TECHNIQUE_BASELINE || p.polygon_sampling_technique > VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) return cudaErrorInvalidValue;
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY: return launch_related_work_traced<VKR_STRATEGY_DIFFUSE_ONLY, VKR_MAXV_TU>(p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS: return launch_related_work_traced<VKR_STRATEGY_DIFFUSE_GGX_MIS, VKR_MAXV_TU>(p, stream);
	default: return cudaErrorInvalidValue;
	}
}
