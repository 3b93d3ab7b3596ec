// vkr_shading_kernel.cu -- the per-screen-tile shading megakernel (sm_90a).
//
// Replaces subpass 1 of the reference frame (src/main.c:1429-1434, the fragment shader
// src/shaders/shading_pass.frag.glsl:824-866 with everything it calls). One CTA shades one
// 16x8 pixel tile; a warp covers an 8x4 pixel patch so that shadow rays of a warp start close
// together and head for the same light. Per frame the kernel reads
//   - the G-buffer as four coalesced float4 planes (64 B/pixel),
//   - the per-frame constant block incl. all polygonal lights (bytes identical to what the
//     reference's write_constants() produces, src/main.c:2114-2188) -> staged once per CTA into
//     shared memory with a bulk async copy (cp.async.bulk + mbarrier, the TMA engine),
//   - 4 LTC texels per pixel (software bilinear, fp32 weights), one RGBA16 noise texel per two
//     2D random numbers,
//   - BVH node pairs and triangles along the shadow rays,
// and writes one float4 of linear radiance per pixel (16 B/pixel).
//
// Execution model (warp-specialised). A CTA shades one 16x8 pixel tile with 4 SHADING warps (8x4 pixel patches: sampling,
// BRDF and MIS arithmetic per pixel in registers) and 8 TRACE warps that only traverse the BVH. Shading lanes push
// their shadow rays (direction, light-plane distance, the radiance to add if the ray is unoccluded) into a ring buffer
// in shared memory using __ballot_sync compaction; trace lanes pull rays one at a time as soon as their previous ray
// has terminated, so traversal runs with full warps although the rays come from lanes that may be idle and although
// ray lengths differ (vkr_ray_stream.cuh). After the split the trace warps hand most of their registers to the shading
// warps (setmaxnreg: 56 vs 128 per thread), so 24 warps are resident per SM instead of the 12 a monolithic kernel with
// 168 registers gets. Results are added to the owning pixel strictly in submission order, which keeps the
// floating-point sums identical to the reference's sequential loop. Without shadow rays (TRACE = false) the kernel is
// launched with the shading warps only.
// Compile with -fmad=false (see vkr_device_math.cuh).
#include "vkr_tile_launch.cuh"
#include "vkr_shade_light.cuh"

// The counters edition (-DVKR_TRACE_STATS, vkr_trace_counter_t) is a kernel of its own name: the host stubs of two editions of one template
// would be merged by the linker.
#ifdef VKR_TRACE_STATS
#define shading_kernel shading_kernel_counters
#define VKR_LAUNCHER_PREFIX vkr_launch_shading_kernel_stats_v
#else
#define VKR_LAUNCHER_PREFIX vkr_launch_shading_kernel_v
#endif

namespace vkr {

template <int STRATEGY, int MAXP, bool BIASED, bool OPTIMAL, bool TRACE>
__global__ void VKR_TILE_LAUNCH_BOUNDS(TRACE)
shading_kernel(const shading_kernel_params p) {
	shade_tile<MAXP, OPTIMAL, TRACE>(p, psa_light_shader<STRATEGY, MAXP, BIASED, OPTIMAL, TRACE>());
}

} // namespace vkr

using namespace vkr;

constexpr int kMaxP = VKR_MAXV_TU + 1;   // MAXP: vertices of a light after clipping to the horizon

// the kernels of one strategy, with and without shadow rays
template <int STRATEGY, bool BIASED, bool OPTIMAL = false>
static cudaError_t launch(const shading_kernel_params& p, cudaStream_t stream) {
	return launch_tile_kernel<OPTIMAL>(shading_kernel<STRATEGY, kMaxP, BIASED, OPTIMAL, true>, shading_kernel<STRATEGY, kMaxP, BIASED, OPTIMAL, false>, p, stream);
}

template <bool BIASED>
static cudaError_t launch_strategy(const shading_kernel_params& p, cudaStream_t stream) {
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY: return launch<VKR_STRATEGY_DIFFUSE_ONLY, BIASED>(p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS: return launch<VKR_STRATEGY_DIFFUSE_GGX_MIS, BIASED>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY: return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY, BIASED>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_MIS:
		if (p.mis_heuristic == VKR_MIS_OPTIMAL) return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, BIASED, true>(p, stream);
		return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, BIASED>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM: return launch<VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM, BIASED>(p, stream);
	default: return cudaErrorInvalidValue;
	}
}

cudaError_t VKR_TILE_LAUNCHER(VKR_LAUNCHER_PREFIX)(const shading_kernel_params& p, cudaStream_t stream) {
	if (!tile_launch_valid(p, false)) return cudaErrorInvalidValue;
	return p.biased_sampling ? launch_strategy<true>(p, stream) : launch_strategy<false>(p, stream);
}
