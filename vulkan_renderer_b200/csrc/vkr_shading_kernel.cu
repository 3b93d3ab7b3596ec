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
#include "vkr_shading_tile.cuh"
#include "vkr_shade_light.cuh"

// The counters edition (-DVKR_TRACE_STATS, vkr_trace_counter_t) is a kernel of its own name: the host stubs of two editions of one template
// would be merged by the linker.
#ifdef VKR_TRACE_STATS
#define shading_kernel shading_kernel_counters
#define VKR_LAUNCHER_PREFIX vkr_launch_shading_kernel_stats_maxp
#else
#define VKR_LAUNCHER_PREFIX vkr_launch_shading_kernel_maxp
#endif

#ifndef VKR_TRACED_CTAS_PER_SM
#define VKR_TRACED_CTAS_PER_SM 2   // CTAs per SM the register allocation of the kernels with shadow rays is made for (tuning knob, with VKR_SHADE_REGS / VKR_TRACE_REGS)
#endif

namespace vkr {

template <int STRATEGY, int MAXP, bool BIASED, bool OPTIMAL, bool TRACE>
__global__ void __launch_bounds__(TRACE ? kShadeThreads + kTraceThreads : kShadeThreads, TRACE ? VKR_TRACED_CTAS_PER_SM : 3)
shading_kernel(const shading_kernel_params p) {
	shade_tile<MAXP, OPTIMAL, TRACE>(p, psa_light_shader<STRATEGY, MAXP, BIASED, OPTIMAL, TRACE>());
}

} // namespace vkr

using namespace vkr;

template <int STRATEGY, int MAXP, bool BIASED, bool OPTIMAL, bool TRACE>
static cudaError_t launch_traced(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.tile_count <= 0) return cudaSuccess;
	const int threads = TRACE ? kShadeThreads + kTraceThreads : kShadeThreads;
	const size_t smem = p.constants_smem_bytes + (TRACE ? sizeof(float) * stream_floats_per_warp(OPTIMAL) * kShadeWarps + sizeof(int) * (size_t) p.stack_depth * kTraceThreads : 0);
	auto kernel = shading_kernel<STRATEGY, MAXP, BIASED, OPTIMAL, TRACE>;
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

template <int STRATEGY, int MAXP, bool BIASED, bool OPTIMAL>
static cudaError_t launch_variant(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.trace_shadow_rays != 0 && p.tri_count != 0) return launch_traced<STRATEGY, MAXP, BIASED, OPTIMAL, true>(p, stream);
	return launch_traced<STRATEGY, MAXP, BIASED, OPTIMAL, false>(p, stream);
}

template <int MAXP, bool BIASED>
static cudaError_t launch_strategy(const shading_kernel_params& p, cudaStream_t stream) {
	switch (p.sampling_strategies) {
	case VKR_STRATEGY_DIFFUSE_ONLY: return launch_variant<VKR_STRATEGY_DIFFUSE_ONLY, MAXP, BIASED, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_GGX_MIS: return launch_variant<VKR_STRATEGY_DIFFUSE_GGX_MIS, MAXP, BIASED, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY: return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY, MAXP, BIASED, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_MIS:
		if (p.mis_heuristic == VKR_MIS_OPTIMAL) return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, MAXP, BIASED, true>(p, stream);
		return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_MIS, MAXP, BIASED, false>(p, stream);
	case VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM: return launch_variant<VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM, MAXP, BIASED, false>(p, stream);
	default: return cudaErrorInvalidValue;
	}
}

// One translation unit per vertex bound (built with -DVKR_MAXP_TU=4 .. 8, __graft_entry__.py): MAXP = light vertices + 1.
#ifndef VKR_MAXP_TU
#error "compile with -DVKR_MAXP_TU=<4..8>"
#endif
#define VKR_CONCAT2(a, b) a##b
#define VKR_CONCAT(a, b) VKR_CONCAT2(a, b)
cudaError_t VKR_CONCAT(VKR_LAUNCHER_PREFIX, VKR_MAXP_TU)(const shading_kernel_params& p, cudaStream_t stream) {
	if (p.stack_depth < 2 || p.stack_depth > kMaxStackDepth) return cudaErrorInvalidValue;
	if (p.trace_shadow_rays != 0 && p.tri_count != 0 && p.bvh_width != VKR_BVH_WIDTH) return cudaErrorInvalidValue; // the scene's BVH layout must be the one these kernels walk
	return p.biased_sampling ? launch_strategy<VKR_MAXP_TU, true>(p, stream) : launch_strategy<VKR_MAXP_TU, false>(p, stream);
}
