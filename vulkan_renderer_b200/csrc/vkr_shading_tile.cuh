// vkr_shading_tile.cuh -- one 16x8 pixel tile of the shading pass: everything of the megakernel except how ONE light is sampled.
//
// shade_tile() is the body of every shading kernel (vkr_shading_kernel.cu: projected solid angle sampling, the path the
// benchmark runs; vkr_related_work_kernel.cu: the related-work techniques). It stages the constant block, splits the CTA into
// shading and trace warps, reads the G-buffer, sets up LTC frame and noise stream, loops over the lights through the
// LightShader functor, resolves the shadow rays and runs the output stage (src/shaders/shading_pass.frag.glsl:824-893).
// See vkr_shading_kernel.cu for the execution model. Compile with -fmad=false (see vkr_device_math.cuh).
#pragma once
#include <cuda_fp16.h>
#include "vkr_shade_common.cuh"
#include "vkr_ray_stream.cuh"

namespace vkr {

constexpr int kTileW = 16, kTileH = 8, kShadeThreads = kTileW * kTileH;
static_assert(kShadeThreads == 32 * kShadeWarps, "one shading warp per 8x4 patch");
constexpr int kTraceThreads = 32 * kTraceWarps;
constexpr int kShadeRegs = 128, kTraceRegs = 56;   // registers per thread of the shading and the trace warps after the split (setmaxnreg; DESIGN.md)
// Dynamic shared memory of a tile: the constant block (constants_smem_bytes), then, with shadow rays, the ray streams of the shading warps (these
// bytes) and the traversal stacks of the trace lanes (stack_depth ints each). tile_smem_bytes() (vkr_tile_launch.cuh) sizes launches by it.
VKR_DEV constexpr size_t tile_streams_bytes(bool optimal) { return sizeof(float) * stream_floats_per_warp(optimal) * kShadeWarps; }

// LightShader: void operator()(bool on, const shading_point&, const ltc_state&, const unsigned char* light, noise_stream&,
//   const shading_kernel_params&, const unsigned char* cb, uint32_t px, uint32_t py, ray_producer&, pixel_sum&, int lane) const
// -- one polygonal light for the warp's 32 pixels; control flow must be warp-uniform (`on` masks lanes).
template <int MAXP, bool OPTIMAL, bool TRACE, bool LIGHT_TEXTURES = false, class LightShader>
VKR_DEV void shade_tile(const shading_kernel_params& p, const LightShader& shade) {
	__builtin_assume(threadIdx.x < (unsigned) (TRACE ? kShadeThreads + kTraceThreads : kShadeThreads)); // the kernels' __launch_bounds__, for the inlined body
	extern __shared__ __align__(16) unsigned char smem[];
	unsigned char* cb = smem;                                   // constant block incl. lights
	float* stream_base = reinterpret_cast<float*>(smem + p.constants_smem_bytes);
	int* stack_base = reinterpret_cast<int*>(smem + p.constants_smem_bytes + tile_streams_bytes(OPTIMAL));
	__shared__ __align__(8) unsigned long long mbar;
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	// --- stage the constant block with one bulk async copy (TMA engine), completion on an mbarrier
	const uint32_t mbar_addr = (uint32_t) __cvta_generic_to_shared(&mbar);
	const uint32_t cb_addr = (uint32_t) __cvta_generic_to_shared(cb);
	if (threadIdx.x == 0) {
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mbar_addr));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	if (TRACE && threadIdx.x < kShadeWarps) { // stream control words {head, tail, closed, -}
		int* control = reinterpret_cast<int*>(stream_base + stream_floats_per_warp(OPTIMAL) * threadIdx.x + stream_control_at(OPTIMAL));
		control[0] = 0; control[1] = 0; control[2] = -1; control[3] = 0;
	}
	__syncthreads();
	if (TRACE) {
		// --- role split: from here on the two kinds of warps never meet at a CTA-wide barrier again
		if (warp >= kShadeWarps) {
			asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kTraceRegs));
			const int t = warp - kShadeWarps;
			trace_stream<OPTIMAL>(smem_addr(stream_base + stream_floats_per_warp(OPTIMAL) * (t & (kShadeWarps - 1))), p.bvh_tris,
				smem_addr(stack_base + p.stack_depth * 32 * t + lane), lane, p.stats, p.bvh_nodes_i);
			return;
		}
		asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kShadeRegs));
	}
	if (threadIdx.x == 0) {
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar_addr), "r"(p.constants_bytes) : "memory");
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
			:: "r"(cb_addr), "l"(p.constants), "r"(p.constants_bytes), "r"(mbar_addr) : "memory");
	}
	{
		uint32_t done = 0;
		while (!done) {
			asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0; selp.u32 %0, 1, 0, q; }" : "=r"(done) : "r"(mbar_addr) : "memory");
		}
	}
	// --- pixel of this thread: warps cover 8x4 patches of the 16x8 tile
	const int lx = (warp & 1) * 8 + (lane & 7), ly = (warp >> 1) * 4 + (lane >> 3);
	const int tiles_x = (p.width + kTileW - 1) / kTileW;
	const int tile = p.tile_list ? (int) __ldg(p.tile_list + blockIdx.x) : (int) blockIdx.x;
	const int x = (tile % tiles_x) * kTileW + lx;
	const int y = (tile / tiles_x) * kTileH + ly;
	unsigned long long tile_begin_ns = 0;
	if (p.tile_cost && lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tile_begin_ns));
	const bool in_frame = x < p.width && y < p.height;
	const size_t pixel = in_frame ? ((size_t) y * p.width + x) : 0;
	const size_t plane = (size_t) p.width * p.height;
	const float4 g0 = __ldg(p.gbuffer + pixel), g1 = __ldg(p.gbuffer + plane + pixel);
	const bool valid = in_frame && g1.w != 0.0f;
	const f3 camera = make3(ldf(cb, OFF_CAMERA), ldf(cb, OFF_CAMERA + 4), ldf(cb, OFF_CAMERA + 8));
	const float exposure = ldf(cb, OFF_EXPOSURE);
	f3 color = make3(0.0f, 0.0f, 0.0f);
	shading_point sp;
	sp.position = make3(g0.x, g0.y, g0.z);
	sp.roughness = g0.w;
	sp.normal = make3(g1.x, g1.y, g1.z);
	const int light_stride = L_FIXED + 16 * (MAXP - 1) * 2 + 16 * (MAXP - 3);
	if (p.show_polygonal_lights && in_frame) { // shading_pass.frag.glsl:841-850
		f3 end; float end_w;
		f3 view_direction = make3(0.0f, 0.0f, 0.0f); // only textured lights look at it (:844, 847)
		if (valid) { end = sp.position; end_w = 1.0f; }
		if (!valid || LIGHT_TEXTURES) {
			const float fx = (float) x, fy = (float) y;
			view_direction = make3(
				fmaf(ldf(cb, OFF_PIXEL_TO_RAY + 8), 1.0f, fmaf(ldf(cb, OFF_PIXEL_TO_RAY + 4), fy, ldf(cb, OFF_PIXEL_TO_RAY) * fx)),
				fmaf(ldf(cb, OFF_PIXEL_TO_RAY + 24), 1.0f, fmaf(ldf(cb, OFF_PIXEL_TO_RAY + 20), fy, ldf(cb, OFF_PIXEL_TO_RAY + 16) * fx)),
				fmaf(ldf(cb, OFF_PIXEL_TO_RAY + 40), 1.0f, fmaf(ldf(cb, OFF_PIXEL_TO_RAY + 36), fy, ldf(cb, OFF_PIXEL_TO_RAY + 32) * fx)));
			if (!valid) { end = view_direction; end_w = 0.0f; }
			if (LIGHT_TEXTURES) view_direction = normalize(view_direction);
		}
		for (int li = 0; li != p.light_count; ++li) {
			const unsigned char* light = cb + CONSTANTS_FIXED + li * light_stride;
			if (light_ray_intersection<MAXP - 1>(light, camera, end, end_w))
				color = color + light_radiance<LIGHT_TEXTURES>(p, light, camera, view_direction);
		}
	}
	// --- the warp's ray stream; trace lanes fetch ray origins from it by owner lane
	ray_producer q;
	q.base = smem_addr(stream_base + stream_floats_per_warp(OPTIMAL) * warp); q.fill = 0; q.resolved = 0;
#ifdef VKR_TRACE_STATS
	q.stat_resolve_polls = 0; q.stat_candidates = 0;
#endif
	q.pad0 = false;
	q.pad1 = false;
	if (TRACE) {
		float* origin = stream_base + stream_floats_per_warp(OPTIMAL) * warp + stream_origin_at(OPTIMAL);
		origin[lane] = sp.position.x; origin[32 + lane] = sp.position.y; origin[64 + lane] = sp.position.z;
	}
	pixel_sum acc;
	acc.color = color; acc.light = make3(0.0f, 0.0f, 0.0f); acc.inv_samples = 1.0f / (float) p.sample_count;
	acc.submit_parity = 0u; acc.resolve_parity = 0u; acc.pushed = false;
	__syncwarp(kFullMask);
	if (__any_sync(kFullMask, valid)) {
		ltc_state l = {};
		noise_stream ns;
		ns.z = 0.0f; ns.w = 0.0f; ns.available = 0; ns.sample_index = 0;
		sp.diffuse_albedo = make3(0.0f, 0.0f, 0.0f); sp.fresnel_0 = make3(0.0f, 0.0f, 0.0f);
		sp.outgoing = make3(0.0f, 0.0f, 1.0f); sp.lambert_outgoing = 0.0f;
		if (valid) {
			const float4 g2 = __ldg(p.gbuffer + 2 * plane + pixel), g3 = __ldg(p.gbuffer + 3 * plane + pixel);
			sp.diffuse_albedo = make3(g2.x, g2.y, g2.z);
			sp.fresnel_0 = make3(g3.x, g3.y, g3.z);
			sp.outgoing = normalize(camera - sp.position);
			sp.lambert_outgoing = dot(sp.normal, sp.outgoing);
			get_ltc_coefficients(l, p, cb, sp);
		}
#pragma unroll 1
		for (int li = 0; li != p.light_count; ++li) {
			const unsigned char* light = cb + CONSTANTS_FIXED + li * light_stride;
			shade(valid, sp, l, light, ns, p, cb, (uint32_t) x, (uint32_t) y, q, acc, lane);
		}
	}
	if (TRACE) close_stream<OPTIMAL>(q, lane, acc, p.stats);
	color = acc.color;
	if (p.tile_cost && lane == 0) { // what this tile cost: the slowest of its four shading warps (which wait for their shadow rays)
		unsigned long long now; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
		const unsigned long long ns = now - tile_begin_ns;
		atomicMax(p.tile_cost + tile, (uint32_t) (ns > 0xffffffffull ? 0xffffffffull : ns));
	}
	if (!in_frame) return;
	f3 final_color = color;
	if (isnan(color.x) || isnan(color.y) || isnan(color.z) || isinf(color.x) || isinf(color.y) || isinf(color.z))
		final_color = make3(1.0f / exposure, 0.0f / exposure, 0.8f / exposure);
	f3 out_color = make3(final_color.x * exposure, final_color.y * exposure, final_color.z * exposure);
	out_color = output_stage(out_color, ldu(cb, OFF_FRAME_BITS), p.output_srgb != 0);
	const float4 texel = make_float4(out_color.x, out_color.y, out_color.z, 1.0f);
	p.out[pixel] = texel;
	// the other GPUs' copies of the frame: a warp writes four 128-byte row segments per peer, straight over NVLink
	for (int k = 0; k < p.out_peer_count; ++k) p.out_peers[k][pixel] = texel;
}

} // namespace vkr
