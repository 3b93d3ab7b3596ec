// vkr_ray_stream.cuh -- shadow-ray streams of the warp-specialised shading megakernel.
//
// A CTA has two kinds of warps (vkr_shading_kernel.cu): SHADING warps sample the lights and evaluate BRDF and MIS
// weights for an 8x4 pixel patch, TRACE warps do nothing but BVH traversal. They talk through one ring buffer per
// shading warp in shared memory:
//
//   shading warp (producer)                  ring of kRing entries                     2 trace warps (consumers)
//   submit(): __ballot_sync compaction  -->  dir, tmax, owner, contribution  -->  every idle LANE draws a ticket
//   publishes `tail` after every sample      result byte: 0xFF pending / 0 / 1        (atomicAdd on `head`), waits until
//   resolve(): adds contributions of    <--                                  <--   tail > ticket, traces, stores result
//   finished entries, oldest first
//
// Trace lanes refill themselves individually, so traversal runs at full warp width whatever the ray lengths are and
// however many pixels of the patch are idle (background, lights below the horizon); a trace warp never waits for the
// end of a batch. The shading warp only resolves when it needs ring space (or at the end of a light), adding the
// contributions of its own pixel strictly in submission order, which keeps the floating-point sums identical to the
// reference's sequential loop (shading_pass.frag.glsl:608-637). Trace warps give their registers to the shading warps
// (setmaxnreg), which is what lets 24 warps per SM live where the monolithic kernel had 12.
#pragma once
#include "vkr_trace.cuh"

namespace vkr {

constexpr int kRing = 256;                   // entries per shading warp (power of two)
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kShadeWarps = 4, kTraceWarps = 8;   // per CTA; trace warp t serves the stream of shading warp t & 3
constexpr unsigned kPending = 0xffu;
// The node loop is left once fewer than this many lanes of a trace warp descend (lane utilisation only, never results). On an H100 (400 W) the C3 frame
// took 381.4 / 381.5 ms with 8, 388.6 / 391.2 ms with 16 and 442.7 / 443.1 ms with 24 (second frame of two alternating runs each, same frame hash).
constexpr int kNodeLoopMinLanes = 8;
constexpr unsigned kResolveSleepNs = 512;     // a shading warp's nap while shadow-ray results it needs are still pending

// In-kernel statistics (vkr_trace_counter_t, include/vkr_b200.h): compiled in with -DVKR_TRACE_STATS (the counters edition of the quad-light
// kernels, vkr_shading_kernel_stats.cu -> vkr_shading_pass_run_with_counters); the kernels that are timed carry none of it.
#ifdef VKR_TRACE_STATS
#define VKR_STAT(x) (++(x))
#define VKR_STAT_ADD(x, n) ((x) += (n))
#else
#define VKR_STAT(x) ((void) 0)
#define VKR_STAT_ADD(x, n) ((void) 0)
#endif
VKR_DEV void stat_flush(unsigned long long* stats, int index, unsigned value) {
#if defined(VKR_TRACE_STATS) && defined(__CUDA_ARCH__)
	value = __reduce_add_sync(kFullMask, value);
	if ((threadIdx.x & 31) == 0 && value != 0u && stats) atomicAdd(stats + index, (unsigned long long) value);
#endif
}

// Shared memory of one stream, as float offsets from its base. 7 (or 10, MIS_HEURISTIC_OPTIMAL) float arrays, owner and
// result bytes, 96 floats of ray origins, 4 ints of control.
enum : int {
	S_DX = 0, S_DY = kRing, S_DZ = 2 * kRing, S_TMAX = 3 * kRing,     // ray direction (world), far end = light plane
	S_CX = 4 * kRing, S_CY = 5 * kRing, S_CZ = 6 * kRing,              // contribution if the ray is unoccluded
	S_OX = 7 * kRing, S_OY = 8 * kRing, S_OZ = 9 * kRing               // contribution if it is occluded (OPTIMAL only)
};
VKR_DEV constexpr int stream_bytes_at(bool optimal) { return (optimal ? 10 : 7) * kRing; }           // owner[kRing] bytes: lane of the owning pixel; bit 7: known to be occluded (n.w <= 0)
VKR_DEV constexpr int stream_origin_at(bool optimal) { return stream_bytes_at(optimal) + 2 * kRing / 4; }  // after result[kRing] bytes: kPending / 0 visible / 1 occluded
VKR_DEV constexpr int stream_control_at(bool optimal) { return stream_origin_at(optimal) + 96; }     // {head: next ticket, tail: entries published, closed: -1 or the final tail, -}
VKR_DEV constexpr size_t stream_floats_per_warp(bool optimal) { return (size_t) stream_control_at(optimal) + 4; }

VKR_DEV uint32_t smem_addr(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }
VKR_DEV uint32_t lds_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
VKR_DEV void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
VKR_DEV float lds_f(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory"); return v; }
VKR_DEV void sts_f(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" :: "r"(a), "f"(v) : "memory"); }
VKR_DEV unsigned lds_u8(uint32_t a) { unsigned v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
VKR_DEV void sts_u8(uint32_t a, unsigned v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
VKR_DEV int ld_acquire(uint32_t a) { int v; asm volatile("ld.acquire.cta.shared::cta.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
VKR_DEV void st_release(uint32_t a, int v) { asm volatile("st.release.cta.shared::cta.b32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
VKR_DEV unsigned ld_acquire_u8(uint32_t a) { unsigned v; asm volatile("ld.acquire.cta.shared::cta.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
VKR_DEV void st_release_u8(uint32_t a, unsigned v) { asm volatile("st.release.cta.shared::cta.u8 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
VKR_DEV int atom_add_shared(uint32_t a, int v) { int old; asm volatile("atom.relaxed.cta.shared::cta.add.s32 %0, [%1], %2;" : "=r"(old) : "r"(a), "r"(v) : "memory"); return old; }

// ---------------------------------------------------------------------------------------------------------------------
// Producer side (shading warps)
struct ray_producer {
	uint32_t base;   // shared-memory address of the stream
	int fill;        // warp-uniform: entries written and published so far (absolute index; slot = index & (kRing - 1))
	int resolved;    // warp-uniform: entries below this index have been added to their pixels, their slots are free
#ifdef VKR_TRACE_STATS
	unsigned stat_resolve_polls, stat_candidates;
#endif
	// Two bytes no code reads, set once in shade_tile(). Without them nvcc allocates the registers of 14 of the 24 kernels of every
	// vkr_shading_kernel.cu object differently (the same instructions, in another order); with them those kernels keep their tuned machine code.
	bool pad0, pad1;
};

// Radiance sums of one pixel. The reference adds the samples of a light into a per-light sum, scales it by 1/S and
// adds it to the pixel (shading_pass.frag.glsl:695-711, 853-857). Shadow-ray results arrive late, so the per-light sum
// is closed lazily: every entry carries the parity of "lights with entries" of its pixel, and when the parity of the
// next resolved entry differs from that of the previous one, the previous light is complete.
struct pixel_sum {
	f3 color;          // pixel radiance so far (all closed lights)
	f3 light;          // sum over the resolved samples of the light that is currently open
	float inv_samples; // 1 / S
	unsigned submit_parity, resolve_parity;  // bit 5 of the owner byte
	bool pushed;       // this pixel has pushed an entry for the light being sampled
};
VKR_DEV void close_light(pixel_sum& acc) {
	acc.color = acc.color + acc.light * acc.inv_samples;
	acc.light = make3(0.0f, 0.0f, 0.0f);
}

// Adds the contributions of entries [q.resolved, min(q.resolved + 32, q.fill)) to their owners, oldest first; waits for
// the trace warps where results are still pending.
template <bool OPTIMAL>
VKR_DEV void resolve_chunk(ray_producer& q, int lane, pixel_sum& acc) {
	const uint32_t bytes = q.base + 4u * stream_bytes_at(OPTIMAL);
	const int first = q.resolved;
	const int n = min(32, q.fill - first);
	const uint32_t slot = (uint32_t) (first + lane) & (kRing - 1);
	const bool valid = lane < n;
	while (true) {
		const unsigned r = valid ? ld_acquire_u8(bytes + kRing + slot) : 0u;
		if (!__any_sync(kFullMask, r == kPending)) break;
		VKR_STAT(q.stat_resolve_polls);
		__nanosleep(kResolveSleepNs);
	}
	const unsigned own = valid ? (lds_u8(bytes + slot) & 31u) : 32u;
	unsigned mine = __ballot_sync(kFullMask, valid);
#pragma unroll
	for (int b = 0; b != 5; ++b) {
		const unsigned bits = __ballot_sync(kFullMask, (own >> b) & 1u);
		mine &= ((lane >> b) & 1) ? bits : ~bits;
	}
	while (mine) {
		const uint32_t e = (uint32_t) (first + __ffs(mine) - 1) & (kRing - 1);
		mine &= mine - 1;
		const uint32_t a = q.base + 4u * e;
		const unsigned parity = lds_u8(bytes + e) & 32u;
		if (parity != acc.resolve_parity) { close_light(acc); acc.resolve_parity = parity; }
		if (!lds_u8(bytes + kRing + e)) acc.light = acc.light + make3(lds_f(a + 4u * S_CX), lds_f(a + 4u * S_CY), lds_f(a + 4u * S_CZ));
		else if (OPTIMAL) acc.light = acc.light + make3(lds_f(a + 4u * S_OX), lds_f(a + 4u * S_OY), lds_f(a + 4u * S_OZ));
	}
	q.resolved = first + n;
	__syncwarp(kFullMask);
}

// Warp-convergent: every lane calls it once per candidate sample. has = this lane contributes something.
// need_trace = visibility is not known yet (n.w > 0); otherwise the sample is known to be occluded.
// finish (warp-uniform) = end of a light. Nothing waits here: the light's sum is closed when its last entry resolves.
template <bool TRACE, bool OPTIMAL>
VKR_DEV void submit(ray_producer& q, int lane, bool has, bool need_trace, f3 dir_world, float tmax, f3 c_visible, f3 c_occluded, pixel_sum& acc, bool finish) {
	if constexpr (!TRACE) { // no shadow rays: visibility = (n.w > 0), nothing is ever pending, add in place
		if (has) {
			if (need_trace) acc.light = acc.light + c_visible;
			else if (OPTIMAL) acc.light = acc.light + c_occluded;
		}
		if (finish) close_light(acc);
	}
	else {
		const bool push = has && (need_trace || OPTIMAL);
		if (has) VKR_STAT(q.stat_candidates);
		const unsigned mask = __ballot_sync(kFullMask, push);
		if (mask) {
			const int k = __popc(mask);
			while (q.fill + k - q.resolved > kRing) resolve_chunk<OPTIMAL>(q, lane, acc);
			if (push) {
				const uint32_t e = (uint32_t) (q.fill + __popc(mask & ((1u << lane) - 1u))) & (kRing - 1);
				const uint32_t a = q.base + 4u * e;
				sts_f(a + 4u * S_DX, dir_world.x); sts_f(a + 4u * S_DY, dir_world.y); sts_f(a + 4u * S_DZ, dir_world.z); sts_f(a + 4u * S_TMAX, tmax);
				sts_f(a + 4u * S_CX, c_visible.x); sts_f(a + 4u * S_CY, c_visible.y); sts_f(a + 4u * S_CZ, c_visible.z);
				if (OPTIMAL) { sts_f(a + 4u * S_OX, c_occluded.x); sts_f(a + 4u * S_OY, c_occluded.y); sts_f(a + 4u * S_OZ, c_occluded.z); }
				const uint32_t bytes = q.base + 4u * stream_bytes_at(OPTIMAL);
				sts_u8(bytes + e, (unsigned) lane | acc.submit_parity | (need_trace ? 0u : 128u));
				// Every entry is completed by the trace lane that drew its ticket, also the ones known to be occluded (optimal MIS): a slot whose result
				// were set here could be resolved and reused while the lane holding its ticket has not looked at it yet, and that lane would then trace
				// the newer entry a second time and store its result late, possibly onto a still newer entry of the slot.
				sts_u8(bytes + kRing + e, kPending);
				acc.pushed = true;
			}
			q.fill += k;
			__syncwarp(kFullMask);
			if (lane == 0) st_release(q.base + 4u * stream_control_at(OPTIMAL) + 4u, q.fill);
		}
		if (finish && acc.pushed) { acc.submit_parity ^= 32u; acc.pushed = false; }
	}
}

// End of the tile: resolves what is still pending, closes the last light and tells the trace warps that no ticket
// >= fill will ever be served.
template <bool OPTIMAL>
VKR_DEV void close_stream(ray_producer& q, int lane, pixel_sum& acc, unsigned long long* stats = nullptr) {
	while (q.resolved != q.fill) resolve_chunk<OPTIMAL>(q, lane, acc);
	close_light(acc);
	__syncwarp(kFullMask);
	if (lane == 0) st_release(q.base + 4u * stream_control_at(OPTIMAL) + 8u, q.fill);
#ifdef VKR_TRACE_STATS
	stat_flush(stats, 10, lane == 0 ? (unsigned) q.fill : 0u);
	stat_flush(stats, 11, lane == 0 ? q.stat_resolve_polls : 0u);   // warp-uniform count
	stat_flush(stats, 12, q.stat_candidates);
#endif
}

// ---------------------------------------------------------------------------------------------------------------------
// Consumer side (trace warps): runs until the stream is closed and drained. stack = shared-memory address of this
// lane's column of the warp's traversal stack (128 B between levels = one slot per lane).
// The trace warps walk the interleaved node pairs (vkr_trace.cuh: the two children's numbers side by side). Frames are bit-identical with the plain
// float pairs; on an H100 (SXM, 700 W) the C3 frame takes 396.1 - 396.4 ms with them and 400.9 - 404.2 ms with the plain pairs (steady-state frames of
// two alternating runs each), worth the second copy of the pairs made at scene load. nodes_i comes last because nvcc orders the kernel parameter loads
// by the arguments, and this order keeps the counters edition's machine code.
template <bool OPTIMAL>
VKR_DEV void trace_stream(const uint32_t base, const float4* __restrict__ tris, const uint32_t stack_bottom, int lane, unsigned long long* stats, const float4* __restrict__ nodes_i)
{
#ifdef VKR_TRACE_STATS
	unsigned st_rays = 0, st_hits = 0, st_cache_hits = 0, st_visits = 0, st_leaves = 0, st_tris = 0, st_iters = 0, st_node_iters = 0, st_known = 0, st_polls = 0;
#endif
	const unsigned lt_mask = (1u << lane) - 1u;
	const float tmin = 1.0e-3f; // shading_pass.frag.glsl:124
	const uint32_t bytes = base + 4u * stream_bytes_at(OPTIMAL);
	const uint32_t origin = base + 4u * stream_origin_at(OPTIMAL);
	const uint32_t control = base + 4u * stream_control_at(OPTIMAL);
	// The stack is addressed through ONE loop-carried register with a kTraversalDone sentinel at the bottom, so a pop
	// never needs an "empty" test.
	uint32_t top = stack_bottom;
	auto push = [&](int v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(top), "r"(v) : "memory"); top += 128u; };
	auto pop = [&]() { int v; top -= 128u; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(top) : "memory"); return v; };
	int ticket = -1;             // >= 0: index of the entry this lane will trace next, not published yet
	uint32_t entry = 0;          // slot of the ray in flight
	bool active = false;         // a ray is in flight
	bool hit = false;
	bool finished = false;       // the stream is closed and this lane's ticket lies beyond its end
	int node = kTraversalDone, leaf = 0;
	int cached_triangle = -1;    // slot of the last triangle that occluded a ray of this lane
	f3 o = make3(0.0f, 0.0f, 0.0f), d = make3(0.0f, 0.0f, 1.0f);
	float tmax = 0.0f;
	ray_slabs r = make_slabs<false>(make3(0.0f, 0.0f, 0.0f), make3(0.0f, 0.0f, 1.0f));
	while (true) {
		// --- lanes whose ray has terminated draw a ticket and start on it as soon as it is published
		const bool wants = !active && ticket < 0 && !finished;
		const unsigned want = __ballot_sync(kFullMask, wants);
		if (want) {
			const int leader = __ffs(want) - 1;
			int first = 0;
			if (lane == leader) first = atom_add_shared(control, __popc(want));
			first = __shfl_sync(kFullMask, first, leader);
			if (wants) ticket = first + __popc(want & lt_mask);
		}
		if (ticket >= 0) {
			if (ticket < ld_acquire(control + 4u)) {
				entry = (uint32_t) ticket & (kRing - 1);
				ticket = -1;
				const unsigned own = lds_u8(bytes + entry);
				if (own & 128u) { // known to be occluded (n.w <= 0): no ray, but the ticket holder is the one who completes the entry (see submit())
					VKR_STAT(st_known);
					st_release_u8(bytes + kRing + entry, 1u);
				}
				else {
					VKR_STAT(st_rays);
					const uint32_t oa = origin + 4u * (own & 31u), ea = base + 4u * entry;
					o = make3(lds_f(oa), lds_f(oa + 128u), lds_f(oa + 256u));
					d = make3(lds_f(ea + 4u * S_DX), lds_f(ea + 4u * S_DY), lds_f(ea + 4u * S_DZ));
					tmax = lds_f(ea + 4u * S_TMAX);
					active = true;
					hit = false;
					node = kTraversalDone; leaf = 0;
					float t;
					if (tmax > tmin) { // tmax <= tmin / NaN: undefined in Vulkan, defined as "miss" (DESIGN.md)
						if (cached_triangle >= 0 && ray_triangle(tris + 3 * (size_t) cached_triangle, o, d, tmin, tmax, &t)) { hit = true; VKR_STAT(st_cache_hits); }
						else {
							r = make_clamped_slabs(o, d);   // no NaN slab distance: the integer min / max of ray_box_pair<true> (vkr_trace.cuh)
							top = stack_bottom; push(kTraversalDone);
							node = 0;
						}
					}
				}
			}
			else {
				const int end = ld_acquire(control + 8u);
				if (end >= 0 && ticket >= end) { finished = true; ticket = -1; }
			}
		}
		if (!__any_sync(kFullMask, active)) {
			if (__all_sync(kFullMask, finished)) break;
			if (lane == 0) VKR_STAT(st_polls);
			__nanosleep(100); // nothing published yet: leave the issue slots to the other warps
			continue;
		}
		if (lane == 0) VKR_STAT(st_iters);
		// --- descend until this lane holds two leaves or is out of nodes
		while ((unsigned) node < (unsigned) kTraversalDone) {   // node >= 0 && node != kTraversalDone, one compare
			float tn0, tn1;
			VKR_STAT(st_visits);
			if ((__activemask() & lt_mask) == 0u) VKR_STAT(st_node_iters);
			// one interleaved pair: the slab arithmetic of both children side by side. The node's address is base + 32-bit byte offset (a tree has fewer
			// than 2^26 pairs: vkr_host.cpp), so that the step needs no 64-bit multiply.
			const float4* nd = reinterpret_cast<const float4*>(reinterpret_cast<const char*>(nodes_i) + (size_t) ((uint32_t) node << 6));
			float4 q0, q1, q2, q3;
			ldg_32_bytes(nd, q0, q1); ldg_32_bytes(nd + 2, q2, q3);
			const int ref0 = __float_as_int(q3.x), ref1 = __float_as_int(q3.y);
			bool h0, h1;
			{
				const float a[8] = { q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w }, b[4] = { q2.x, q2.y, q2.z, q2.w };
				ray_box_pair<true>(a, b, r, tmin, tmax, &h0, &h1, &tn0, &tn1);   // 0 < tmin < tmax: rays with tmax <= tmin never start
			}
			{ // The decisions at the end of the visit, written as predicated instructions (inline PTX) instead of an if / else chain, so the step has no
			  // divergent branch (BSSY / BRA / BSYNC): if both children are hit, the nearer one is entered (occluders close to the surface end the query
			  // early) and the other is pushed; if one is hit, it is entered; if none, the stack is popped. The first leaf met is put aside in `leaf` and the
			  // lane keeps descending. (tn <= tf is false for NaN like in ray_box().)
				const int h0i = h0, h1i = h1;
				asm volatile("{\n\t.reg .pred h0, h1, both, none, second, take;\n\t.reg .b32 far;\n\t"
					"setp.ne.b32 h0, %3, 0;\n\tsetp.ne.b32 h1, %4, 0;\n\t"
					"setp.lt.f32 second, %6, %5;\n\t"                 // child 1 is nearer ...
					"and.pred both, h0, h1;\n\t"
					"or.pred none, h0, h1;\n\tnot.pred none, none;\n\t"
					"not.pred take, h0;\n\tor.pred second, second, take;\n\tand.pred second, second, h1;\n\t"   // ... or the only one hit: it is entered
					"selp.b32 %1, %8, %7, second;\n\tselp.b32 far, %7, %8, second;\n\t"
					"@both st.shared.b32 [%0], far;\n\t@both add.u32 %0, %0, 128;\n\t"
					"@none sub.u32 %0, %0, 128;\n\t@none ld.shared.b32 %1, [%0];\n\t"
					// postpone the first leaf, keep descending
					"setp.lt.s32 take, %1, 0;\n\tsetp.eq.and.s32 take, %2, 0, take;\n\t"
					"@take mov.b32 %2, %1;\n\t@take sub.u32 %0, %0, 128;\n\t@take ld.shared.b32 %1, [%0];\n\t"
					"}"
					: "+r"(top), "=&r"(node), "+r"(leaf) : "r"(h0i), "r"(h1i), "f"(tn0), "f"(tn1), "r"(ref0), "r"(ref1) : "memory");
			}
			// lanes that are done or hold two leaves wait at the loop exit: once too few are left descending, let
			// everybody test triangles and fetch new rays (affects lane utilisation only, not results)
			if (__popc(__activemask()) < kNodeLoopMinLanes) break;
		}
		__syncwarp(kFullMask);
		// --- leaves: `leaf` and possibly `node` (a second leaf)
		while (leaf != 0) {
			const int first = (leaf & 0x7fffffff) >> 4, count = leaf & 15;
			float t;
			VKR_STAT(st_leaves); VKR_STAT_ADD(st_tris, (unsigned) count);
			for (int i = 0; i != count; ++i)
				if (ray_triangle(tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) { hit = true; cached_triangle = first + i; }
			leaf = 0;
			if (hit) node = kTraversalDone;
			else if (node < 0) {
				leaf = node;
				node = pop();
			}
		}
		// --- a ray ends when it hit something or ran out of nodes
		if (active && node == kTraversalDone && leaf == 0) {
			st_release_u8(bytes + kRing + entry, hit ? 1u : 0u);
			if (hit) VKR_STAT(st_hits);
			active = false;
		}
		__syncwarp(kFullMask);
	}
#ifdef VKR_TRACE_STATS
	stat_flush(stats, 0, st_rays); stat_flush(stats, 1, st_hits); stat_flush(stats, 2, st_cache_hits); stat_flush(stats, 3, st_visits); stat_flush(stats, 4, st_leaves);
	stat_flush(stats, 5, st_tris); stat_flush(stats, 6, st_iters); stat_flush(stats, 7, st_node_iters); stat_flush(stats, 8, st_known); stat_flush(stats, 9, st_polls);
	stat_flush(stats, 13, 0u);   // slot 13 counted the sibling steps of anchored rays, an edition that is gone; flushing a zero keeps this edition's machine code
#endif
}

} // namespace vkr
