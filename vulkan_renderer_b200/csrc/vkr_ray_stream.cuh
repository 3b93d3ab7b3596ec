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
#include "vkr_anchor.cuh"

namespace vkr {

// Anchored shadow rays (vkr_anchor.cuh): rays start at the siblings of their pixel's origin path that the light's cone touches instead of at the root.
// A compile-time edition of the kernels (-DVKR_ANCHORED=1); frames are bit-identical either way.
#ifndef VKR_ANCHORED
#define VKR_ANCHORED 0
#endif

#ifndef VKR_RING
#define VKR_RING 256
#endif
constexpr int kRing = VKR_RING;              // entries per shading warp (power of two)
constexpr unsigned kFullMask = 0xffffffffu;
#ifndef VKR_TRACE_GROUPS
#define VKR_TRACE_GROUPS 2
#endif
constexpr int kShadeWarps = 4, kTraceWarps = 4 * VKR_TRACE_GROUPS;   // per CTA; trace warp t serves the stream of shading warp t & 3
constexpr unsigned kPending = 0xffu;
#ifndef VKR_BVH_WIDTH
#define VKR_BVH_WIDTH 2   // children per node of the shadow BVH the trace warps walk; 4 = experimental variant (see trace_stream)
#endif
// The node loop is left once fewer than this many lanes of a trace warp descend (lane utilisation only, never results). On an H100 (400 W) the C3 frame
// took 381.4 / 381.5 ms with 8, 388.6 / 391.2 ms with 16 and 442.7 / 443.1 ms with 24 (second frame of two alternating runs each, same frame hash).
#ifndef VKR_NODE_LOOP_MIN_LANES
#define VKR_NODE_LOOP_MIN_LANES 8
#endif
constexpr int kNodeLoopMinLanes = VKR_NODE_LOOP_MIN_LANES;
// Tuning knobs of the trace warps' round (lane utilisation only, never results): a new batch of rays is set up once at least VKR_REFILL_MIN_LANES lanes are
// free (or none is busy): ray set-up is a long divergent stretch that should run with many lanes; VKR_LEAF_ONCE: a round tests one leaf per lane, a second
// leaf waits for the next round, when more lanes have one.
#ifndef VKR_REFILL_MIN_LANES
#define VKR_REFILL_MIN_LANES 1
#endif
// 1 (default): the decisions at the end of a node visit -- which child is entered, what is pushed, when the stack is popped, the leaf that is put aside --
// are written as predicated instructions (inline PTX) instead of an if / else chain: no divergent branch with its BSSY / BRA / BSYNC inside the visit.
// 0 keeps the C++ form (the anchored and 4-wide editions need it).
#ifndef VKR_LEAN_NODE_STEP
#define VKR_LEAN_NODE_STEP (!VKR_ANCHORED && VKR_BVH_WIDTH == 2)
#endif
#ifndef VKR_LEAF_ONCE
#define VKR_LEAF_ONCE 0
#endif
// 0: a lane leaves the node loop with the first leaf it meets (one leaf reference is picked up after the loop) instead of putting one leaf aside and descending on
#ifndef VKR_LEAF_POSTPONE
#define VKR_LEAF_POSTPONE 1
#endif
#ifndef VKR_STACK_TOP_IN_REGISTER
#define VKR_STACK_TOP_IN_REGISTER 0
#endif
#ifndef VKR_TRACE_RELOAD_RAY
#define VKR_TRACE_RELOAD_RAY 0
#endif
// The four shading warps of a CTA can walk their sample loop in loose lock step (a named barrier per iteration: 1 = per sample pair, 2 = per technique),
// so that they fetch the loop's 32 KB of instructions together instead of four times. Only tiles in which all four warps have pixels to shade use it
// (the barrier needs all of them).
#ifndef VKR_SHADING_LOCKSTEP
#define VKR_SHADING_LOCKSTEP 0
#endif
#ifndef VKR_NODE_LOOP_CHECK_EVERY
#define VKR_NODE_LOOP_CHECK_EVERY 1   // power of two: the node loop counts its descending lanes every this many steps
#endif
VKR_DEV void shading_lockstep_barrier() {
#if defined(__CUDA_ARCH__)
	asm volatile("bar.sync 1, 128;" ::: "memory");
#endif
}
// 1: the trace warps walk the quantised node pairs (32 bytes, vkr_trace.cuh) instead of the float pairs: half the bytes per visit, bit-identical frames,
// but more instructions per visit and more triangle tests behind the fatter boxes. Kept as a compile-time edition; not with anchored rays or the 4-wide variant.
#ifndef VKR_QUANTISED_NODES
#define VKR_QUANTISED_NODES 0
#endif
// 1 (default): the trace warps walk the interleaved node pairs (vkr_trace.cuh: the two children's numbers side by side) instead of the plain float pairs.
// Bit-identical frames either way. On an H100 (SXM, 700 W) the C3 frame takes 396.1 - 396.4 ms with them and 400.9 - 404.2 ms with the plain pairs
// (tools/build_variant.sh + tools/quick_time.py, steady-state frames of two alternating runs each), worth the second copy of the pairs made at scene load.
#ifndef VKR_INTERLEAVED_NODES
#define VKR_INTERLEAVED_NODES (!VKR_ANCHORED && !VKR_QUANTISED_NODES && VKR_BVH_WIDTH == 2)
#endif
#if VKR_ANCHORED && VKR_BVH_WIDTH != 2
#error "anchored rays walk node pairs"
#endif
#if VKR_LEAN_NODE_STEP && (VKR_ANCHORED || VKR_BVH_WIDTH != 2 || VKR_STACK_TOP_IN_REGISTER)
#error "the predicated node step: not with anchored rays, 4-wide nodes or the stack top in a register (-DVKR_LEAN_NODE_STEP=0)"
#endif
#if VKR_INTERLEAVED_NODES && (VKR_ANCHORED || VKR_QUANTISED_NODES || VKR_BVH_WIDTH != 2)
#error "interleaved node pairs: not with anchored rays, quantised pairs or 4-wide nodes"
#endif
#ifndef VKR_RESOLVE_SLEEP_NS
#define VKR_RESOLVE_SLEEP_NS 512
#endif

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
// anchored rays: per entry the sibling mask of its ray; per pixel (lane) the origin path, its tail and length, and the cone + mask of the light being sampled
VKR_DEV constexpr int stream_mask_at(bool optimal) { return stream_control_at(optimal) + 4; }
VKR_DEV constexpr int stream_path_at(bool optimal) { return stream_mask_at(optimal) + kRing; }      // [kPathLevels + 2][32]: entries, then tail, then count
VKR_DEV constexpr int stream_cone_at(bool optimal) { return stream_path_at(optimal) + 32 * (kPathLevels + 2); }   // [6][32]: axis xyz, cos2_valid, len2_valid, mask
VKR_DEV constexpr size_t stream_floats_per_warp(bool optimal) { return VKR_ANCHORED ? (size_t) stream_cone_at(optimal) + 6 * 32 : (size_t) stream_control_at(optimal) + 4; }

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
	bool cone_set;   // this lane has stored a cone and a sibling mask for the light it is sampling (set_light_cone); else its rays keep all siblings
	bool lockstep;   // warp-uniform: this tile's shading warps keep in step (VKR_SHADING_LOCKSTEP)
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
		__nanosleep(VKR_RESOLVE_SLEEP_NS);
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

#define OPTIMAL_STREAM_HAS_CONE(q) ((q).cone_set)
// Called by a light shader at the start of a light (warp-convergent; `on` = this lane samples the light): the cone around the light as seen from the
// pixel and the siblings of the pixel's origin path that the cone touches, for submit() to hand to the rays. vertices: world-space vertices of the light,
// 16 bytes apart. Light shaders that do not call it leave all siblings to their rays.
template <bool TRACE, bool OPTIMAL>
VKR_DEV void set_light_cone(ray_producer& q, int lane, bool on, f3 origin, const unsigned char* vertices, int vertex_count, const float4* __restrict__ nodes) {
#if VKR_ANCHORED
	if constexpr (TRACE) {
		q.cone_set = false;
		if (on) {
			const light_cone c = make_light_cone(origin, vertices, vertex_count);
			if (c.enabled) {
				const uint32_t path = q.base + 4u * (uint32_t) stream_path_at(OPTIMAL) + 4u * (uint32_t) lane;
				const int count = (int) lds_u32(path + 128u * (uint32_t) (kPathLevels + 1));
				const uint32_t siblings = cull_siblings(nodes, origin, c, count, [&](int k) { return lds_u32(path + 128u * (uint32_t) k); });
				const uint32_t ca = q.base + 4u * (uint32_t) stream_cone_at(OPTIMAL) + 4u * (uint32_t) lane;
				sts_f(ca, c.axis.x); sts_f(ca + 128u, c.axis.y); sts_f(ca + 256u, c.axis.z); sts_f(ca + 384u, c.cos2_valid); sts_f(ca + 512u, c.len2_valid); sts_u32(ca + 640u, siblings);
				q.cone_set = true;
			}
		}
	}
#endif
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
#if VKR_ANCHORED
				{ // the siblings this ray has to look at: the light's mask if the ray is inside the cone the mask was made for (vkr_anchor.cuh), else all
					uint32_t siblings = kAllSiblings;
					if (OPTIMAL_STREAM_HAS_CONE(q)) {
						const uint32_t ca = q.base + 4u * (uint32_t) stream_cone_at(OPTIMAL) + 4u * (uint32_t) lane;
						const f3 axis = make3(lds_f(ca), lds_f(ca + 128u), lds_f(ca + 256u));
						const float aw = dot(axis, dir_world), ww = dot(dir_world, dir_world);
						if (aw > 0.0f && aw * aw >= lds_f(ca + 384u) * ww && tmax * tmax * ww <= lds_f(ca + 512u)) siblings = lds_u32(ca + 640u);
					}
					sts_u32(q.base + 4u * (uint32_t) stream_mask_at(OPTIMAL) + 4u * e, siblings);
				}
#endif
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
template <bool OPTIMAL>
VKR_DEV void trace_stream(const uint32_t base, const float4* __restrict__ nodes, const float4* __restrict__ tris, const uint32_t stack_bottom, int lane, unsigned long long* stats = nullptr,
	const uint4* __restrict__ nodes_q = nullptr, f3 grid_min = f3(), f3 grid_scale = f3(), const float4* __restrict__ nodes_i = nullptr)
{
#ifdef VKR_TRACE_STATS
	unsigned st_rays = 0, st_hits = 0, st_cache_hits = 0, st_visits = 0, st_leaves = 0, st_tris = 0, st_iters = 0, st_node_iters = 0, st_known = 0, st_polls = 0, st_siblings = 0;
#endif
	const unsigned lt_mask = (1u << lane) - 1u;
	const float tmin = 1.0e-3f; // shading_pass.frag.glsl:124
	const uint32_t bytes = base + 4u * stream_bytes_at(OPTIMAL);
	const uint32_t origin = base + 4u * stream_origin_at(OPTIMAL);
	const uint32_t control = base + 4u * stream_control_at(OPTIMAL);
	// The stack is addressed through ONE loop-carried register with a kTraversalDone sentinel at the bottom, so a pop
	// never needs an "empty" test.
	uint32_t top = stack_bottom;
#if VKR_STACK_TOP_IN_REGISTER
	// The top element lives in a register: a pop hands it out at once and refills the register with a load whose result is not needed before the next
	// pop or push, so the latency of the shared-memory load (the address of the next node hangs on it) is off the critical path of the step.
	int stack_top = kTraversalDone;
	auto push = [&](int v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(top), "r"(stack_top) : "memory"); top += 128u; stack_top = v; };
	auto pop = [&]() { const int v = stack_top; top -= 128u; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(stack_top) : "r"(top) : "memory"); return v; };
#else
	auto push = [&](int v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(top), "r"(v) : "memory"); top += 128u; };
	auto pop = [&]() { int v; top -= 128u; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(top) : "memory"); return v; };
#endif
	int ticket = -1;             // >= 0: index of the entry this lane will trace next, not published yet
	uint32_t entry = 0;          // slot of the ray in flight
	bool active = false;         // a ray is in flight
	bool hit = false;
	bool finished = false;       // the stream is closed and this lane's ticket lies beyond its end
	int node = kTraversalDone, leaf = 0;
#if VKR_ANCHORED
	uint32_t pending = 0u;       // levels of the origin path whose siblings this ray still has to visit (deepest first)
	uint32_t path = 0u;          // shared-memory address of the origin path of the ray's pixel
#endif
	int cached_triangle = -1;    // slot of the last triangle that occluded a ray of this lane
#if VKR_TRACE_RELOAD_RAY
	// origin and direction are not kept across the node loop (which only needs the slab form of the ray): the leaf tests read them again from the
	// ring, six registers less per trace lane
	unsigned own_lane = 0;
#else
	f3 o = make3(0.0f, 0.0f, 0.0f), d = make3(0.0f, 0.0f, 1.0f);
#endif
	float tmax = 0.0f;
#if VKR_QUANTISED_NODES
	ray_grid r = make_ray_grid(make3(0.0f, 0.0f, 0.0f), make3(0.0f, 0.0f, 1.0f), grid_min, grid_scale);
#else
	ray_slabs r = make_slabs<false>(make3(0.0f, 0.0f, 0.0f), make3(0.0f, 0.0f, 1.0f));
#endif
	while (true) {
		// --- lanes whose ray has terminated draw a ticket and start on it as soon as it is published
		const bool wants = !active && ticket < 0 && !finished;
		const unsigned want = __ballot_sync(kFullMask, wants);
#if VKR_REFILL_MIN_LANES > 1
		const unsigned busy = __ballot_sync(kFullMask, active);
		const bool refill = busy == 0u || __popc(~busy) >= VKR_REFILL_MIN_LANES;   // warp-uniform
#else
		const bool refill = true;
#endif
		if (want && refill) {
			const int leader = __ffs(want) - 1;
			int first = 0;
			if (lane == leader) first = atom_add_shared(control, __popc(want));
			first = __shfl_sync(kFullMask, first, leader);
			if (wants) ticket = first + __popc(want & lt_mask);
		}
		if (ticket >= 0 && refill) {
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
#if VKR_TRACE_RELOAD_RAY
					own_lane = own & 31u;
					const f3 o = make3(lds_f(oa), lds_f(oa + 128u), lds_f(oa + 256u));
					const f3 d = make3(lds_f(ea + 4u * S_DX), lds_f(ea + 4u * S_DY), lds_f(ea + 4u * S_DZ));
#else
					o = make3(lds_f(oa), lds_f(oa + 128u), lds_f(oa + 256u));
					d = make3(lds_f(ea + 4u * S_DX), lds_f(ea + 4u * S_DY), lds_f(ea + 4u * S_DZ));
#endif
					tmax = lds_f(ea + 4u * S_TMAX);
					active = true;
					hit = false;
					node = kTraversalDone; leaf = 0;
#if VKR_ANCHORED
					pending = 0u;
#endif
					float t;
#ifdef VKR_NULL_TRACE   // diagnostic edition: every ray is a miss at once -- what is left is the time of the shading warps and the ring (the frame is wrong, of course)
					if (false) {
#else
					if (tmax > tmin) { // tmax <= tmin / NaN: undefined in Vulkan, defined as "miss" (DESIGN.md)
#endif
#ifndef VKR_NO_OCCLUDER_CACHE
						if (cached_triangle >= 0 && ray_triangle(tris + 3 * (size_t) cached_triangle, o, d, tmin, tmax, &t)) { hit = true; VKR_STAT(st_cache_hits); }
#else
						if (false) {}
#endif
						else {
#if VKR_QUANTISED_NODES
							r = make_ray_grid(o, d, grid_min, grid_scale);
#elif VKR_INTERLEAVED_NODES
							r = make_clamped_slabs(o, d);   // no NaN slab distance: the integer min / max of ray_box_pair<true> (vkr_trace.cuh)
#else
							r = make_slabs<false>(o, d);   // shading rays: no direction component below 2^-64 but zero (vkr_trace.cuh)
#endif
							top = stack_bottom; push(kTraversalDone);
#if VKR_ANCHORED
							// start at the end of the pixel's origin path; the siblings along it follow when the stack runs empty
							path = base + 4u * (uint32_t) stream_path_at(OPTIMAL) + 4u * (own & 31u);
							const uint32_t count = lds_u32(path + 128u * (uint32_t) (kPathLevels + 1));
							pending = lds_u32(base + 4u * (uint32_t) stream_mask_at(OPTIMAL) + 4u * entry) & ((1u << count) - 1u);   // count <= kPathLevels < 32
							node = (int) lds_u32(path + 128u * (uint32_t) kPathLevels);
							if (node < 0) { leaf = node; node = pop(); }
#else
							node = 0;
#endif
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
#if VKR_NODE_LOOP_CHECK_EVERY > 1
		unsigned node_steps = 0u;
#endif
		// --- descend until this lane holds two leaves or is out of nodes
#if VKR_BVH_WIDTH == 4
		// EXPERIMENTAL variant (tools/build_variant.sh ... "-DVKR_BVH_WIDTH=4" with VKR_BVH_WIDTH=4 in the environment when the scene is loaded): 128-byte
		// nodes with four children (vkr_bvh.h: host_bvh4), half as many steps per ray. The nearest hit child is entered, the others go on the stack
		// (leaves too: pop() hands them back like any reference). The node step is bvh4_descend_step() of vkr_trace.cuh, shared with occluded4(), which is tested
		// on the CPU; this warp loop around it was written without GPU access.
		while (node >= 0 && node != kTraversalDone) {
			VKR_STAT(st_visits);
			if ((__activemask() & lt_mask) == 0u) VKR_STAT(st_node_iters);
			node = bvh4_descend_step(nodes, node, r, tmin, tmax, push); // nearest hit child; the other hit children are on the stack now
			if (node == kTraversalDone) node = pop();
			if (node < 0 && leaf == 0) { // postpone the first leaf, keep descending
				leaf = node;
				node = pop();
			}
			if (kNodeLoopMinLanes > 0 && __popc(__activemask()) < kNodeLoopMinLanes) break;
		}
#else
#if VKR_ANCHORED
		while (node >= 0 && (node != kTraversalDone || (pending != 0u && active && !hit))) {
			int skip = 2;   // the child of this pair that is not looked at: none
			if (node == kTraversalDone) { // the stack is empty: on to the deepest sibling of the origin path that is left, i.e. a visit of its parent pair without the path's child
				const int k = 31 - __clz((int) pending);
				pending &= ~(1u << k);
				const uint32_t e = lds_u32(path + 128u * (uint32_t) k);
				node = (int) (e >> 1); skip = (int) (e & 1u);
				top = stack_bottom; push(kTraversalDone);
				VKR_STAT(st_siblings);
			}
#else
		while ((unsigned) node < (unsigned) kTraversalDone) {   // node >= 0 && node != kTraversalDone, one compare
			const int skip = 2;
#endif
			float tn0, tn1;
			VKR_STAT(st_visits);
			if ((__activemask() & lt_mask) == 0u) VKR_STAT(st_node_iters);
#if VKR_QUANTISED_NODES
			float4 q0, q1;   // one 32-byte pair: six words of 16-bit box coordinates, two references
			ldg_32_bytes(reinterpret_cast<const float4*>(nodes_q) + 2 * (size_t) node, q0, q1);
			const int ref0 = __float_as_int(q1.z), ref1 = __float_as_int(q1.w);
			const bool h0 = ray_box_grid(__float_as_uint(q0.x), __float_as_uint(q0.y), __float_as_uint(q0.z), r, tmin, tmax, &tn0);
			const bool h1 = ray_box_grid(__float_as_uint(q0.w), __float_as_uint(q1.x), __float_as_uint(q1.y), r, tmin, tmax, &tn1);
#elif VKR_INTERLEAVED_NODES
			// one interleaved pair (vkr_trace.cuh): the slab arithmetic of both children side by side
			const float4* nd = reinterpret_cast<const float4*>(reinterpret_cast<const char*>(nodes_i) + (size_t) ((uint32_t) node << 6));
			float4 q0, q1, q2, q3;
			ldg_32_bytes(nd, q0, q1); ldg_32_bytes(nd + 2, q2, q3);
			const int ref0 = __float_as_int(q3.x), ref1 = __float_as_int(q3.y);
			bool h0, h1;
			{
				const float a[8] = { q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w }, b[4] = { q2.x, q2.y, q2.z, q2.w };
				ray_box_pair<true>(a, b, r, tmin, tmax, &h0, &h1, &tn0, &tn1);   // 0 < tmin < tmax: rays with tmax <= tmin never start
			}
#else
#if VKR_LEAN_NODE_STEP
			// the node's address as base + 32-bit byte offset (a tree has fewer than 2^26 pairs: vkr_host.cpp), so that the step needs no 64-bit multiply
			const float4* nd = reinterpret_cast<const float4*>(reinterpret_cast<const char*>(nodes) + (size_t) ((uint32_t) node << 6));
#else
			const float4* nd = nodes + 4 * (size_t) node;
#endif
			float4 q0, q1, q2, q3;
			ldg_32_bytes(nd, q0, q1); ldg_32_bytes(nd + 2, q2, q3);
			const int ref0 = __float_as_int(q3.x), ref1 = __float_as_int(q3.y);
			const bool h0 = ray_box(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, r, tmin, tmax, &tn0) && skip != 0;
			const bool h1 = ray_box(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, r, tmin, tmax, &tn1) && skip != 1;
#endif
#if VKR_LEAN_NODE_STEP
			{ // The same decisions as below, written out as predicates: no divergent branch (BSSY / BRA / BSYNC) in the step, the far child is stored and the
			  // stack is popped under predicates. (h0, h1 and the distances come from ray_box(); tn <= tf is false for NaN like there.)
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
#if VKR_LEAF_POSTPONE
					// postpone the first leaf, keep descending
					"setp.lt.s32 take, %1, 0;\n\tsetp.eq.and.s32 take, %2, 0, take;\n\t"
					"@take mov.b32 %2, %1;\n\t@take sub.u32 %0, %0, 128;\n\t@take ld.shared.b32 %1, [%0];\n\t"
#endif
					"}"
					: "+r"(top), "=&r"(node), "+r"(leaf) : "r"(h0i), "r"(h1i), "f"(tn0), "f"(tn1), "r"(ref0), "r"(ref1) : "memory");
			}
#else
			if (h0 && h1) {
				const bool swap = tn1 < tn0;   // nearer child first: occluders close to the surface end the query early
				node = swap ? ref1 : ref0;
				push(swap ? ref0 : ref1);
			}
			else if (h0) node = ref0;
			else if (h1) node = ref1;
			else node = pop();
#endif
#if !VKR_LEAN_NODE_STEP && VKR_LEAF_POSTPONE
			if (node < 0 && leaf == 0) { // postpone the first leaf, keep descending
				leaf = node;
				node = pop();
			}
#endif
			// lanes that are done or hold two leaves wait at the loop exit: once too few are left descending, let
			// everybody test triangles and fetch new rays (affects lane utilisation only, not results)
#if VKR_NODE_LOOP_CHECK_EVERY > 1
			if ((++node_steps & (VKR_NODE_LOOP_CHECK_EVERY - 1)) != 0) continue;   // the head count costs four instructions of a step: look every other step only
#endif
			if (kNodeLoopMinLanes > 0 && __popc(__activemask()) < kNodeLoopMinLanes) break;
		}
#endif
		__syncwarp(kFullMask);
#if !VKR_LEAF_POSTPONE
		if (active && node < 0 && leaf == 0) { leaf = node; node = pop(); }
#endif
		// --- leaves: `leaf` and possibly `node` (a second leaf)
#if VKR_LEAF_ONCE
		if (leaf != 0) {
#else
		while (leaf != 0) {
#endif
			const int first = (leaf & 0x7fffffff) >> 4, count = leaf & 15;
			float t;
#if VKR_TRACE_RELOAD_RAY
			const uint32_t oa = origin + 4u * own_lane, ea = base + 4u * entry;
			const f3 o = make3(lds_f(oa), lds_f(oa + 128u), lds_f(oa + 256u));
			const f3 d = make3(lds_f(ea + 4u * S_DX), lds_f(ea + 4u * S_DY), lds_f(ea + 4u * S_DZ));
#endif
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
#if VKR_ANCHORED
		if (active && node == kTraversalDone && leaf == 0 && (hit || pending == 0u)) {
#else
		if (active && node == kTraversalDone && leaf == 0) {
#endif
			st_release_u8(bytes + kRing + entry, hit ? 1u : 0u);
			if (hit) VKR_STAT(st_hits);
			active = false;
		}
		__syncwarp(kFullMask);
	}
#ifdef VKR_TRACE_STATS
	stat_flush(stats, 0, st_rays); stat_flush(stats, 1, st_hits); stat_flush(stats, 2, st_cache_hits); stat_flush(stats, 3, st_visits); stat_flush(stats, 4, st_leaves);
	stat_flush(stats, 5, st_tris); stat_flush(stats, 6, st_iters); stat_flush(stats, 7, st_node_iters); stat_flush(stats, 8, st_known); stat_flush(stats, 9, st_polls); stat_flush(stats, 13, st_siblings);
#endif
}

} // namespace vkr
