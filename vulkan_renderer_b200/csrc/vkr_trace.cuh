// vkr_trace.cuh -- software BVH2 traversal for shadow (any-hit) and primary (closest-hit) rays.
//
// Replaces the VK_KHR_ray_query calls of the reference (src/shaders/shading_pass.frag.glsl:120-138)
// and the driver-built acceleration structure (src/scene.c:142-406). No RT cores, no OptiX.
//
// Layout in HBM (built once on the host, vkr_bvh.cpp):
//   node  = 64 B = 4 x float4: both children's boxes + both child references ("node pair"),
//           so one 64-B sector-aligned fetch decides both children.
//             q0 = (c0.x, c0.y, c0.z, h0.x)  q1 = (h0.y, h0.z, c1.x, c1.y)
//             q2 = (c1.z, h1.x, h1.y, h1.z)  q3 = (ref0, ref1, -, -) as int bits
//           c = box centre, h = half extent (rounded up)
//           ref >= 0: inner node index; ref < 0: leaf, (ref & 0x7fffffff) = first_triangle << 4 | count
//   tri   = 48 B = 3 x float4: v0.xyz e1.x | e1.yz e2.xy | e2.z - - -   (e1 = v1 - v0, e2 = v2 - v0)
//
// Arithmetic: the TRIANGLE predicate is part of the parity contract (DESIGN.md: Moeller-Trumbore,
// fp32, fixed operation order, no culling, open interval); hit/miss is the OR over all triangles and
// does not depend on traversal order. The BOX test only has to be conservative. With boxes stored as
// centre c and half extent h the near/far slab distances are (c - o)/d -+ h/|d|: three FFMAs per axis
// and no per-axis min/max, which moves the work from the ALU pipe (FMNMX, the busiest pipe of the
// traversal loop) to the FMA pipe. Its rounding error is below 1/64 of the padding the builder adds
// to every box (vkr_bvh.cpp), so no triangle the predicate accepts is culled.
// The shading kernel's trace warps (ray_box_pair<true>) take the max of the near and the min of the far
// distances as signed integers on the float bits (sm_90 DPX: VIMNMX3). That is exact for 0 < tmin < tmax
// and slab distances that are never NaN, which the set-up guarantees by clamping the reciprocal to +-2^64
// (make_clamped_slabs): with |id| <= 2^64, c*id - o*id is finite for coordinates below 2^60 and its
// rounding stays the few ulp the padding covers; a zero component then tests the origin against that
// axis's slab instead of dropping the axis.
#pragma once
#include "vkr_device_math.cuh"

namespace vkr {

struct bvh_view {
	const float4* nodes;
	const float4* tris;
	const uint32_t* tri_ids; // original triangle index per slot (closest-hit only)
	uint32_t tri_count;
};

constexpr int kMaxStackDepth = 64;      // the builder guarantees depth < 62 (vkr_host.cpp)
constexpr int kTraversalDone = 0x7fffffff;

VKR_DEV bool ray_triangle(const float4* __restrict__ tri, f3 o, f3 d, float tmin, float tmax, float* out_t) {
	const float4 a = __ldg(tri), b = __ldg(tri + 1), c = __ldg(tri + 2);
	const f3 p0 = make3(a.x, a.y, a.z);
	const f3 e1 = make3(a.w, b.x, b.y);
	const f3 e2 = make3(b.z, b.w, c.x);
	const f3 pv = cross(d, e2);
	const float det = dot(e1, pv);
	if (det == 0.0f) return false;
	const float inv_det = 1.0f / det;
	const f3 tv = o - p0;
	const float u = dot(tv, pv) * inv_det;
	if (!(u >= 0.0f && u <= 1.0f)) return false;
	const f3 qv = cross(tv, e1);
	const float v = dot(d, qv) * inv_det;
	if (!(v >= 0.0f && u + v <= 1.0f)) return false;
	const float t = dot(e2, qv) * inv_det;
	if (!(t > tmin && t < tmax)) return false;
	*out_t = t;
	return true;
}

// One 32-byte half of a node as two 128-bit loads through the read-only path (LDG.E.128.CONSTANT, the widest load sm_90 has): a node pair is
// four of these, all of it in the two sectors of one 64-byte aligned pair.
VKR_DEV void ldg_32_bytes(const float4* __restrict__ p, float4& a, float4& b) {
	a = __ldg(p); b = __ldg(p + 1);
}

// Reciprocal for the slab test only: the box test has to be conservative, not exact (header), so the hardware's approximation does (MUFU.RCP: relative
// error 2^-23, i.e. one more rounding of the size the padding of the boxes is made for; denormal components flush to zero, whose reciprocal is infinite,
// and an infinite or NaN slab distance leaves the slab unconstrained). Saves three IEEE divisions (range check, refinement, slow path) per ray set-up.
VKR_DEV float unguarded_slab_reciprocal(float x) {
#if defined(__CUDA_ARCH__) && !defined(VKR_EXACT_SLAB_RECIPROCAL)
	float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
#else
	return 1.0f / x;
#endif
}
// Components below 2^-64 in magnitude get an infinite reciprocal too, which drops that axis from the test (always conservative). A finite but huge
// reciprocal (1/FLT_MIN = 2^126) makes o / d overflow to infinity while c / d - o / d is finite, and the slab test culls boxes the ray crosses.
// With |id| <= 2^64 no product or fma of the slab test overflows for coordinates below 2^60.
VKR_DEV float slab_reciprocal(float x) {
	const float y = unguarded_slab_reciprocal(x);
	return (fabsf(x) < 5.421010862427522e-20f) ? copysignf(__int_as_float(0x7f800000), x) : y;   // 2^-64
}

// Ray in the form the slab test wants: id = 1/d, oid = o/d. GUARDED = false is for the compile-time editions of the trace warps' loop
// (vkr_ray_stream.cuh): their rays point from a surface point to a point on a light, normalised, so a nonzero component is far above 2^-64 for any
// scene with coordinates above 1e-12.
struct ray_slabs { f3 id, oid; };
template <bool GUARDED = true>
VKR_DEV ray_slabs make_slabs(f3 o, f3 d) {
	ray_slabs r;
	if (GUARDED) r.id = make3(slab_reciprocal(d.x), slab_reciprocal(d.y), slab_reciprocal(d.z));
	else r.id = make3(unguarded_slab_reciprocal(d.x), unguarded_slab_reciprocal(d.y), unguarded_slab_reciprocal(d.z));
	r.oid = make3(o.x * r.id.x, o.y * r.id.y, o.z * r.id.z);
	return r;
}
// Set-up for the integer min / max of ray_box_pair<true>: the reciprocal clamped to [-2^64, 2^64] (zero and denormal components get +-2^64 with
// their sign, a NaN component -2^64), so every slab distance is finite or +-infinity and never NaN: with finite operands neither o * id nor an fma of
// the slab test can be NaN, an overflow only saturates. For coordinates below 2^60 in magnitude nothing overflows (2^60 * 2^64 = 2^124), and the
// rounding of c * id - o * id is a few ulp of the coordinates, the same error the unclamped test has (header). The clamp is conservative: an axis whose
// component is below 2^-64 keeps the slab [(c - h - o) * 2^64, (c + h - o) * 2^64] (times the sign). A triangle in the box hit at distance t lies at
// least the padding (2^-16 of the scene extent) inside the slab, and the ray moves less than t * 2^-64 along that axis, so the slab reaches from below
// -(pad - t 2^-64) 2^64 < 0 to above (pad - t 2^-64) 2^64 > t as long as t < pad * 2^63 -- 2^47 scene extents. Exactly zero components, which the
// unclamped test drops from the test (NaN slab distances), now test the origin against the slab, so such rays may visit fewer pairs; their answers stay.
VKR_DEV float clamped_slab_reciprocal(float x) {
	const float big = 18446744073709551616.0f;   // 2^64
	return fminf(fmaxf(unguarded_slab_reciprocal(x), -big), big);
}
VKR_DEV ray_slabs make_clamped_slabs(f3 o, f3 d) {
	ray_slabs r;
	r.id = make3(clamped_slab_reciprocal(d.x), clamped_slab_reciprocal(d.y), clamped_slab_reciprocal(d.z));
	r.oid = make3(o.x * r.id.x, o.y * r.id.y, o.z * r.id.z);
	return r;
}

// Signed 32-bit max / min of three (sm_90 DPX: one VIMNMX3) and of two. The host build of this header runs the same integer semantics.
VKR_DEV int imax3_s32(int a, int b, int c) {
#if defined(__CUDA_ARCH__)
	return __vimax3_s32(a, b, c);
#else
	const int m = (a > b) ? a : b; return (m > c) ? m : c;
#endif
}
VKR_DEV int imin3_s32(int a, int b, int c) {
#if defined(__CUDA_ARCH__)
	return __vimin3_s32(a, b, c);
#else
	const int m = (a < b) ? a : b; return (m < c) ? m : c;
#endif
}
VKR_DEV int imax_s32(int a, int b) { return (a > b) ? a : b; }
VKR_DEV int imin_s32(int a, int b) { return (a < b) ? a : b; }

// Conservative slab test (see header) of the box with centre c and half extent h. Returns the entry distance in
// *t_near. NaNs (inf - inf for axis-parallel rays) drop out of fminf/fmaxf, which leaves that slab unconstrained.
VKR_DEV bool ray_box(float cx, float cy, float cz, float hx, float hy, float hz, const ray_slabs& r, float tmin, float tmax, float* t_near) {
	const float mx = fmaf(cx, r.id.x, -r.oid.x), my = fmaf(cy, r.id.y, -r.oid.y), mz = fmaf(cz, r.id.z, -r.oid.z);
	const float ax = fabsf(r.id.x), ay = fabsf(r.id.y), az = fabsf(r.id.z);
	const float tn = fmaxf(fmaxf(fmaf(-hx, ax, mx), fmaf(-hy, ay, my)), fmaxf(fmaf(-hz, az, mz), tmin));
	const float tf = fminf(fminf(fmaf(hx, ax, mx), fmaf(hy, ay, my)), fminf(fmaf(hz, az, mz), tmax));
	*t_near = tn;
	return tn <= tf;
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// Interleaved node pairs: the same 64 bytes per pair with the two children's numbers next to each other,
//   float 0..7   c0.x c1.x  c0.y c1.y  c0.z c1.z  h0.x h1.x        float 8..15   h0.y h1.y  h0.z h1.z  ref0 ref1  -  -
// so that the loads of a visit leave (child 0, child 1) side by side and the slab arithmetic of both children is one pairwise routine, ray_box_pair().
// Each of its 18 FFMAs is an IEEE fma with the operands of ray_box(), so a visit decides exactly as with the plain pairs.
VKR_DEV void interleave_node_pair(const float4* __restrict__ pair, float* out16) {
	const float4 q0 = pair[0], q1 = pair[1], q2 = pair[2], q3 = pair[3];
	out16[0] = q0.x; out16[1] = q1.z; out16[2] = q0.y; out16[3] = q1.w; out16[4] = q0.z; out16[5] = q2.x;   // centres
	out16[6] = q0.w; out16[7] = q2.y; out16[8] = q1.x; out16[9] = q2.z; out16[10] = q1.y; out16[11] = q2.w; // half extents
	out16[12] = q3.x; out16[13] = q3.y; out16[14] = 0.0f; out16[15] = 0.0f;
}
// (d0, d1) = (a0, a1) * s + (c0, c1): two FFMAs (sm_90 has no packed fp32 FMA)
VKR_DEV void fma_pair(float& d0, float& d1, float a0, float a1, float s, float c0, float c1) {
	d0 = fmaf(a0, s, c0); d1 = fmaf(a1, s, c1);
}
// ray_box() for the two children of an interleaved pair (a = floats 0..7, b = floats 8..11)
// DPX = true (the trace warps of the shading kernel): near and far distances are combined as signed integers on the float bits, one VIMNMX3 + one
// VIMNMX per child and side instead of three FMNMX. That gives fmaxf / fminf's answers when (1) no distance is NaN -- the slabs come from
// make_clamped_slabs() -- and (2) 0 < tmin < tmax: the max then includes the positive tmin, and positive floats order like their bits as integers, so
// tn is exactly fmaxf's; if a far distance is negative (or -0) the integer min is some negative value (or -0) where fminf's is the most negative one,
// and both fail tn <= tf; otherwise all far distances are positive and the min is exact. The order of two hit children compares two positive tn.
template <bool DPX = false>
VKR_DEV void ray_box_pair(const float (&a)[8], const float (&b)[4], const ray_slabs& r, float tmin, float tmax, bool* h0, bool* h1, float* tn0, float* tn1) {
	float mx0, mx1, my0, my1, mz0, mz1, nx0, nx1, ny0, ny1, nz0, nz1, fx0, fx1, fy0, fy1, fz0, fz1;
	const float nox = -r.oid.x, noy = -r.oid.y, noz = -r.oid.z;
	fma_pair(mx0, mx1, a[0], a[1], r.id.x, nox, nox); fma_pair(my0, my1, a[2], a[3], r.id.y, noy, noy); fma_pair(mz0, mz1, a[4], a[5], r.id.z, noz, noz);
	const float ax = fabsf(r.id.x), ay = fabsf(r.id.y), az = fabsf(r.id.z);
	fma_pair(nx0, nx1, a[6], a[7], -ax, mx0, mx1); fma_pair(ny0, ny1, b[0], b[1], -ay, my0, my1); fma_pair(nz0, nz1, b[2], b[3], -az, mz0, mz1);
	fma_pair(fx0, fx1, a[6], a[7], ax, mx0, mx1); fma_pair(fy0, fy1, b[0], b[1], ay, my0, my1); fma_pair(fz0, fz1, b[2], b[3], az, mz0, mz1);
	float tf0, tf1;
	if (DPX) {
		const int lo = __float_as_int(tmin), hi = __float_as_int(tmax);
		*tn0 = __int_as_float(imax_s32(imax3_s32(__float_as_int(nx0), __float_as_int(ny0), __float_as_int(nz0)), lo));
		*tn1 = __int_as_float(imax_s32(imax3_s32(__float_as_int(nx1), __float_as_int(ny1), __float_as_int(nz1)), lo));
		tf0 = __int_as_float(imin_s32(imin3_s32(__float_as_int(fx0), __float_as_int(fy0), __float_as_int(fz0)), hi));
		tf1 = __int_as_float(imin_s32(imin3_s32(__float_as_int(fx1), __float_as_int(fy1), __float_as_int(fz1)), hi));
	}
	else {
		*tn0 = fmaxf(fmaxf(nx0, ny0), fmaxf(nz0, tmin)); *tn1 = fmaxf(fmaxf(nx1, ny1), fmaxf(nz1, tmin));
		tf0 = fminf(fminf(fx0, fy0), fminf(fz0, tmax)); tf1 = fminf(fminf(fx1, fy1), fminf(fz1, tmax));
	}
	*h0 = *tn0 <= tf0; *h1 = *tn1 <= tf1;
}
// Per-thread any-hit query over interleaved pairs (16 floats each): the reference form of the trace warps' loop, run on the CPU against occluded().
// DPX = true is the form the shading kernel runs (clamped set-up, integer min / max); false the fmaxf form with the guarded set-up.
template <bool DPX = false>
VKR_DEV bool occluded_interleaved(const float* __restrict__ pairs16, const float4* __restrict__ tris, f3 o, f3 d, float tmin, float tmax, int* stack, int stride, int* visits) {
	if (!(tmax > tmin)) return false;
	const ray_slabs r = DPX ? make_clamped_slabs(o, d) : make_slabs(o, d);
	int sp = 0, node = 0;
	float t, tn0, tn1;
	while (true) {
		if (node < 0) {
			const int first = (node & 0x7fffffff) >> 4, count = node & 15;
			for (int i = 0; i != count; ++i)
				if (ray_triangle(tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) return true;
			if (sp == 0) return false;
			--sp; node = stack[sp * stride];
			continue;
		}
		if (visits) ++*visits;
		const float* w = pairs16 + 16 * (size_t) node;
		const float a[8] = { w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7] }, b[4] = { w[8], w[9], w[10], w[11] };
		bool h0, h1;
		ray_box_pair<DPX>(a, b, r, tmin, tmax, &h0, &h1, &tn0, &tn1);
		const int ref0 = __float_as_int(w[12]), ref1 = __float_as_int(w[13]);
		if (h0 && h1) { const bool swap = tn1 < tn0; stack[sp * stride] = swap ? ref0 : ref1; ++sp; node = swap ? ref1 : ref0; }
		else if (h0) node = ref0;
		else if (h1) node = ref1;
		else { if (sp == 0) return false; --sp; node = stack[sp * stride]; }
	}
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// Quantised node pairs: an edition of the trace warps' loop with half the bytes per visit (VKR_QUANTISED_NODES, vkr_ray_stream.cuh). A pair shrinks from
// 64 to 32 bytes -- one sector per lane -- by storing the two child boxes as 16-bit coordinates on a grid over the scene's bounding box:
//   word 0..2  child 0: x, y, z as (low | high << 16)      word 3..5  child 1      word 6, 7  the two child references (as in the float pairs)
// Boxes are rounded outwards to the grid and one more cell (below), so the test stays conservative; the triangle predicate is untouched and hit / miss
// remains the OR over the triangles it accepts. The ray is taken to grid coordinates once (t is invariant under per-axis scaling), a plane's
// coordinate q becomes the float 2^23 + q with one byte permutation (no integer-to-float conversion), and the slab distance one FFMA:
// (2^23 + q) * id - (2^23 * id + o_grid * id). The rounding of that constant is worth at most 0.504 grid cells -- the extra cell of padding.
struct ray_grid { f3 id, c; unsigned near_x, near_y, near_z; };   // c = -(2^23 * id + o_grid * id); near_*: byte selectors of the plane the ray enters through
constexpr unsigned kGridMagic = 0x4B000000u;   // float 2^23
VKR_DEV ray_grid make_ray_grid(f3 o, f3 d, f3 grid_min, f3 grid_scale) {
	ray_grid g;
	const f3 og = make3((o.x - grid_min.x) * grid_scale.x, (o.y - grid_min.y) * grid_scale.y, (o.z - grid_min.z) * grid_scale.z);
	const f3 dg = make3(d.x * grid_scale.x, d.y * grid_scale.y, d.z * grid_scale.z);
	g.id = make3(slab_reciprocal(dg.x), slab_reciprocal(dg.y), slab_reciprocal(dg.z));
	g.c = make3(-fmaf(8388608.0f, g.id.x, og.x * g.id.x), -fmaf(8388608.0f, g.id.y, og.y * g.id.y), -fmaf(8388608.0f, g.id.z, og.z * g.id.z));
	g.near_x = (dg.x < 0.0f) ? 0x7632u : 0x7610u; g.near_y = (dg.y < 0.0f) ? 0x7632u : 0x7610u; g.near_z = (dg.z < 0.0f) ? 0x7632u : 0x7610u;
	return g;
}
VKR_DEV float grid_plane(unsigned word, unsigned selector) { // float(2^23 + the 16-bit half of `word` that `selector` names)
#if defined(__CUDA_ARCH__)
	return __uint_as_float(__byte_perm(word, kGridMagic, selector));
#else
	return __uint_as_float(kGridMagic | ((selector == 0x7632u) ? (word >> 16) : (word & 0xffffu)));
#endif
}
// Slab test of one quantised child box (its three words). NaNs (a direction component of zero) drop out of fminf / fmaxf as in ray_box().
VKR_DEV bool ray_box_grid(unsigned wx, unsigned wy, unsigned wz, const ray_grid& g, float tmin, float tmax, float* t_near) {
	const float nx = fmaf(grid_plane(wx, g.near_x), g.id.x, g.c.x), ny = fmaf(grid_plane(wy, g.near_y), g.id.y, g.c.y), nz = fmaf(grid_plane(wz, g.near_z), g.id.z, g.c.z);
	const float fx = fmaf(grid_plane(wx, g.near_x ^ 0x0022u), g.id.x, g.c.x), fy = fmaf(grid_plane(wy, g.near_y ^ 0x0022u), g.id.y, g.c.y), fz = fmaf(grid_plane(wz, g.near_z ^ 0x0022u), g.id.z, g.c.z);
	const float tn = fmaxf(fmaxf(nx, ny), fmaxf(nz, tmin));
	const float tf = fminf(fminf(fx, fy), fminf(fz, tmax));
	*t_near = tn;
	return tn <= tf;
}
// One float node pair -> its quantised form (8 words). Used by the quantisation kernel (vkr_lbvh_gpu.cu) and by the CPU tests.
VKR_DEV void quantise_node_pair(const float4* __restrict__ pair, const float* grid_min, const float* grid_scale, unsigned* out8) {
	const float4 q0 = pair[0], q1 = pair[1], q2 = pair[2], q3 = pair[3];
	const float c[2][3] = { { q0.x, q0.y, q0.z }, { q1.z, q1.w, q2.x } }, h[2][3] = { { q0.w, q1.x, q1.y }, { q2.y, q2.z, q2.w } };
	for (int k = 0; k != 2; ++k)
		for (int a = 0; a != 3; ++a) {
			// outwards to the grid, then one cell more; an empty child (negative half extent) stays empty: low > high
			float lo = floorf(((c[k][a] - h[k][a]) - grid_min[a]) * grid_scale[a]) - 1.0f, hi = ceilf(((c[k][a] + h[k][a]) - grid_min[a]) * grid_scale[a]) + 1.0f;
			if (h[k][a] < 0.0f) { lo = 65535.0f; hi = 0.0f; }
			lo = fminf(fmaxf(lo, 0.0f), 65535.0f); hi = fminf(fmaxf(hi, 0.0f), 65535.0f);
			out8[3 * k + a] = (unsigned) lo | ((unsigned) hi << 16);
		}
	out8[6] = __float_as_uint(q3.x); out8[7] = __float_as_uint(q3.y);
}
// Per-thread any-hit query over quantised pairs: the reference form of the trace warps' loop (vkr_ray_stream.cuh), run on the CPU against occluded().
VKR_DEV bool occluded_grid(const unsigned* __restrict__ pairs8, const float4* __restrict__ tris, const float* grid_min, const float* grid_scale, f3 o, f3 d, float tmin, float tmax, int* stack, int stride, int* visits) {
	if (!(tmax > tmin)) return false;
	const ray_grid g = make_ray_grid(o, d, make3(grid_min[0], grid_min[1], grid_min[2]), make3(grid_scale[0], grid_scale[1], grid_scale[2]));
	int sp = 0, node = 0;
	float t, tn0, tn1;
	while (true) {
		if (node < 0) {
			const int first = (node & 0x7fffffff) >> 4, count = node & 15;
			for (int i = 0; i != count; ++i)
				if (ray_triangle(tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) return true;
			if (sp == 0) return false;
			--sp; node = stack[sp * stride];
			continue;
		}
		if (visits) ++*visits;
		const unsigned* w = pairs8 + 8 * (size_t) node;
		const bool h0 = ray_box_grid(w[0], w[1], w[2], g, tmin, tmax, &tn0), h1 = ray_box_grid(w[3], w[4], w[5], g, tmin, tmax, &tn1);
		const int ref0 = (int) w[6], ref1 = (int) w[7];
		if (h0 && h1) { const bool swap = tn1 < tn0; stack[sp * stride] = swap ? ref0 : ref1; ++sp; node = swap ? ref1 : ref0; }
		else if (h0) node = ref0;
		else if (h1) node = ref1;
		else { if (sp == 0) return false; --sp; node = stack[sp * stride]; }
	}
}

// Per-thread any-hit query (probe kernel vkr_trace_shadow_rays); the shading kernel's own traversal loop lives in
// vkr_ray_stream.cuh (trace warps), built from the same ray_box / ray_triangle.
VKR_DEV bool occluded(const bvh_view& bvh, f3 o, f3 d, float tmin, float tmax, int* stack, int stride) {
	if (!(tmax > tmin)) return false;
	const ray_slabs r = make_slabs(o, d);
	int sp = 0;
	int node = 0;
	float t, tn0, tn1;
	while (true) {
		const float4* n = bvh.nodes + 4 * (size_t) node;
		const float4 q0 = __ldg(n), q1 = __ldg(n + 1), q2 = __ldg(n + 2), q3 = __ldg(n + 3);
		const int ref0 = __float_as_int(q3.x), ref1 = __float_as_int(q3.y);
		bool h0 = ray_box(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, r, tmin, tmax, &tn0);
		bool h1 = ray_box(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, r, tmin, tmax, &tn1);
		if (h0 && ref0 < 0) {
			const int first = (ref0 & 0x7fffffff) >> 4, count = ref0 & 15;
			for (int i = 0; i != count; ++i)
				if (ray_triangle(bvh.tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) return true;
			h0 = false;
		}
		if (h1 && ref1 < 0) {
			const int first = (ref1 & 0x7fffffff) >> 4, count = ref1 & 15;
			for (int i = 0; i != count; ++i)
				if (ray_triangle(bvh.tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) return true;
			h1 = false;
		}
		if (h0 && h1) { stack[sp * stride] = ref1; ++sp; node = ref0; }
		else if (h0) node = ref0;
		else if (h1) node = ref1;
		else {
			if (sp == 0) return false;
			--sp; node = stack[sp * stride];
		}
	}
}

// One step through a 4-wide node (vkr_bvh.h: host_bvh4; 8 x float4 per node: child c has centre and half extent at floats [6c, 6c + 6), the four
// references as int bits in the seventh float4). Tests the four boxes, returns the reference of the nearest hit child and hands the other hit
// children (inner nodes and leaves alike) to push(); returns kTraversalDone if no child is hit. Shared by occluded4() below (tested on the CPU)
// and by the experimental 4-wide form of the trace warps' loop (vkr_ray_stream.cuh, VKR_BVH_WIDTH == 4).
template <class Push>
VKR_DEV int bvh4_descend_step(const float4* __restrict__ nodes4, int node, const ray_slabs& r, float tmin, float tmax, Push&& push) {
	const float4* nd = nodes4 + 8 * (size_t) node;
	float4 q0, q1, q2, q3, q4, q5, q6, q7;
	ldg_32_bytes(nd, q0, q1); ldg_32_bytes(nd + 2, q2, q3); ldg_32_bytes(nd + 4, q4, q5); ldg_32_bytes(nd + 6, q6, q7);
	const int ref0 = __float_as_int(q6.x), ref1 = __float_as_int(q6.y), ref2 = __float_as_int(q6.z), ref3 = __float_as_int(q6.w);
	float tn0, tn1, tn2, tn3;
	const bool h0 = ray_box(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, r, tmin, tmax, &tn0);
	const bool h1 = ray_box(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, r, tmin, tmax, &tn1);
	const bool h2 = ray_box(q3.x, q3.y, q3.z, q3.w, q4.x, q4.y, r, tmin, tmax, &tn2);
	const bool h3 = ray_box(q4.z, q4.w, q5.x, q5.y, q5.z, q5.w, r, tmin, tmax, &tn3);
	int best = -1; float best_t = 0.0f;
	if (h0) { best = 0; best_t = tn0; }
	if (h1 && (best < 0 || tn1 < best_t)) { best = 1; best_t = tn1; }
	if (h2 && (best < 0 || tn2 < best_t)) { best = 2; best_t = tn2; }
	if (h3 && (best < 0 || tn3 < best_t)) { best = 3; best_t = tn3; }
	if (h0 && best != 0) push(ref0);
	if (h1 && best != 1) push(ref1);
	if (h2 && best != 2) push(ref2);
	if (h3 && best != 3) push(ref3);
	return (best < 0) ? kTraversalDone : ((best == 0) ? ref0 : ((best == 1) ? ref1 : ((best == 2) ? ref2 : ref3)));
}

// Any-hit query over 4-wide nodes. Same predicate, same answer as occluded(); a step decides four children at once, so a ray takes about half as
// many steps. `steps` counts the nodes fetched (statistics for the tests, may be null).
VKR_DEV bool occluded4(const float4* __restrict__ nodes4, const float4* __restrict__ tris, f3 o, f3 d, float tmin, float tmax, int* stack, int stride, int* steps) {
	if (!(tmax > tmin)) return false;
	const ray_slabs r = make_slabs(o, d);
	int sp = 0;
	int node = 0;
	float t;
	auto push = [&](int ref) { stack[sp * stride] = ref; ++sp; };
	while (true) {
		if (node < 0) { // a leaf
			const int first = (node & 0x7fffffff) >> 4, count = node & 15;
			for (int i = 0; i != count; ++i)
				if (ray_triangle(tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) return true;
			node = kTraversalDone;
		}
		else {
			if (steps) ++*steps;
			node = bvh4_descend_step(nodes4, node, r, tmin, tmax, push);
		}
		if (node == kTraversalDone) {
			if (sp == 0) return false;
			--sp; node = stack[sp * stride];
		}
	}
}

// Closest-hit query, ties in t resolve to the lowest original triangle index (order independent).
VKR_DEV int closest_hit(const bvh_view& bvh, f3 o, f3 d, float tmin, float tmax, int* stack, int stride) {
	const ray_slabs r = make_slabs(o, d);
	int sp = 0;
	int node = 0;
	int best = -1;
	float best_t = tmax;
	float t, tn0, tn1;
	while (true) {
		const float4* n = bvh.nodes + 4 * (size_t) node;
		const float4 q0 = __ldg(n), q1 = __ldg(n + 1), q2 = __ldg(n + 2), q3 = __ldg(n + 3);
		const int ref0 = __float_as_int(q3.x), ref1 = __float_as_int(q3.y);
		// closed upper bound so that equal-t candidates are still visited for the tie rule
		bool h0 = ray_box(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, r, tmin, best_t, &tn0);
		bool h1 = ray_box(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, r, tmin, best_t, &tn1);
#pragma unroll
		for (int c = 0; c != 2; ++c) {
			const int ref = c ? ref1 : ref0;
			const bool h = c ? h1 : h0;
			if (h && ref < 0) {
				const int first = (ref & 0x7fffffff) >> 4, count = ref & 15;
				for (int i = 0; i != count; ++i) {
					if (ray_triangle(bvh.tris + 3 * (size_t) (first + i), o, d, tmin, __int_as_float(0x7f800000), &t)) {
						const int id_ = (int) __ldg(bvh.tri_ids + first + i);
						if (t < best_t || (t == best_t && best >= 0 && id_ < best)) { best_t = t; best = id_; }
					}
				}
				if (c) h1 = false; else h0 = false;
			}
		}
		if (h0 && h1) {
			const bool swap = tn1 < tn0;
			stack[sp * stride] = swap ? ref0 : ref1; ++sp; node = swap ? ref1 : ref0;
		}
		else if (h0) node = ref0;
		else if (h1) node = ref1;
		else {
			if (sp == 0) return best;
			--sp; node = stack[sp * stride];
		}
	}
}

} // namespace vkr
