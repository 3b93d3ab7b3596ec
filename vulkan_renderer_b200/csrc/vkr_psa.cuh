// vkr_psa.cuh -- projected-solid-angle sampling of convex polygons for sm_90a.
//
// Implements the numerical recipe of Peters, "BRDF Importance Sampling for Polygonal Lights"
// (SIGGRAPH 2021) as the reference renderer evaluates it
//   src/shaders/polygon_sampling.glsl:261-805  (ellipses, sector areas, sampling)
//   src/shaders/polygon_clipping.glsl:19-225   (horizon clipping, vertex order per case)
// The recipe (initial guess + exactly two refinement steps, expression order, fma placement)
// is part of the parity contract (SURVEY Appendix C); the code organisation is ours:
// register-resident polygons with compile-time indices only (no local-memory arrays), a
// compile-time vertex bound MAXP, warp-uniform early-outs left to the caller.
#pragma once
#include "vkr_device_math.cuh"

namespace vkr {

template <int MAXP>
struct psa_polygon {
	int vertex_count;
	f2 vertices[MAXP];
	f2 ellipses[MAXP];       // ellipse of the next CCW edge per vertex (sign bit of x = inner)
	f2 inner_ellipse_0;      // x > 0 <=> zenith inside the polygon (central case)
	float sector_psa[MAXP];
	float psa;
};

// Field-wise select between two register-resident polygons (lets one inlined copy of sample_psa serve both)
template <int MAXP>
VKR_DEV psa_polygon<MAXP> select_polygon(bool second, const psa_polygon<MAXP>& a, const psa_polygon<MAXP>& b) {
	psa_polygon<MAXP> r;
	r.vertex_count = second ? b.vertex_count : a.vertex_count;
	r.inner_ellipse_0.x = second ? b.inner_ellipse_0.x : a.inner_ellipse_0.x;
	r.inner_ellipse_0.y = second ? b.inner_ellipse_0.y : a.inner_ellipse_0.y;
	r.psa = second ? b.psa : a.psa;
#pragma unroll
	for (int i = 0; i != MAXP; ++i) {
		r.vertices[i].x = second ? b.vertices[i].x : a.vertices[i].x; r.vertices[i].y = second ? b.vertices[i].y : a.vertices[i].y;
		r.ellipses[i].x = second ? b.ellipses[i].x : a.ellipses[i].x; r.ellipses[i].y = second ? b.ellipses[i].y : a.ellipses[i].y;
		r.sector_psa[i] = second ? b.sector_psa[i] : a.sector_psa[i];
	}
	return r;
}

// Crossing of segment a->b with the horizon plane z = 0 (polygon_clipping.glsl:19-25)
VKR_DEV f3 horizon_crossing(f3 a, f3 b) {
	const float w = a.z / (a.z - b.z);
	return make3(fmaf(w, b.x, fmaf(-w, a.x, a.x)), fmaf(w, b.y, fmaf(-w, a.y, a.y)), 0.0f);
}

// Clips a convex polygon with n in 3..7 (<= MAXP-1) vertices against z >= 0. The slot each
// output vertex lands in follows the reference (the first vertex defines sector 0 later on).
// The first output vertex is repeated at index vc when vc < MAXP. Returns vc (0, or 3..n+1).
template <int MAXP>
VKR_DEV int clip_polygon(int n, f3 (&v)[MAXP]) {
	static_assert(MAXP >= 4 && MAXP <= 8, "light polygons with 3 to 7 vertices");
	f3 in[MAXP - 1];
#pragma unroll
	for (int i = 0; i != MAXP - 1; ++i) in[i] = v[i];
	unsigned bits = 0;
#pragma unroll
	for (int i = 0; i != MAXP - 1; ++i) bits |= (in[i].z > 0.0f && i < n) ? (1u << i) : 0u;
	int vc = 0;
#define P(k) in[k]
#define OUT(slot, value) v[slot] = (value)
#define X(k) horizon_crossing(in[k], in[(k + 1) % VKR_CLIP_N])
	if (n == 3) {
#define VKR_CLIP_N 3
		switch (bits) {
#include "vkr_clip_cases.inc"
		default: vc = 0; break;
		}
#undef VKR_CLIP_N
	}
	if constexpr (MAXP >= 5) if (n == 4) {
#define VKR_CLIP_N 4
		switch (bits) {
#include "vkr_clip_cases.inc"
		default: vc = 0; break;
		}
#undef VKR_CLIP_N
	}
	if constexpr (MAXP >= 6) if (n == 5) {
#define VKR_CLIP_N 5
		switch (bits) {
#include "vkr_clip_cases.inc"
		default: vc = 0; break;
		}
#undef VKR_CLIP_N
	}
	if constexpr (MAXP >= 7) if (n == 6) {
#define VKR_CLIP_N 6
		switch (bits) {
#include "vkr_clip_cases.inc"
		default: vc = 0; break;
		}
#undef VKR_CLIP_N
	}
	if constexpr (MAXP >= 8) if (n == 7) {
#define VKR_CLIP_N 7
		switch (bits) {
#include "vkr_clip_cases.inc"
		default: vc = 0; break;
		}
#undef VKR_CLIP_N
	}
#undef X
#undef OUT
#undef P
#pragma unroll
	for (int i = 3; i != MAXP; ++i)
		if (i == vc) v[i] = v[0];
	return vc;
}

VKR_DEV float fast_positive_atan(float y) { // polygon_sampling.glsl:83-97
	float rx, ry, rz;
	rx = (fabsf(y) > 1.0f) ? (1.0f / fabsf(y)) : fabsf(y);
	ry = rx * rx;
	rz = fmaf(ry, 0.02083509974181652f, -0.08513300120830536f);
	rz = fmaf(ry, rz, 0.18014100193977356f);
	rz = fmaf(ry, rz, -0.3302994966506958f);
	ry = fmaf(ry, rz, 0.9998660087585449f);
	rz = fmaf(-2.0f * ry, rx, kHalfPi);
	rz = (fabsf(y) > 1.0f) ? rz : 0.0f;
	rx = fmaf(rx, ry, rz);
	return (y < 0.0f) ? (kPi - rx) : rx;
}

template <bool BIASED>
VKR_DEV float positive_atan(float tangent) { // :104-111
	if (BIASED) return fast_positive_atan(tangent);
	const float offset = (tangent < 0.0f) ? kPi : 0.0f;
	return atan_poly(tangent) + offset;
}

VKR_DEV float mix_fma(float x, float y, float a) { return fmaf(a, y, fmaf(-a, x, x)); } // :183-185

VKR_DEV float kahan(float a, float b, float c, float d) { // :261-268
	const float cd = c * d;
	const float error = fmaf(c, d, -cd);
	const float result = fmaf(a, b, -cd);
	return result - error;
}
VKR_DEV f2 rotate_90(f2 a) { return make2(-a.y, a.x); }
VKR_DEV bool is_inner_ellipse(f2 e) { return (__float_as_uint(e.x) & 0x80000000u) != 0; }

VKR_DEV f2 ellipse_from_edge(f3 a, f3 b) { // :317-326
	const float nx = kahan(a.y, b.z, a.z, b.y);
	const float ny = kahan(a.z, b.x, a.x, b.z);
	const float nz = kahan(a.x, b.y, a.y, b.x);
	float scaling = 1.0f / nz;
	scaling = (__float_as_uint(nx) & 0x80000000u) ? -scaling : scaling;
	f2 e = make2(nx * scaling, ny * scaling);
	e.x = (nz != 0.0f) ? e.x : __int_as_float(0x7f800000);
	return e;
}
VKR_DEV f2 ellipse_transform(f2 e, f2 p) { // :332-334
	const float d = dot(e, p);
	return make2(fmaf(d, e.x, p.x), fmaf(d, e.y, p.y));
}
VKR_DEV float ellipse_det(f2 e) { return fmaf(e.x, e.x, fmaf(e.y, e.y, 1.0f)); }
VKR_DEV float ellipse_rsqrt_det(f2 e) { return rsqrt_ieee(ellipse_det(e)); }
VKR_DEV float ellipse_direction_factor_rsq(f2 e, f2 dir) {
	const float ed = dot(e, dir);
	const float dd = dot(dir, dir);
	return fmaf(ed, ed, dd);
}
VKR_DEV float ellipse_direction_factor(f2 e, f2 dir) { return rsqrt_ieee(ellipse_direction_factor_rsq(e, dir)); }
VKR_DEV float ellipse_normalized_direction_factor(f2 e, f2 ndir) {
	const float ed = dot(e, ndir);
	return rsqrt_ieee(fmaf(ed, ed, 1.0f));
}

template <bool BIASED>
VKR_DEV float area_between_from_tangents(float inner_rsqrt_det, float inner_tangent, float outer_rsqrt_det, float outer_tangent) { // :377-382
	const float inner_area = inner_rsqrt_det * positive_atan<BIASED>(inner_tangent);
	const float result = fmaf(outer_rsqrt_det, positive_atan<BIASED>(outer_tangent), -inner_area);
	return (result > 0.0f) ? (0.5f * result) : 0.0f;
}
template <bool BIASED>
VKR_DEV float area_between_ellipses_in_sector(f2 inner, float inner_rsqrt_det, f2 outer, float outer_rsqrt_det, f2 dir_0, f2 dir_1) { // :390-397
	const float det_dirs = max_glsl(+0.0f, dot(dir_1, rotate_90(dir_0)));
	const float inner_dot = inner_rsqrt_det * dot(dir_0, ellipse_transform(inner, dir_1));
	const float outer_dot = outer_rsqrt_det * dot(dir_0, ellipse_transform(outer, dir_1));
	return area_between_from_tangents<BIASED>(inner_rsqrt_det, det_dirs / inner_dot, outer_rsqrt_det, det_dirs / outer_dot);
}
template <bool BIASED>
VKR_DEV float ellipse_area_in_sector(f2 e, f2 dir_0, f2 dir_1) { // :405-412
	const float rsd = ellipse_rsqrt_det(e);
	const float det_dirs = max_glsl(+0.0f, dot(dir_1, rotate_90(dir_0)));
	const float edot = rsd * dot(dir_0, ellipse_transform(e, dir_1));
	const float area = 0.5f * rsd * positive_atan<BIASED>(det_dirs / edot);
	return (rsd > 0.0f) ? area : 0.0f;
}

// One comparator of the azimuth sorting network (:421-435); L and R are compile-time slots
template <int L, int R, int MAXP>
VKR_DEV void compare_and_swap(psa_polygon<MAXP>& p) {
	const f2 l = p.vertices[L], r = p.vertices[R];
	const float normal_z = kahan(l.x, -r.y, l.y, -r.x);
	const bool swap = (normal_z == 0.0f) ? (fabsf(p.ellipses[R].x) == __int_as_float(0x7f800000)) : (normal_z > 0.0f);
	p.vertices[L] = swap ? r : l;
	p.vertices[R] = swap ? l : r;
	const f2 el = p.ellipses[L], er = p.ellipses[R];
	p.ellipses[L] = swap ? er : el;
	p.ellipses[R] = swap ? el : er;
}

template <int MAXP>
VKR_DEV void sort_convex_polygon_vertices(psa_polygon<MAXP>& p) { // :440-505, one network per vertex count
	if (p.vertex_count == 3) compare_and_swap<1, 2>(p);
	if constexpr (MAXP >= 4) if (p.vertex_count == 4) compare_and_swap<1, 3>(p);
	if constexpr (MAXP >= 5) if (p.vertex_count == 5) {
		compare_and_swap<2, 4>(p); compare_and_swap<1, 3>(p); compare_and_swap<1, 2>(p); compare_and_swap<0, 3>(p); compare_and_swap<3, 4>(p);
	}
	if constexpr (MAXP >= 6) if (p.vertex_count == 6) {
		compare_and_swap<3, 5>(p); compare_and_swap<2, 4>(p); compare_and_swap<1, 5>(p); compare_and_swap<0, 4>(p); compare_and_swap<4, 5>(p); compare_and_swap<1, 3>(p);
	}
	if constexpr (MAXP >= 7) if (p.vertex_count == 7) {
		compare_and_swap<2, 5>(p); compare_and_swap<1, 6>(p); compare_and_swap<5, 6>(p); compare_and_swap<3, 4>(p); compare_and_swap<0, 4>(p);
		compare_and_swap<4, 6>(p); compare_and_swap<1, 3>(p); compare_and_swap<3, 5>(p); compare_and_swap<4, 5>(p);
	}
	if constexpr (MAXP >= 8) if (p.vertex_count == 8) {
		compare_and_swap<2, 6>(p); compare_and_swap<3, 7>(p); compare_and_swap<1, 5>(p); compare_and_swap<0, 4>(p); compare_and_swap<4, 6>(p);
		compare_and_swap<5, 7>(p); compare_and_swap<6, 7>(p); compare_and_swap<4, 5>(p); compare_and_swap<1, 3>(p);
	}
	compare_and_swap<0, 2>(p);
	if constexpr (MAXP >= 4) if (p.vertex_count >= 4) compare_and_swap<2, 3>(p);
	compare_and_swap<0, 1>(p);
}

// :521-589. v[vc] must repeat v[0] when vc < MAXP.
template <int MAXP, bool BIASED>
VKR_DEV void prepare_psa(psa_polygon<MAXP>& p, int vertex_count, const f3 (&v)[MAXP]) {
	p.vertex_count = vertex_count;
	p.inner_ellipse_0 = make2(1.0f, 0.0f);
	p.vertices[0] = make2(v[0].x, v[0].y);
	p.ellipses[0] = ellipse_from_edge(v[0], v[1]);
	f2 previous = p.ellipses[0];
#pragma unroll
	for (int i = 1; i != MAXP; ++i) {
		p.vertices[i] = make2(v[i].x, v[i].y);
		p.ellipses[i] = make2(0.0f, 0.0f);
		if (!(i > 2 && i >= vertex_count)) {
			const f2 e = ellipse_from_edge(v[i], v[(i + 1) % MAXP]);
			const bool inner = is_inner_ellipse(e);
			p.ellipses[i] = inner ? previous : e;
			p.inner_ellipse_0 = (is_inner_ellipse(previous) && !inner) ? previous : p.inner_ellipse_0;
			previous = e;
		}
	}
	{
		const f2 e = p.ellipses[0];
		const bool inner = is_inner_ellipse(e);
		p.ellipses[0] = inner ? previous : e;
		p.inner_ellipse_0 = (is_inner_ellipse(previous) && !inner) ? previous : p.inner_ellipse_0;
	}
	p.psa = 0.0f;
#pragma unroll
	for (int i = 0; i != MAXP; ++i) p.sector_psa[i] = 0.0f;
	if (p.inner_ellipse_0.x > 0.0f) {
#pragma unroll
		for (int i = 0; i != MAXP; ++i) {
			if (!(i > 2 && i >= vertex_count)) {
				p.sector_psa[i] = ellipse_area_in_sector<BIASED>(p.ellipses[i], p.vertices[i], p.vertices[(i + 1) % MAXP]);
				p.psa += p.sector_psa[i];
			}
		}
	}
	else {
		sort_convex_polygon_vertices(p);
		f2 inner = p.inner_ellipse_0;
		float inner_rsd = ellipse_rsqrt_det(inner);
		f2 outer = make2(0.0f, 0.0f);
		float outer_rsd = 0.0f;
#pragma unroll
		for (int i = 0; i != MAXP - 1; ++i) {
			if (!(i > 1 && i + 1 >= vertex_count)) {
				const f2 ve = p.ellipses[i];
				const bool vinner = is_inner_ellipse(ve);
				const float vrsd = ellipse_rsqrt_det(ve);
				if (i == 0) { outer = ve; outer_rsd = vrsd; }
				else {
					inner = vinner ? ve : inner;
					inner_rsd = vinner ? vrsd : inner_rsd;
					outer = vinner ? outer : ve;
					outer_rsd = vinner ? outer_rsd : vrsd;
				}
				p.sector_psa[i] = area_between_ellipses_in_sector<BIASED>(inner, inner_rsd, outer, outer_rsd, p.vertices[i], p.vertices[i + 1]);
				p.psa += p.sector_psa[i];
			}
		}
	}
}

VKR_DEV f2 normalize_approx_and_flip(f2 rhs, f2 semi_circle) { // :599-611
	float scaling = fabsf(rhs.x) + fabsf(rhs.y);
	scaling = __uint_as_float(__float_as_uint(scaling) ^ 0x7F800000u);
	scaling = (dot(rhs, semi_circle) >= 0.0f) ? scaling : -scaling;
	return make2(scaling * rhs.x, scaling * rhs.y);
}

// 2x2 matrix in GLSL column-major naming: mCR = column C, row R
struct m22 { float m00, m01, m10, m11; };
VKR_DEV m22 outer_product(f2 c, f2 r) { m22 m; m.m00 = c.x * r.x; m.m01 = c.y * r.x; m.m10 = c.x * r.y; m.m11 = c.y * r.y; return m; }
VKR_DEV m22 operator-(m22 a, m22 b) { m22 m; m.m00 = a.m00 - b.m00; m.m01 = a.m01 - b.m01; m.m10 = a.m10 - b.m10; m.m11 = a.m11 - b.m11; return m; }
VKR_DEV f2 solve_homogeneous_quadratic(m22 q) { // :625-630 (Blinn)
	const float coeff_xy = 0.5f * (q.m01 + q.m10);
	const float sqrt_discriminant = sqrtf(max_glsl(0.0f, coeff_xy * coeff_xy - q.m00 * q.m11));
	const float scaled_root = fabsf(coeff_xy) + sqrt_discriminant;
	return (coeff_xy >= 0.0f) ? make2(scaled_root, -q.m00) : make2(q.m11, scaled_root);
}

template <bool BIASED>
VKR_DEV f2 sample_sector_between_ellipses(f2 rnd, float target_area, f2 inner, f2 outer, f2 dir_0, f2 dir_1) { // :645-739, 2 iterations
	const f2 q0 = normalize(dir_0);
	f2 q2 = normalize(dir_1);
	const f2 q1 = q0 + q2;
	const float ni0 = ellipse_normalized_direction_factor(inner, q0);
	const float ni1 = ellipse_direction_factor(inner, q1);
	float ni2 = ellipse_normalized_direction_factor(inner, q2);
	const float no0 = ellipse_normalized_direction_factor(outer, q0);
	const float no1 = ellipse_direction_factor(outer, q1);
	float no2 = ellipse_normalized_direction_factor(outer, q2);
	const float sector_area_0 = no0 * no1 - ni0 * ni1;
	const float sector_area_1 = no1 * no2 - ni1 * ni2;
	float target_quad_area = mix_fma(-sector_area_0, sector_area_1, rnd.x);
	const bool first = target_quad_area <= 0.0f;
	q2 = first ? q0 : q2;
	ni2 = first ? ni0 : ni2;
	no2 = first ? no0 : no2;
	target_quad_area += first ? sector_area_0 : -sector_area_1;
	target_quad_area *= fabsf(q1.x * q2.y - q2.x * q1.y);
	f2 quad_normal_i = q1 * ni1 + q2 * ni2;
	f2 quad_normal_o = q1 * no1 + q2 * no2;
	quad_normal_i = ellipse_transform(inner, quad_normal_i);
	quad_normal_o = ellipse_transform(outer, quad_normal_o);
	const float quad_offset_i = dot(quad_normal_i, q1) * ni1;
	const float quad_offset_o = dot(quad_normal_o, q1) * no1;
	const f2 r90 = rotate_90(q2);
	m22 quadratic = outer_product(r90 * (quad_offset_o * no2), quad_normal_i)
		- outer_product(r90 * (quad_offset_i * ni2) + quad_normal_i * target_quad_area, quad_normal_o);
	f2 current = solve_homogeneous_quadratic(quadratic);
	if (!BIASED) {
		const int iterations = (fabsf(rnd.x - 0.5f) <= 0.5f - 1.0e-5f) ? 2 : 0;
		const float inner_rsd = ellipse_rsqrt_det(inner);
		const float outer_rsd = ellipse_rsqrt_det(outer);
#pragma unroll 1
		for (int i = 0; i != iterations; ++i) {
			current = normalize_approx_and_flip(current, q1);
			const f2 inner_dir = ellipse_transform(inner, current);
			const f2 outer_dir = ellipse_transform(outer, current);
			const float det_dirs = max_glsl(+0.0f, dot(current, rotate_90(q0)));
			const float error = target_area - area_between_from_tangents<BIASED>(
				inner_rsd, det_dirs / (inner_rsd * dot(q0, inner_dir)),
				outer_rsd, det_dirs / (outer_rsd * dot(q0, outer_dir)));
			quadratic = outer_product(inner_dir - outer_dir, rotate_90(current)) - outer_product(inner_dir * (2.0f * error), outer_dir);
			current = solve_homogeneous_quadratic(quadratic);
		}
	}
	current = (dot(current, q1) >= 0.0f) ? current : make2(-current.x, -current.y);
	const float inner_factor = 1.0f / ellipse_direction_factor_rsq(inner, current);
	const float outer_factor = 1.0f / ellipse_direction_factor_rsq(outer, current);
	const float s = sqrtf(mix_fma(inner_factor, outer_factor, rnd.y));
	return make2(current.x * s, current.y * s);
}

// :749-805
template <int MAXP, bool BIASED>
VKR_DEV f3 sample_psa(const psa_polygon<MAXP>& p, f2 rnd) {
	float target = rnd.x * p.psa;
	f2 xy;
	if (p.inner_ellipse_0.x > 0.0f) {
		f2 outer = p.ellipses[0];
		f2 dir_0 = p.vertices[0];
		bool done = target < p.sector_psa[0];
#pragma unroll
		for (int i = 1; i != MAXP; ++i) {
			if (!done) {
				target -= p.sector_psa[i - 1];
				outer = p.ellipses[i];
				dir_0 = p.vertices[i];
				done = (i >= 2 && i + 1 == p.vertex_count) || target < p.sector_psa[i];
			}
		}
		const float sqrt_det = sqrtf(ellipse_det(outer));
		const float angle = 2.0f * target * sqrt_det;
		float sa, ca;
		sincos_cw(angle, &sa, &ca);
		ca = ca * sqrt_det;
		const f2 t = rotate_90(ellipse_transform(outer, dir_0));
		xy = make2(ca * dir_0.x + sa * t.x, ca * dir_0.y + sa * t.y);
		const float s = sqrtf(rnd.y / ellipse_direction_factor_rsq(outer, xy));
		xy = make2(xy.x * s, xy.y * s);
	}
	else {
		f2 inner = p.inner_ellipse_0;
		f2 outer = p.ellipses[0];
		f2 dir_0 = p.vertices[0];
		f2 dir_1 = p.vertices[1];
		float sector = p.sector_psa[0];
		bool done = target < sector; // (i = 0: the vertex-count exit needs i >= 1)
#pragma unroll
		for (int i = 1; i != MAXP - 1; ++i) {
			if (!done) {
				const f2 ve = p.ellipses[i];
				target -= p.sector_psa[i - 1];
				const bool vinner = is_inner_ellipse(ve);
				inner = vinner ? ve : inner;
				outer = vinner ? outer : ve;
				dir_0 = p.vertices[i];
				dir_1 = p.vertices[i + 1];
				sector = p.sector_psa[i];
				done = (i + 2 == p.vertex_count) || target < sector;
			}
		}
		rnd.x = target / sector;
		xy = sample_sector_between_ellipses<BIASED>(rnd, target, inner, outer, dir_0, dir_1);
	}
	return make3(xy.x, xy.y, sqrtf(max_glsl(0.0f, fmaf(-xy.x, xy.x, fmaf(-xy.y, xy.y, 1.0f)))));
}

// Error of a sample due to the iterative procedure (:823-883), for the error display modes of the shader (shading_pass.frag.glsl:489-493,
// 549-563): x = backward error (in the first random number), y = x times the projected solid angle, z = forward error in radians.
template <int MAXP, bool BIASED>
VKR_DEV f3 sampling_error(const psa_polygon<MAXP>& p, f2 rnd, f3 sampled_dir) {
	float target = rnd.x * p.psa;
	if (p.inner_ellipse_0.x > 0.0f) return make3(0.0f, 0.0f, 0.0f); // the central case is exact up to rounding
	float sector = 0.0f;
	f2 outer = make2(0.0f, 0.0f), inner = p.inner_ellipse_0, dir_0 = make2(0.0f, 0.0f);
	bool go = true;
#pragma unroll
	for (int i = 0; i != MAXP - 1; ++i) {
		go = go && !((i > 1 && i + 1 == p.vertex_count) || (i > 0 && target < 0.0f));
		if (go) {
			sector = p.sector_psa[i];
			target -= sector;
			const f2 ve = p.ellipses[i];
			const bool vinner = is_inner_ellipse(ve);
			if (i == 0) outer = ve;
			else {
				inner = vinner ? ve : inner;
				outer = vinner ? outer : ve;
			}
			dir_0 = p.vertices[i];
		}
	}
	target += sector;
	const f2 sxy = make2(sampled_dir.x, sampled_dir.y);
	const float sampled_psa = area_between_ellipses_in_sector<BIASED>(inner, ellipse_rsqrt_det(inner), outer, ellipse_rsqrt_det(outer), dir_0, sxy);
	const float scaled_backward_error = target - sampled_psa;
	const float backward_error = scaled_backward_error / p.psa;
	// derivative of the sampled direction with respect to the projected solid angle; cm0 / cm1 = columns of the constraint matrix before its transpose
	const f2 inner_dir = ellipse_transform(inner, sxy);
	const f2 outer_dir = ellipse_transform(outer, sxy);
	const float inner_factor = 1.0f / dot(sxy, inner_dir);
	const float outer_factor = 1.0f / dot(sxy, outer_dir);
	const f2 cm0 = rotate_90(sxy) * (0.5f * (inner_factor - outer_factor));
	f2 cm1 = inner_dir * ((1.0f - rnd.y) / (inner_factor * inner_factor));
	cm1 = cm1 + outer_dir * (rnd.y / (outer_factor * outer_factor));
	const float rcp_det = 1.0f / (cm0.x * cm1.y - cm0.y * cm1.x);
	f3 derivative;
	derivative.x = rcp_det * cm1.y;
	derivative.y = rcp_det * -cm1.x;
	derivative.z = -dot(sxy, make2(derivative.x, derivative.y)) / sampled_dir.z;
	const float forward_error = sqrtf(dot(derivative, derivative)) * scaled_backward_error;
	return make3(backward_error, scaled_backward_error, forward_error);
}

} // namespace vkr
