// vkr_related_work.cuh -- the related-work polygon sampling techniques of the reference renderer for sm_90a
// (SURVEY 8 row f4): the samplers the paper compares projected solid angle sampling against.
//   src/shaders/polygon_sampling_related_work.glsl:38-1048  Turk (area), Urena (rectangle solid angle), Arvo (solid angle and
//                                                           projected solid angle), Hart et al. (bilinear / biquadratic cosine warps)
//   src/shaders/polygon_sampling.glsl:120-225               solid angle sampling of the reference's authors
//   src/shaders/cubic_solver.glsl:29-76
// Each technique is one specialisation of rw_sampler<TECHNIQUE, MAXV>: prepare() runs once per (pixel, light), sample() once
// per sample and returns a world-space direction with its solid-angle density. MAXV = compile-time bound on the light's vertex
// count; the techniques that clip at the horizon work on MAXV + 1 vertices (src/main.c:194-216). All polygon indices are
// compile-time constants after unrolling, so the polygons live in registers. Expression order and fma placement follow the
// GLSL text (arithmetic contract, vkr_device_math.cuh); compile with -fmad=false.
// This header uses no warp intrinsics: tests/device_on_host.cpp compiles it for the CPU and holds it against the oracle.
#pragma once
#include "vkr_psa.cuh"

// sample_polygon_technique_t (src/polygonal_light.h:30-66)
enum { VKR_TECHNIQUE_BASELINE = 0, VKR_TECHNIQUE_AREA_TURK = 1, VKR_TECHNIQUE_RECTANGLE_SOLID_ANGLE_URENA = 2, VKR_TECHNIQUE_SOLID_ANGLE_ARVO = 3,
	VKR_TECHNIQUE_SOLID_ANGLE = 4, VKR_TECHNIQUE_CLIPPED_SOLID_ANGLE = 5, VKR_TECHNIQUE_BILINEAR_COSINE_WARP_HART = 6, VKR_TECHNIQUE_BILINEAR_COSINE_WARP_CLIPPING_HART = 7,
	VKR_TECHNIQUE_BIQUADRATIC_COSINE_WARP_HART = 8, VKR_TECHNIQUE_BIQUADRATIC_COSINE_WARP_CLIPPING_HART = 9, VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO = 10,
	VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE = 11, VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_BIASED = 12 };

namespace vkr {

VKR_DEV f3 neg(f3 a) { return make3(-a.x, -a.y, -a.z); }
// a*x + b*y (+ c*z): componentwise products and sums, left to right
VKR_DEV f3 lin2(float a, f3 x, float b, f3 y) { return x * a + y * b; }
VKR_DEV f3 lin3(float a, f3 x, float b, f3 y, float c, f3 z) { return (x * a + y * b) + z * c; }

// One polygonal light as the samplers see it (polygonal_light_utility.glsl:26-83), read from the constant block
template <int MAXV>
struct rw_light {
	int vertex_count;
	f3 vertices_world[MAXV];
	f2 fan_areas[MAXV - 2];
	f3 translation, rotation_0, rotation_1, rotation_2;   // columns of the rotation
	float scaling_x, scaling_y, area;
	f3 plane_normal;
	float plane_w;
};

VKR_DEV float rw_ldf(const unsigned char* p, int off) { return *reinterpret_cast<const float*>(p + off); }

template <int MAXV>
VKR_DEV void rw_load_light(rw_light<MAXV>& l, const unsigned char* light) {
	l.scaling_x = rw_ldf(light, 12); l.scaling_y = rw_ldf(light, 28); l.area = rw_ldf(light, 144);
	l.translation = make3(rw_ldf(light, 16), rw_ldf(light, 20), rw_ldf(light, 24));
	l.plane_normal = make3(rw_ldf(light, 64), rw_ldf(light, 68), rw_ldf(light, 72));
	l.plane_w = rw_ldf(light, 76);
	l.vertex_count = *reinterpret_cast<const int*>(light + 80);
	l.rotation_0 = make3(rw_ldf(light, 96), rw_ldf(light, 112), rw_ldf(light, 128));
	l.rotation_1 = make3(rw_ldf(light, 100), rw_ldf(light, 116), rw_ldf(light, 132));
	l.rotation_2 = make3(rw_ldf(light, 104), rw_ldf(light, 120), rw_ldf(light, 136));
	const unsigned char* vw = light + 160 + 16 * MAXV;
	const unsigned char* fa = vw + 16 * MAXV;
#pragma unroll
	for (int i = 0; i != MAXV; ++i) l.vertices_world[i] = make3(rw_ldf(vw, 16 * i), rw_ldf(vw, 16 * i + 4), rw_ldf(vw, 16 * i + 8));
#pragma unroll
	for (int i = 0; i != MAXV - 2; ++i) l.fan_areas[i] = make2(rw_ldf(fa, 16 * i), rw_ldf(fa, 16 * i + 4));
}

// Shading space of one pixel: rows of world_to_shading_space and its translation column (ltc_utility.glsl:85-88)
struct rw_frame {
	f3 rx, ry, rz, t;
};
VKR_DEV f3 rw_to_shading(const rw_frame& f, f3 v, bool flip) { // (world_to_shading_space * vec4(v, 1)), row y negated if flip
	const f3 q = make3(
		fmaf(f.t.x, 1.0f, fmaf(f.rx.z, v.z, fmaf(f.rx.y, v.y, f.rx.x * v.x))),
		fmaf(f.t.y, 1.0f, fmaf(f.ry.z, v.z, fmaf(f.ry.y, v.y, f.ry.x * v.x))),
		fmaf(f.t.z, 1.0f, fmaf(f.rz.z, v.z, fmaf(f.rz.y, v.y, f.rz.x * v.x))));
	return make3(q.x, flip ? -q.y : q.y, q.z);
}
VKR_DEV f3 rw_to_world(const rw_frame& f, f3 d, bool flip) { // (transpose(world_to_shading_space) * d).xyz
	const float dy = flip ? -d.y : d.y;
	return make3(
		fmaf(f.rz.x, d.z, fmaf(f.ry.x, dy, f.rx.x * d.x)),
		fmaf(f.rz.y, d.z, fmaf(f.ry.y, dy, f.rx.y * d.x)),
		fmaf(f.rz.z, d.z, fmaf(f.ry.z, dy, f.rx.z * d.x)));
}

// ---------------------------------------------------------------------------------------------------------------------
// Solid angle sampling ("ours", polygon_sampling.glsl:61-225): triangle fan around vertex 0
template <int MAXP>
struct sa_polygon {
	int vertex_count;
	f3 dirs[MAXP];
	f3 params[MAXP - 2];   // per fan triangle: |det|, dot(v0 + v1, v2), 1 + dot(v0, v1)
	float fan[MAXP - 2];   // solid angle of the fan up to triangle i
	float solid_angle;
};

template <int MAXP>
VKR_DEV void prepare_sa(sa_polygon<MAXP>& p, int vertex_count, const f3 (&vertices)[MAXP], f3 shading_position) { // :120-175
	p.vertex_count = vertex_count;
#pragma unroll
	for (int i = 0; i != MAXP; ++i) p.dirs[i] = normalize(vertices[i] - shading_position);
	const float householder_sign = (p.dirs[0].x > 0.0f) ? -1.0f : 1.0f;
	const float hs = 1.0f / (fabsf(p.dirs[0].x) + 1.0f);
	const f2 householder_yz = make2(p.dirs[0].y * hs, p.dirs[0].z * hs);
	p.solid_angle = 0.0f;
	float previous_dot_1_2 = dot(p.dirs[0], p.dirs[1]);
#pragma unroll
	for (int i = 0; i != MAXP - 2; ++i) {
		p.params[i] = make3(0.0f, 0.0f, 0.0f); p.fan[i] = 0.0f;
		if (!(i >= 1 && i + 2 >= vertex_count)) {
			const f3 v0 = p.dirs[i + 1], v1 = p.dirs[0], v2 = p.dirs[i + 2];
			const float dot_0_1 = previous_dot_1_2;
			const float dot_0_2 = dot(v0, v2);
			const float dot_1_2 = dot(v1, v2);
			previous_dot_1_2 = dot_1_2;
			const float dot_householder_0 = fmaf(-householder_sign, v0.x, dot_0_1);
			const float dot_householder_2 = fmaf(-householder_sign, v2.x, dot_1_2);
			const f2 c0 = make2(fmaf(-dot_householder_0, householder_yz.x, v0.y), fmaf(-dot_householder_0, householder_yz.y, v0.z));
			const f2 c1 = make2(fmaf(-dot_householder_2, householder_yz.x, v2.y), fmaf(-dot_householder_2, householder_yz.y, v2.z));
			const float simplex_volume = fabsf(c0.x * c1.y - c1.x * c0.y);
			const float dot_0_2_plus_1_2 = dot_0_2 + dot_1_2;
			const float one_plus_dot_0_1 = 1.0f + dot_0_1;
			const float tangent = simplex_volume / (one_plus_dot_0_1 + dot_0_2_plus_1_2);
			const float triangle_solid_angle = 2.0f * positive_atan<false>(tangent);
			p.solid_angle += triangle_solid_angle;
			p.fan[i] = p.solid_angle;
			p.params[i] = make3(simplex_volume, dot_0_2_plus_1_2, one_plus_dot_0_1);
		}
	}
}

template <int MAXP>
VKR_DEV f3 sample_sa(const sa_polygon<MAXP>& p, f2 rnd) { // :194-225
	const float target_solid_angle = p.solid_angle * rnd.x;
	float subtriangle_solid_angle = target_solid_angle;
	f3 parameters = p.params[0];
	f3 v0 = p.dirs[1], v2 = p.dirs[2];
	const f3 v1 = p.dirs[0];
	bool go = true;
#pragma unroll
	for (int i = 0; i < MAXP - 3; ++i) {
		go = go && !(i + 3 >= p.vertex_count || p.fan[i] >= target_solid_angle);
		if (go) {
			subtriangle_solid_angle = target_solid_angle - p.fan[i];
			v0 = p.dirs[i + 2];
			v2 = p.dirs[i + 3];
			parameters = p.params[i + 1];
		}
	}
	float sn, cs;
	sincos_cw(0.5f * subtriangle_solid_angle, &sn, &cs);
	const f3 offset = lin2(parameters.x * cs - parameters.y * sn, v0, parameters.z * sn, v2);
	const float f = 2.0f * (dot(v0, offset) / dot(offset, offset));
	const f3 new_vertex_2 = make3(fmaf(f, offset.x, -v0.x), fmaf(f, offset.y, -v0.y), fmaf(f, offset.z, -v0.z));
	const float s2 = dot(v1, new_vertex_2);
	const float s = mix_fma(1.0f, s2, rnd.y);
	const float denominator = fmaf(-s2, s2, 1.0f);
	float t_normed = sqrtf(fmaf(-s, s, 1.0f) / denominator);
	t_normed = (denominator > 0.0f) ? t_normed : rnd.y;
	return lin2(fmaf(-t_normed, s2, s), v1, t_normed, new_vertex_2);
}

// ---------------------------------------------------------------------------------------------------------------------
// Cubic solver (cubic_solver.glsl:29-76). Returns true if there are three real roots.
VKR_DEV bool solve_cubic(float (&roots)[3], float c0, float c1, float c2, float c3) {
	c0 /= c3; c1 /= c3; c2 /= c3;
	c1 /= 3.0f; c2 /= 3.0f;
	const float delta0 = fmaf(-c2, c2, c1);
	const float delta1 = fmaf(-c1, c2, c0);
	const float delta2 = c2 * c0 - c1 * c1;
	const float discriminant = 4.0f * delta0 * delta2 - delta1 * delta1;
	const float sqrt_abs_discriminant = sqrtf(fabsf(discriminant));
	const float depressed0 = fmaf(-2.0f * c2, delta0, delta1), depressed1 = delta0;
	if (discriminant >= 0.0f) {
		const float theta = atan2_poly(sqrt_abs_discriminant, -depressed0) * (1.0f / 3.0f);
		float cr0, cr1;
		sincos_cw(theta, &cr1, &cr0);
		const float sqrt_075 = 0.866025388240814208984375f; // sqrt(0.75f) rounded to nearest
		const float r1 = fmaf(-sqrt_075, cr1, -0.5f * cr0);
		const float r2 = fmaf(+sqrt_075, cr1, -0.5f * cr0);
		const float scale = 2.0f * sqrtf(-depressed1);
		roots[0] = fmaf(scale, cr0, -c2);
		roots[1] = fmaf(scale, r1, -c2);
		roots[2] = fmaf(scale, r2, -c2);
		return true;
	}
	const float signed_sqrt_discriminant = (depressed0 < 0.0f) ? sqrt_abs_discriminant : -sqrt_abs_discriminant;
	const float quadratic_root = 0.5f * (signed_sqrt_discriminant - depressed0);
	float cube_root_0 = pow_contract(fabsf(quadratic_root), 1.0f / 3.0f);
	cube_root_0 = (quadratic_root < 0.0f) ? -cube_root_0 : cube_root_0;
	const float cube_root_1 = -depressed1 / cube_root_0;
	const float cubic_root = cube_root_0 + cube_root_1;
	roots[0] = cubic_root - c2;
	return false;
}

// ---------------------------------------------------------------------------------------------------------------------
// Hart et al.: warps of primary sample space towards a bilinear / biquadratic approximation of the cosine term
VKR_DEV float linear_warp(float random_number, float density_0, float density_1) { // related_work.glsl:360-374
	const float lerped_density_sq = mix_fma(density_0 * density_0, density_1 * density_1, random_number);
	const float divisor = density_0 + sqrtf(lerped_density_sq);
	return random_number * (density_0 + density_1) / divisor;
}
VKR_DEV float quadratic_warp(float random_number, float density_0, float density_1, float density_2) { // :471-493
	const float q0 = density_0, q1 = 2.0f * (density_1 - density_0), q2 = density_0 - 2.0f * density_1 + density_2;
	const float c1 = q0, c2 = 0.5f * q1, c3 = (1.0f / 3.0f) * q2;
	random_number *= dot(make3(c1, c2, c3), make3(1.0f, 1.0f, 1.0f));
	const float c0 = -random_number;
	float roots[3] = { 0.0f, 0.0f, 0.0f };
	if (solve_cubic(roots, c0, c1, c2, c3)) {
		float result = roots[0];
		result = (roots[1] >= 0.0f && roots[1] <= 1.0f) ? roots[1] : result;
		result = (roots[2] >= 0.0f && roots[2] <= 1.0f) ? roots[2] : result;
		return result;
	}
	return roots[0];
}
VKR_DEV float quadratic_bezier(float b_0_0, float b_0_1, float b_0_2, float location) { // :499-503
	const float b_1_0 = mix_fma(b_0_0, b_0_1, location);
	const float b_1_1 = mix_fma(b_0_1, b_0_2, location);
	return mix_fma(b_1_0, b_1_1, location);
}

template <int MAXP>
struct bilinear_hart {
	sa_polygon<MAXP> polygon;
	float density_0;
	f2 density_1;
};
template <int MAXP>
VKR_DEV void prepare_bilinear_hart(bilinear_hart<MAXP>& h, int vertex_count, const f3 (&vertices)[MAXP]) { // :327-354
	prepare_sa<MAXP>(h.polygon, vertex_count, vertices, make3(0.0f, 0.0f, 0.0f));
	h.density_0 = max_glsl(0.0f, h.polygon.dirs[0].z);
	h.density_1.x = max_glsl(0.0f, h.polygon.dirs[1].z);
	h.density_1.y = h.polygon.dirs[2].z;
#pragma unroll
	for (int i = 3; i < MAXP; ++i) h.density_1.y = (i < vertex_count) ? h.polygon.dirs[i].z : h.density_1.y;
	h.density_1.y = max_glsl(0.0f, h.density_1.y);
	const float density_sum = 2.0f * h.density_0 + h.density_1.x + h.density_1.y;
	const float normalization = 4.0f / (h.polygon.solid_angle * density_sum);
	h.density_0 *= normalization;
	h.density_1 = h.density_1 * normalization;
	const float inv_solid_angle = 1.0f / h.polygon.solid_angle;
	h.density_0 = (density_sum <= 0.0f) ? inv_solid_angle : h.density_0;
	h.density_1 = (density_sum <= 0.0f) ? make2(inv_solid_angle, inv_solid_angle) : h.density_1;
}
template <int MAXP>
VKR_DEV f3 sample_bilinear_hart(float* out_density, const bilinear_hart<MAXP>& h, f2 rnd) { // :385-395
	rnd.y = linear_warp(rnd.y, 2.0f * h.density_0, dot(h.density_1, make2(1.0f, 1.0f)));
	const float density_0 = mix_fma(h.density_0, h.density_1.x, rnd.y);
	const float density_1 = mix_fma(h.density_0, h.density_1.y, rnd.y);
	rnd.x = linear_warp(rnd.x, density_0, density_1);
	*out_density = mix_fma(density_0, density_1, rnd.x);
	return sample_sa<MAXP>(h.polygon, rnd);
}

template <int MAXP>
struct biquadratic_hart {
	sa_polygon<MAXP> polygon;
	float density_0;
	f3 density_1, density_2;
};
VKR_DEV float biquadratic_middle_row(f3 vertex_0, f3 far_vertex) { // one iteration of the loop at :437-446
	const float s2 = dot(vertex_0, far_vertex);
	const float s = fmaf(0.5f, s2, 0.5f);
	const float t = sqrtf(max_glsl(0.0f, fmaf(-s, s, 1.0f)));
	const float t_axis_z = fmaf(-s2, vertex_0.z, far_vertex.z);
	const float normalization_t_axis = rsqrt_ieee(2.0f * fmaf(-s2, s2, 1.0f));
	const float sample_z = s * vertex_0.z + (t * normalization_t_axis) * t_axis_z;
	return max_glsl(0.0f, sample_z);
}
template <int MAXP>
VKR_DEV void prepare_biquadratic_hart(biquadratic_hart<MAXP>& h, int vertex_count, const f3 (&vertices)[MAXP]) { // :417-464
	prepare_sa<MAXP>(h.polygon, vertex_count, vertices, make3(0.0f, 0.0f, 0.0f));
	f3 last_vertex = h.polygon.dirs[2];
#pragma unroll
	for (int i = 3; i < MAXP; ++i) last_vertex = (i < vertex_count) ? h.polygon.dirs[i] : last_vertex;
	const f3 vertex_0 = h.polygon.dirs[0];
	h.density_0 = max_glsl(0.0f, vertex_0.z);
	h.density_2.x = max_glsl(0.0f, h.polygon.dirs[1].z);
	h.density_2.z = max_glsl(0.0f, last_vertex.z);
	const f3 sample_2_1 = sample_sa<MAXP>(h.polygon, make2(0.5f, 1.0f));
	h.density_2.y = max_glsl(0.0f, sample_2_1.z);
	h.density_1.x = biquadratic_middle_row(vertex_0, vertex_0);
	h.density_1.y = biquadratic_middle_row(vertex_0, sample_2_1);
	h.density_1.z = biquadratic_middle_row(vertex_0, last_vertex);
	const f3 ones = make3(1.0f, 1.0f, 1.0f);
	const float density_sum = 3.0f * h.density_0 + dot(h.density_1, ones) + dot(h.density_2, ones);
	const float normalization = 9.0f / (h.polygon.solid_angle * density_sum);
	h.density_0 *= normalization;
	h.density_1 = h.density_1 * normalization;
	h.density_2 = h.density_2 * normalization;
	const float inv_solid_angle = 1.0f / h.polygon.solid_angle;
	const f3 uniform = make3(inv_solid_angle, inv_solid_angle, inv_solid_angle);
	h.density_0 = (density_sum <= 0.0f) ? inv_solid_angle : h.density_0;
	h.density_1 = (density_sum <= 0.0f) ? uniform : h.density_1;
	h.density_2 = (density_sum <= 0.0f) ? uniform : h.density_2;
}
template <int MAXP>
VKR_DEV f3 sample_biquadratic_hart(float* out_density, const biquadratic_hart<MAXP>& h, f2 rnd) { // :508-520
	const f3 ones = make3(1.0f, 1.0f, 1.0f);
	rnd.y = quadratic_warp(rnd.y, 3.0f * h.density_0, dot(h.density_1, ones), dot(h.density_2, ones));
	const float density_0 = quadratic_bezier(h.density_0, h.density_1.x, h.density_2.x, rnd.y);
	const float density_1 = quadratic_bezier(h.density_0, h.density_1.y, h.density_2.y, rnd.y);
	const float density_2 = quadratic_bezier(h.density_0, h.density_1.z, h.density_2.z, rnd.y);
	rnd.x = quadratic_warp(rnd.x, density_0, density_1, density_2);
	*out_density = quadratic_bezier(density_0, density_1, density_2, rnd.x);
	return sample_sa<MAXP>(h.polygon, rnd);
}

// ---------------------------------------------------------------------------------------------------------------------
// Arvo, solid angle (related_work.glsl:209-304)
template <int MAXP>
struct sa_arvo_polygon {
	int vertex_count;
	f3 dirs[MAXP];
	float fan[MAXP - 2];
	f2 opposite[MAXP - 2];   // cosine and sine of the angle between the edges (0, i+1) and (i+1, i+2)
	float solid_angle;
};
template <int MAXP>
VKR_DEV void prepare_sa_arvo(sa_arvo_polygon<MAXP>& p, int vertex_count, const f3 (&vertices)[MAXP], f3 shading_position) { // :229-264
#pragma unroll
	for (int i = 0; i != MAXP; ++i) p.dirs[i] = normalize(vertices[i] - shading_position);
	float solid_angle = 0.0f;
#pragma unroll
	for (int i = 0; i != MAXP - 2; ++i) {
		p.fan[i] = 0.0f; p.opposite[i] = make2(0.0f, 0.0f);
		if (!(i >= 1 && i + 2 >= vertex_count)) {
			const f3 n0 = normalize(cross(p.dirs[i + 1] - p.dirs[0], p.dirs[0]));
			const f3 n1 = normalize(cross(p.dirs[i + 2] - p.dirs[i + 1], p.dirs[i + 1]));
			p.opposite[i].x = -dot(n0, n1);
			p.opposite[i].y = sqrtf(max_glsl(0.0f, fmaf(-p.opposite[i].x, p.opposite[i].x, 1.0f)));
			const float dot_0_1 = dot(p.dirs[0], p.dirs[i + 1]);
			const float dot_0_2 = dot(p.dirs[0], p.dirs[i + 2]);
			const float dot_1_2 = dot(p.dirs[i + 1], p.dirs[i + 2]);
			const float simplex_volume = det3(p.dirs[0], p.dirs[i + 1], p.dirs[i + 2]);
			const float tangent = fabsf(simplex_volume) / (1.0f + dot_0_1 + dot_0_2 + dot_1_2);
			solid_angle += 2.0f * positive_atan<false>(tangent);
			p.fan[i] = solid_angle;
		}
	}
	p.solid_angle = solid_angle;
	p.vertex_count = vertex_count;
}
template <int MAXP>
VKR_DEV f3 sample_sa_arvo(const sa_arvo_polygon<MAXP>& p, f2 rnd) { // :269-304
	const float target_solid_angle = p.solid_angle * rnd.x;
	float subtriangle_solid_angle = target_solid_angle;
	f2 opposite_dir = p.opposite[0];
	f3 t0 = p.dirs[1], t2 = p.dirs[2];
	const f3 t1 = p.dirs[0];
	bool go = true;
#pragma unroll
	for (int i = 0; i < MAXP - 3; ++i) {
		go = go && !(i + 3 >= p.vertex_count || p.fan[i] >= target_solid_angle);
		if (go) {
			subtriangle_solid_angle = target_solid_angle - p.fan[i];
			t0 = p.dirs[i + 2];
			t2 = p.dirs[i + 3];
			opposite_dir = p.opposite[i + 1];
		}
	}
	f2 sd;
	sincos_cw(subtriangle_solid_angle, &sd.y, &sd.x);
	const float pp = sd.y * opposite_dir.x - sd.x * opposite_dir.y;
	const float qq = sd.y * opposite_dir.y + sd.x * opposite_dir.x;
	const float u = qq - opposite_dir.x;
	const float v = pp + opposite_dir.y * dot(t0, t1);
	const float s = ((v * qq - u * pp) * opposite_dir.x - v) / ((v * pp + u * qq) * opposite_dir.y);
	const f3 edge_tangent_2_0 = normalize(t2 - t0 * dot(t0, t2));
	const f3 vertex_2 = lin2(s, t0, sqrtf(clamp_glsl(fmaf(-s, s, 1.0f), 0.0f, 1.0f)), edge_tangent_2_0);
	const float z = 1.0f - rnd.y * (1.0f - dot(vertex_2, t1));
	const f3 edge_tangent_2_1 = normalize(vertex_2 - t1 * dot(t1, vertex_2));
	return lin2(z, t1, sqrtf(clamp_glsl(fmaf(-z, z, 1.0f), 0.0f, 1.0f)), edge_tangent_2_1);
}

// ---------------------------------------------------------------------------------------------------------------------
// Urena et al., rectangle solid angle (related_work.glsl:100-200)
struct urena_rectangle {
	f3 x, y, z;
	float z0, z0sq, x0, y0, y0sq, x1, y1, y1sq, b0, b1, b0sq, k, solid_angle;
};
VKR_DEV void prepare_urena(urena_rectangle& q, f3 s, float exl, float eyl, f3 rotation_0, f3 rotation_1, f3 rotation_2, f3 o) { // :127-170
	q.x = rotation_0; q.y = rotation_1; q.z = rotation_2;
	const f3 d = s - o;
	q.z0 = dot(d, q.z);
	q.z = (q.z0 > 0.0f) ? neg(q.z) : q.z;
	q.z0 = -fabsf(q.z0);
	q.z0sq = q.z0 * q.z0;
	q.x0 = dot(d, q.x);
	q.y0 = dot(d, q.y);
	q.x1 = q.x0 + exl;
	q.y1 = q.y0 + eyl;
	q.y0sq = q.y0 * q.y0;
	q.y1sq = q.y1 * q.y1;
	const f3 v00 = make3(q.x0, q.y0, q.z0), v01 = make3(q.x0, q.y1, q.z0), v10 = make3(q.x1, q.y0, q.z0), v11 = make3(q.x1, q.y1, q.z0);
	const f3 n0 = normalize(cross(v00, v10));
	const f3 n1 = normalize(cross(v10, v11));
	const f3 n2 = normalize(cross(v11, v01));
	const f3 n3 = normalize(cross(v01, v00));
	const float g0 = acos_full(-dot(n0, n1));
	const float g1 = acos_full(-dot(n1, n2));
	const float g2 = acos_full(-dot(n2, n3));
	const float g3 = acos_full(-dot(n3, n0));
	q.b0 = n0.z;
	q.b1 = n2.z;
	q.b0sq = q.b0 * q.b0;
	q.k = 2.0f * kPi - g2 - g3;
	q.solid_angle = g0 + g1 - q.k;
}
VKR_DEV f3 sample_urena(const urena_rectangle& q, f2 rnd) { // :177-200
	const float u = rnd.x, v = rnd.y;
	const float au = fmaf(u, q.solid_angle, q.k);
	float sin_au, cos_au;
	sincos_cw(au, &sin_au, &cos_au);
	const float fu = fmaf(cos_au, q.b0, -q.b1) / sin_au;
	float cu = rsqrt_ieee(fmaf(fu, fu, q.b0sq));
	cu = (fu > 0.0f) ? cu : -cu;
	cu = clamp_glsl(cu, -1.0f, 1.0f);
	float xu = -(cu * q.z0) * rsqrt_ieee(fmaf(-cu, cu, 1.0f));
	xu = clamp_glsl(xu, q.x0, q.x1);
	const float d = sqrtf(xu * xu + q.z0sq);
	const float h0 = q.y0 * rsqrt_ieee(fmaf(d, d, q.y0sq));
	const float h1 = q.y1 * rsqrt_ieee(fmaf(d, d, q.y1sq));
	const float hv = h0 + v * (h1 - h0);
	const float mhv2_1 = fmaf(-hv, hv, 1.0f);
	const float yv = (mhv2_1 >= 0.0f) ? ((hv * d) * rsqrt_ieee(mhv2_1)) : q.y1;
	return normalize(lin3(xu, q.x, yv, q.y, q.z0, q.z));
}

// ---------------------------------------------------------------------------------------------------------------------
// Turk, uniform area sampling (related_work.glsl:38-88)
template <int MAXV>
VKR_DEV f3 sample_area_turk(const rw_light<MAXV>& l, f2 rnd) { // :38-66
	const float target_area = l.fan_areas[MAXV - 3].y * rnd.x;
	float subtriangle_area = target_area;
	float triangle_area = l.fan_areas[0].x;
	f3 t0 = l.vertices_world[1], t2 = l.vertices_world[2];
	const f3 t1 = l.vertices_world[0];
	bool go = true;
#pragma unroll
	for (int i = 0; i < MAXV - 3; ++i) {
		go = go && !(i + 3 >= l.vertex_count || l.fan_areas[i].y >= target_area);
		if (go) {
			subtriangle_area = target_area - l.fan_areas[i].y;
			triangle_area = l.fan_areas[i + 1].x;
			t0 = l.vertices_world[i + 2];
			t2 = l.vertices_world[i + 3];
		}
	}
	rnd.x = subtriangle_area / triangle_area;
	const float sqrt_random_0 = sqrtf(rnd.x);
	return lin3(1.0f - sqrt_random_0, t0, sqrt_random_0 * rnd.y, t1, fmaf(-sqrt_random_0, rnd.y, sqrt_random_0), t2);
}
VKR_DEV float area_sample_density(f3* out_normalized_dir, f3 light_sample, f3 shading_position, f3 light_normal, float light_area) { // :81-88
	f3 dir = light_sample - shading_position;
	const float distance_squared = dot(dir, dir);
	const float normalization = rsqrt_ieee(distance_squared);
	dir = dir * normalization;
	*out_normalized_dir = dir;
	const float projected_area = fabsf(dot(light_normal, dir)) * light_area;
	return distance_squared / projected_area;
}

// ---------------------------------------------------------------------------------------------------------------------
// Arvo, projected solid angle (related_work.glsl:525-1030)
struct edge_arvo {
	float cdf_factor;   // 2 eta_i in Arvo's notes; negative for inner edges
	f2 length_coeffs;
	f2 elevations;
};
VKR_DEV edge_arvo select_edge(bool second, const edge_arvo& a, const edge_arvo& b) {
	edge_arvo r;
	r.cdf_factor = second ? b.cdf_factor : a.cdf_factor;
	r.length_coeffs.x = second ? b.length_coeffs.x : a.length_coeffs.x; r.length_coeffs.y = second ? b.length_coeffs.y : a.length_coeffs.y;
	r.elevations.x = second ? b.elevations.x : a.elevations.x; r.elevations.y = second ? b.elevations.y : a.elevations.y;
	return r;
}
template <int MAXP>
struct psa_arvo_polygon {
	int vertex_count;
	float azimuths[MAXP];
	edge_arvo edges[MAXP];
	edge_arvo inner_edge_0;   // cdf_factor > 0 <=> central case
	float sector_psa[MAXP];
	float psa;
};
VKR_DEV edge_arvo prepare_edge_arvo(f3 vertex_0, f3 vertex_1) { // :582-612
	edge_arvo edge;
	const f3 normal_a = normalize(cross(vertex_0, vertex_1));
	edge.cdf_factor = 0.5f * normal_a.z;
	const f3 ccw_vertex = (edge.cdf_factor > 0.0f) ? vertex_0 : vertex_1;
	const f2 normal_c = rotate_90(normalize(make2(ccw_vertex.x, ccw_vertex.y)));
	const float cos_beta = -dot(make2(normal_a.x, normal_a.y), normal_c);
	const float sin_beta_sq = fmaf(-cos_beta, cos_beta, 1.0f);
	const float csc_beta = rsqrt_ieee(max_glsl(0.0f, sin_beta_sq));
	const float csc_c = rsqrt_ieee(max_glsl(0.0f, fmaf(-ccw_vertex.z, ccw_vertex.z, 1.0f)));
	edge.length_coeffs.x = sin_beta_sq;
	edge.length_coeffs.y = dot(make2(normal_a.x, normal_a.y), rotate_90(normal_c)) * cos_beta;
	edge.length_coeffs = edge.length_coeffs * (csc_beta * csc_c);
	edge.elevations.x = ccw_vertex.z;
	edge.elevations.y = cross(ccw_vertex, normal_a).z;
	edge.elevations.y = (edge.cdf_factor > 0.0f) ? -edge.elevations.y : edge.elevations.y;
	return edge;
}
// Projected solid angle of the triangle (normal, two points on the edge's great circle) and its derivative with respect
// to the second azimuth (:624-668)
VKR_DEV f2 edge_psa_in_sector_derivative_arvo(const edge_arvo& edge, float relative_azimuth_0, float relative_azimuth_1) {
	f2 dir_0, dir_1;
	sincos_cw(relative_azimuth_0, &dir_0.y, &dir_0.x);
	sincos_cw(relative_azimuth_1, &dir_1.y, &dir_1.x);
	const f2 point_0 = make2(dot(edge.length_coeffs, dir_0), dir_0.y);
	const f2 point_1 = make2(dot(edge.length_coeffs, dir_1), dir_1.y);
	const f2 rotated_point = make2(point_0.x * point_1.x + point_0.y * point_1.y, point_0.x * point_1.y - point_0.y * point_1.x);
	const float quotient = fabsf(rotated_point.y) / rotated_point.x;
	const float length = positive_atan<false>(quotient);
	const f2 dir_1_deriv = rotate_90(dir_1);
	const f2 point_1_deriv = make2(dot(edge.length_coeffs, dir_1_deriv), dir_1_deriv.y);
	const f2 rotated_point_deriv = make2(point_0.x * point_1_deriv.x + point_0.y * point_1_deriv.y, point_0.x * point_1_deriv.y - point_0.y * point_1_deriv.x);
	float quotient_derivative = (rotated_point_deriv.y * rotated_point.x - rotated_point.y * rotated_point_deriv.x) / (rotated_point.x * rotated_point.x);
	quotient_derivative = (rotated_point.y < 0.0f) ? (-quotient_derivative) : quotient_derivative;
	const float length_deriv = quotient_derivative / fmaf(quotient, quotient, 1.0f);
	return make2(edge.cdf_factor * length, edge.cdf_factor * length_deriv);
}
VKR_DEV float edge_psa_in_sector_arvo(const edge_arvo& edge, float relative_azimuth_0, float relative_azimuth_1) { // :624-638
	f2 dir_0, dir_1;
	sincos_cw(relative_azimuth_0, &dir_0.y, &dir_0.x);
	sincos_cw(relative_azimuth_1, &dir_1.y, &dir_1.x);
	const f2 point_0 = make2(dot(edge.length_coeffs, dir_0), dir_0.y);
	const f2 point_1 = make2(dot(edge.length_coeffs, dir_1), dir_1.y);
	const f2 rotated_point = make2(point_0.x * point_1.x + point_0.y * point_1.y, point_0.x * point_1.y - point_0.y * point_1.x);
	const float length = positive_atan<false>(fabsf(rotated_point.y) / rotated_point.x);
	return edge.cdf_factor * length;
}
VKR_DEV float edge_elevation_arvo(const edge_arvo& edge, float relative_azimuth) { // :674-680
	f2 dir;
	sincos_cw(relative_azimuth, &dir.y, &dir.x);
	f2 point = make2(dot(edge.length_coeffs, dir), dir.y);
	point = normalize(point);
	return dot(point, edge.elevations);
}
template <int L, int R, int MAXP>
VKR_DEV void compare_and_swap_arvo(psa_arvo_polygon<MAXP>& p) { // :687-695
	const float lhs_azimuth = p.azimuths[L], rhs_azimuth = p.azimuths[R];
	const bool flip = (lhs_azimuth - rhs_azimuth) > 0.0f;
	p.azimuths[L] = flip ? rhs_azimuth : lhs_azimuth;
	p.azimuths[R] = flip ? lhs_azimuth : rhs_azimuth;
	const edge_arvo lhs_edge = p.edges[L], rhs_edge = p.edges[R];
	p.edges[L] = select_edge(flip, lhs_edge, rhs_edge);
	p.edges[R] = select_edge(flip, rhs_edge, lhs_edge);
}
template <int MAXP>
VKR_DEV void sort_convex_polygon_vertices_arvo(psa_arvo_polygon<MAXP>& p) { // :700-769, the networks of polygon_sampling.glsl:440-505
	if (p.vertex_count == 3) compare_and_swap_arvo<1, 2>(p);
	if constexpr (MAXP >= 4) if (p.vertex_count == 4) compare_and_swap_arvo<1, 3>(p);
	if constexpr (MAXP >= 5) if (p.vertex_count == 5) {
		compare_and_swap_arvo<2, 4>(p); compare_and_swap_arvo<1, 3>(p); compare_and_swap_arvo<1, 2>(p); compare_and_swap_arvo<0, 3>(p); compare_and_swap_arvo<3, 4>(p);
	}
	if constexpr (MAXP >= 6) if (p.vertex_count == 6) {
		compare_and_swap_arvo<3, 5>(p); compare_and_swap_arvo<2, 4>(p); compare_and_swap_arvo<1, 5>(p); compare_and_swap_arvo<0, 4>(p); compare_and_swap_arvo<4, 5>(p); compare_and_swap_arvo<1, 3>(p);
	}
	if constexpr (MAXP >= 7) if (p.vertex_count == 7) {
		compare_and_swap_arvo<2, 5>(p); compare_and_swap_arvo<1, 6>(p); compare_and_swap_arvo<5, 6>(p); compare_and_swap_arvo<3, 4>(p); compare_and_swap_arvo<0, 4>(p);
		compare_and_swap_arvo<4, 6>(p); compare_and_swap_arvo<1, 3>(p); compare_and_swap_arvo<3, 5>(p); compare_and_swap_arvo<4, 5>(p);
	}
	if constexpr (MAXP >= 8) if (p.vertex_count == 8) {
		compare_and_swap_arvo<2, 6>(p); compare_and_swap_arvo<3, 7>(p); compare_and_swap_arvo<1, 5>(p); compare_and_swap_arvo<0, 4>(p); compare_and_swap_arvo<4, 6>(p);
		compare_and_swap_arvo<5, 7>(p); compare_and_swap_arvo<6, 7>(p); compare_and_swap_arvo<4, 5>(p); compare_and_swap_arvo<1, 3>(p);
	}
	compare_and_swap_arvo<0, 2>(p);
	if constexpr (MAXP >= 4) if (p.vertex_count >= 4) compare_and_swap_arvo<2, 3>(p);
	compare_and_swap_arvo<0, 1>(p);
}
// :774-851. v[vc] must repeat v[0] when vc < MAXP (clip_polygon does that); v is normalised in place.
template <int MAXP>
VKR_DEV void prepare_psa_arvo(psa_arvo_polygon<MAXP>& p, int vertex_count, f3 (&v)[MAXP]) {
#pragma unroll
	for (int i = 0; i != MAXP; ++i) v[i] = normalize(v[i]);
	p.vertex_count = vertex_count;
	p.inner_edge_0.cdf_factor = 1.0f;
	p.inner_edge_0.length_coeffs = make2(0.0f, 0.0f);
	p.inner_edge_0.elevations = make2(0.0f, 0.0f);
	p.azimuths[0] = atan2_poly(v[0].y, v[0].x);
	p.edges[0] = prepare_edge_arvo(v[0], v[1]);
	edge_arvo previous_edge = p.edges[0];
#pragma unroll
	for (int i = 1; i != MAXP; ++i) {
		float azimuth = atan2_poly(v[i].y, v[i].x);
		azimuth -= (azimuth > p.azimuths[0] + kPi) ? (2.0f * kPi) : 0.0f;
		azimuth += (azimuth < p.azimuths[0] - kPi) ? (2.0f * kPi) : 0.0f;
		p.azimuths[i] = azimuth;
		p.edges[i].cdf_factor = 0.0f; p.edges[i].length_coeffs = make2(0.0f, 0.0f); p.edges[i].elevations = make2(0.0f, 0.0f);
		if (!(i > 2 && i >= vertex_count)) {
			const edge_arvo edge = prepare_edge_arvo(v[i], v[(i + 1) % MAXP]);
			p.edges[i] = select_edge(edge.cdf_factor >= 0.0f, previous_edge, edge);
			p.inner_edge_0 = select_edge(previous_edge.cdf_factor < 0.0f && edge.cdf_factor >= 0.0f, p.inner_edge_0, previous_edge);
			previous_edge = edge;
		}
	}
	{
		const edge_arvo edge = p.edges[0];
		p.edges[0] = select_edge(edge.cdf_factor >= 0.0f, previous_edge, edge);
		p.inner_edge_0 = select_edge(previous_edge.cdf_factor < 0.0f && edge.cdf_factor >= 0.0f, p.inner_edge_0, previous_edge);
	}
	p.psa = 0.0f;
#pragma unroll
	for (int i = 0; i != MAXP; ++i) p.sector_psa[i] = 0.0f;
	if (p.inner_edge_0.cdf_factor > 0.0f) {
#pragma unroll
		for (int i = 0; i != MAXP; ++i) {
			if (!(i > 2 && i >= vertex_count)) {
				p.sector_psa[i] = edge_psa_in_sector_arvo(p.edges[i], 0.0f, p.azimuths[(i + 1) % MAXP] - p.azimuths[i]);
				p.psa += p.sector_psa[i];
			}
		}
	}
	else {
		sort_convex_polygon_vertices_arvo(p);
		edge_arvo inner_edge = p.inner_edge_0;
		float inner_azimuth = p.azimuths[0];
		edge_arvo outer_edge = p.edges[0];
		float outer_azimuth = p.azimuths[0];
#pragma unroll
		for (int i = 0; i != MAXP - 1; ++i) {
			if (!(i > 1 && i + 1 >= vertex_count)) {
				const edge_arvo vertex_edge = p.edges[i];
				const float vertex_azimuth = p.azimuths[i];
				if (i != 0) {
					const bool outer = vertex_edge.cdf_factor >= 0.0f;
					inner_edge = select_edge(outer, vertex_edge, inner_edge);
					inner_azimuth = outer ? inner_azimuth : vertex_azimuth;
					outer_edge = select_edge(outer, outer_edge, vertex_edge);
					outer_azimuth = outer ? vertex_azimuth : outer_azimuth;
				}
				p.sector_psa[i] = edge_psa_in_sector_arvo(outer_edge, p.azimuths[i] - outer_azimuth, p.azimuths[i + 1] - outer_azimuth);
				p.sector_psa[i] += edge_psa_in_sector_arvo(inner_edge, p.azimuths[i] - inner_azimuth, p.azimuths[i + 1] - inner_azimuth);
				p.psa += p.sector_psa[i];
			}
		}
	}
}
VKR_DEV float cubic_interpolation(float sample_x, const float (&x)[4], const float (&y)[4]) { // :856-868
	const float y01 = (y[0] - y[1]) / (x[0] - x[1]);
	const float y12 = (y[1] - y[2]) / (x[1] - x[2]);
	const float y23 = (y[2] - y[3]) / (x[2] - x[3]);
	const float y012 = (y01 - y12) / (x[0] - x[2]);
	const float y123 = (y12 - y23) / (x[1] - x[3]);
	const float y0123 = (y012 - y123) / (x[0] - x[3]);
	return fmaf(sample_x - x[0], fmaf(sample_x - x[1], fmaf(sample_x - x[2], y0123, y012), y01), y[0]);
}
// sample_sector_within_edge (:872-908, HAS_INNER = false) and sample_sector_between_edges (:927-968)
template <bool HAS_INNER>
VKR_DEV f3 sample_sector_arvo(f2 rnd, float target_psa, const edge_arvo& inner_edge, float inner_azimuth, const edge_arvo& outer_edge, float outer_azimuth, float azimuth_0, float azimuth_1, int iteration_count) {
	const float azimuths[4] = { azimuth_0, mix_fma(azimuth_0, azimuth_1, 1.0f / 3.0f), mix_fma(azimuth_0, azimuth_1, 2.0f / 3.0f), azimuth_1 };
	float psas[4];
#pragma unroll
	for (int i = 0; i != 4; ++i) {
		psas[i] = edge_psa_in_sector_arvo(outer_edge, azimuth_0 - outer_azimuth, azimuths[i] - outer_azimuth);
		if (HAS_INNER) psas[i] += edge_psa_in_sector_arvo(inner_edge, azimuth_0 - inner_azimuth, azimuths[i] - inner_azimuth);
	}
	float sampled_azimuth = cubic_interpolation(target_psa, psas, azimuths);
#pragma unroll 1
	for (int i = 0; i != iteration_count; ++i) {
		const f2 outer_psa = edge_psa_in_sector_derivative_arvo(outer_edge, azimuth_0 - outer_azimuth, sampled_azimuth - outer_azimuth);
		float error, derivative;
		if (HAS_INNER) {
			const f2 inner_psa = edge_psa_in_sector_derivative_arvo(inner_edge, azimuth_0 - inner_azimuth, sampled_azimuth - inner_azimuth);
			error = inner_psa.x + outer_psa.x - target_psa;
			derivative = inner_psa.y + outer_psa.y;
		}
		else {
			error = outer_psa.x - target_psa;
			derivative = outer_psa.y;
		}
		sampled_azimuth -= error / derivative;
		sampled_azimuth = clamp_glsl(sampled_azimuth, azimuth_0, azimuth_1);
	}
	f3 sampled_dir;
	sincos_cw(sampled_azimuth, &sampled_dir.y, &sampled_dir.x);
	const float outer_z = edge_elevation_arvo(outer_edge, sampled_azimuth - outer_azimuth);
	if (HAS_INNER) {
		const float inner_z = edge_elevation_arvo(inner_edge, sampled_azimuth - inner_azimuth);
		sampled_dir.z = sqrtf(mix_fma(inner_z * inner_z, outer_z * outer_z, rnd.y));
	}
	else sampled_dir.z = sqrtf(mix_fma(1.0f, outer_z * outer_z, rnd.y));
	const float s = sqrtf(fmaf(-sampled_dir.z, sampled_dir.z, 1.0f));
	sampled_dir.x *= s; sampled_dir.y *= s;
	return sampled_dir;
}
template <int MAXP>
VKR_DEV f3 sample_psa_arvo(const psa_arvo_polygon<MAXP>& p, f2 rnd, int iteration_count) { // :973-1030
	float target = rnd.x * p.psa;
	float sector_psa = 0.0f;
	edge_arvo outer_edge = p.edges[0];
	float outer_azimuth = 0.0f, azimuth_1 = 0.0f;
	if (p.inner_edge_0.cdf_factor > 0.0f) {
		bool go = true;
#pragma unroll
		for (int i = 0; i != MAXP; ++i) {
			go = go && !((i > 2 && i >= p.vertex_count) || (i > 0 && target < 0.0f));
			if (go) {
				sector_psa = p.sector_psa[i];
				target -= sector_psa;
				outer_edge = p.edges[i];
				outer_azimuth = p.azimuths[i];
				azimuth_1 = p.azimuths[(i + 1) % MAXP];
			}
		}
		azimuth_1 = (azimuth_1 < outer_azimuth) ? (azimuth_1 + 2.0f * kPi) : azimuth_1;
		target += sector_psa;
		rnd.x = target / sector_psa;
		rnd.x = clamp_glsl(rnd.x, 0.0f, 1.0f);
		return sample_sector_arvo<false>(rnd, target, outer_edge, 0.0f, outer_edge, outer_azimuth, outer_azimuth, azimuth_1, iteration_count);
	}
	edge_arvo inner_edge = p.inner_edge_0;
	float inner_azimuth = p.azimuths[0];
	float azimuth_0 = 0.0f;
	bool go = true;
#pragma unroll
	for (int i = 0; i != MAXP - 1; ++i) {
		go = go && !((i > 1 && i + 1 >= p.vertex_count) || (i > 0 && target < 0.0f));
		if (go) {
			sector_psa = p.sector_psa[i];
			target -= sector_psa;
			const edge_arvo vertex_edge = p.edges[i];
			const float vertex_azimuth = p.azimuths[i];
			if (i == 0) {
				outer_edge = vertex_edge;
				outer_azimuth = vertex_azimuth;
			}
			else {
				const bool outer = vertex_edge.cdf_factor >= 0.0f;
				inner_edge = select_edge(outer, vertex_edge, inner_edge);
				inner_azimuth = outer ? inner_azimuth : vertex_azimuth;
				outer_edge = select_edge(outer, outer_edge, vertex_edge);
				outer_azimuth = outer ? vertex_azimuth : outer_azimuth;
			}
			azimuth_0 = p.azimuths[i];
			azimuth_1 = p.azimuths[i + 1];
		}
	}
	target += sector_psa;
	rnd.x = target / sector_psa;
	rnd.x = clamp_glsl(rnd.x, 0.0f, 1.0f);
	return sample_sector_arvo<true>(rnd, target, inner_edge, inner_azimuth, outer_edge, outer_azimuth, azimuth_0, azimuth_1, iteration_count);
}

// Backward error of a sample of sample_psa_arvo() and the same times the projected solid angle (:1035-1087)
template <int MAXP>
VKR_DEV f2 sampling_error_arvo(const psa_arvo_polygon<MAXP>& p, f2 rnd, f3 sampled_dir) {
	float target = rnd.x * p.psa;
	if (p.inner_edge_0.cdf_factor > 0.0f) return make2(0.0f, 0.0f);
	edge_arvo outer_edge = p.edges[0], inner_edge = p.inner_edge_0;
	float inner_azimuth = p.azimuths[0], outer_azimuth = 0.0f, sector_psa = 0.0f, azimuth_0 = 0.0f;
	bool go = true;
#pragma unroll
	for (int i = 0; i != MAXP - 1; ++i) {
		go = go && !((i > 1 && i + 1 >= p.vertex_count) || (i > 0 && target < 0.0f));
		if (go) {
			sector_psa = p.sector_psa[i];
			target -= sector_psa;
			const edge_arvo vertex_edge = p.edges[i];
			const float vertex_azimuth = p.azimuths[i];
			if (i == 0) {
				outer_edge = vertex_edge;
				outer_azimuth = vertex_azimuth;
			}
			else {
				const bool outer = vertex_edge.cdf_factor >= 0.0f;
				inner_edge = select_edge(outer, vertex_edge, inner_edge);
				inner_azimuth = outer ? inner_azimuth : vertex_azimuth;
				outer_edge = select_edge(outer, outer_edge, vertex_edge);
				outer_azimuth = outer ? vertex_azimuth : outer_azimuth;
			}
			azimuth_0 = p.azimuths[i];
		}
	}
	target += sector_psa;
	const float sampled_azimuth = atan2_poly(sampled_dir.y, sampled_dir.x);
	const float outer_psa = edge_psa_in_sector_derivative_arvo(outer_edge, azimuth_0 - outer_azimuth, sampled_azimuth - outer_azimuth).x;
	const float inner_psa = edge_psa_in_sector_derivative_arvo(inner_edge, azimuth_0 - inner_azimuth, sampled_azimuth - inner_azimuth).x;
	const float sampled_psa = outer_psa + inner_psa;
	return make2((target - sampled_psa) / p.psa, target - sampled_psa);
}

// Error magnitude -> colour (shading_pass.frag.glsl:80-115): matplotlib's tab20b in linear Rec. 709, one hue per power of ten of
// error_factor * error. An index outside the table (only a NaN error gets there; undefined in GLSL) selects the first colour.
VKR_DEV f3 error_to_color(float error, float error_factor) {
	const float min_exponent = 0.0f, max_exponent = 5.0f;
	const float min_error = pow_contract(10.0f, min_exponent);
	const float max_error = pow_contract(10.0f, max_exponent - 0.01f);
	const float color_count = 20.0f;
	error = clamp_glsl(fabsf(error_factor * error), min_error, max_error);
	const float color_index = fmaf(log2_poly(error), color_count / ((max_exponent - min_exponent) * log2_poly(10.0f)), color_count * -min_exponent / (max_exponent - min_exponent));
	const int index = (color_index >= 0.0f && color_index < 20.0f) ? (int) color_index : 0;
	float r = 0.04092f, g = 0.04374f, b = 0.19120f;
	switch (index) {
#define VKR_COLOR(I, R, G, B) case I: r = R; g = G; b = B; break;
	VKR_COLOR(1, 0.08438f, 0.08866f, 0.36625f) VKR_COLOR(2, 0.14703f, 0.15593f, 0.62396f) VKR_COLOR(3, 0.33245f, 0.34191f, 0.73046f)
	VKR_COLOR(4, 0.12477f, 0.19120f, 0.04092f) VKR_COLOR(5, 0.26225f, 0.36131f, 0.08438f) VKR_COLOR(6, 0.46208f, 0.62396f, 0.14703f) VKR_COLOR(7, 0.61721f, 0.70838f, 0.33245f)
	VKR_COLOR(8, 0.26225f, 0.15293f, 0.03071f) VKR_COLOR(9, 0.50888f, 0.34191f, 0.04092f) VKR_COLOR(10, 0.79910f, 0.49102f, 0.08438f) VKR_COLOR(11, 0.79910f, 0.59720f, 0.29614f)
	VKR_COLOR(12, 0.23074f, 0.04519f, 0.04092f) VKR_COLOR(13, 0.41789f, 0.06663f, 0.06848f) VKR_COLOR(14, 0.67244f, 0.11954f, 0.14703f) VKR_COLOR(15, 0.79910f, 0.30499f, 0.33245f)
	VKR_COLOR(16, 0.19807f, 0.05286f, 0.17144f) VKR_COLOR(17, 0.37626f, 0.08228f, 0.29614f) VKR_COLOR(18, 0.61721f, 0.15293f, 0.50888f) VKR_COLOR(19, 0.73046f, 0.34191f, 0.67244f)
#undef VKR_COLOR
	default: break;
	}
	return make3(r, g, b);
}

// ---------------------------------------------------------------------------------------------------------------------
// One interface over all techniques (shading_pass.frag.glsl:332-481).
//   prepare(): false = this light contributes nothing at this pixel (clipped away / empty projected solid angle)
//   sample():  world-space direction towards the light + its density with respect to solid angle
//   ggx_density_factor(): 1 / solid angle (1 / projected solid angle for Arvo) as the GGX MIS part of the shader uses it (:683-687)
constexpr bool technique_clips(int technique) {
	return technique == VKR_TECHNIQUE_CLIPPED_SOLID_ANGLE || technique == VKR_TECHNIQUE_BILINEAR_COSINE_WARP_CLIPPING_HART
		|| technique == VKR_TECHNIQUE_BIQUADRATIC_COSINE_WARP_CLIPPING_HART || technique == VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO;
}

// Light vertices in shading space, clipped at the horizon if the technique asks for it. Returns the vertex count (0 = nothing left).
template <int MAXV, int MAXP>
VKR_DEV int rw_shading_space_polygon(f3 (&v)[MAXP], const rw_light<MAXV>& l, const rw_frame& frame, bool flip) {
#pragma unroll
	for (int i = 0; i != MAXV; ++i) v[i] = rw_to_shading(frame, l.vertices_world[i], flip);
	if constexpr (MAXP == MAXV) return l.vertex_count;
	else {
		v[MAXP - 1] = make3(0.0f, 0.0f, 0.0f);
		return clip_polygon<MAXP>(l.vertex_count, v);
	}
}

template <int TECHNIQUE, int MAXV> struct rw_sampler;

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_BASELINE, MAXV> { // :335-345
	f3 corner_offset, rotation_0, rotation_1;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3 position, const rw_frame&) {
		corner_offset = l.translation - position; rotation_0 = l.rotation_0; rotation_1 = l.rotation_1;
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const {
		*density = 1.0f;
		return normalize((corner_offset + rotation_0 * rnd.x) + rotation_1 * rnd.y);
	}
	VKR_DEV float ggx_density_factor() const { return 0.0f; }
};

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_AREA_TURK, MAXV> { // :347-353
	rw_light<MAXV> light;
	f3 position;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3 shading_position, const rw_frame&) { light = l; position = shading_position; return true; }
	VKR_DEV f3 sample(f2 rnd, float* density) const {
		const f3 light_sample = sample_area_turk<MAXV>(light, rnd);
		f3 dir;
		*density = area_sample_density(&dir, light_sample, position, light.plane_normal, light.area);
		return dir;
	}
	VKR_DEV float ggx_density_factor() const { return 0.0f; }
};

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_RECTANGLE_SOLID_ANGLE_URENA, MAXV> { // :355-366
	urena_rectangle squad;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3 position, const rw_frame&) {
		prepare_urena(squad, l.translation, l.scaling_x, l.scaling_y, l.rotation_0, l.rotation_1, l.rotation_2, position);
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const { *density = 1.0f / squad.solid_angle; return sample_urena(squad, rnd); }
	VKR_DEV float ggx_density_factor() const { return 1.0f / squad.solid_angle; }
};

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_SOLID_ANGLE_ARVO, MAXV> { // :368-378
	sa_arvo_polygon<MAXV> polygon;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3 position, const rw_frame&) {
		prepare_sa_arvo<MAXV>(polygon, l.vertex_count, l.vertices_world, position);
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const { *density = 1.0f / polygon.solid_angle; return sample_sa_arvo<MAXV>(polygon, rnd); }
	VKR_DEV float ggx_density_factor() const { return 1.0f / polygon.solid_angle; }
};

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_SOLID_ANGLE, MAXV> { // :380-390
	sa_polygon<MAXV> polygon;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3 position, const rw_frame&) {
		prepare_sa<MAXV>(polygon, l.vertex_count, l.vertices_world, position);
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const { *density = 1.0f / polygon.solid_angle; return sample_sa<MAXV>(polygon, rnd); }
	VKR_DEV float ggx_density_factor() const { return 1.0f / polygon.solid_angle; }
};

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_CLIPPED_SOLID_ANGLE, MAXV> { // :392-416
	sa_polygon<MAXV + 1> polygon;
	rw_frame frame;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3, const rw_frame& f) {
		frame = f;
		f3 v[MAXV + 1];
		const int vc = rw_shading_space_polygon<MAXV, MAXV + 1>(v, l, f, false);
		if (vc == 0) return false;
		prepare_sa<MAXV + 1>(polygon, vc, v, make3(0.0f, 0.0f, 0.0f));
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const { *density = 1.0f / polygon.solid_angle; return rw_to_world(frame, sample_sa<MAXV + 1>(polygon, rnd), false); }
	VKR_DEV float ggx_density_factor() const { return 1.0f / polygon.solid_angle; }
};

template <int MAXV, bool CLIP> struct rw_bilinear_sampler { // :392-405, 418-427
	static constexpr int MAXP = CLIP ? MAXV + 1 : MAXV;
	bilinear_hart<MAXP> polygon;
	rw_frame frame;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3, const rw_frame& f) {
		frame = f;
		f3 v[MAXP];
		const int vc = rw_shading_space_polygon<MAXV, MAXP>(v, l, f, false);
		if (vc == 0) return false;
		prepare_bilinear_hart<MAXP>(polygon, vc, v);
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const { return rw_to_world(frame, sample_bilinear_hart<MAXP>(density, polygon, rnd), false); }
	VKR_DEV float ggx_density_factor() const { return 0.0f; }
};
template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_BILINEAR_COSINE_WARP_HART, MAXV> : rw_bilinear_sampler<MAXV, false> {};
template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_BILINEAR_COSINE_WARP_CLIPPING_HART, MAXV> : rw_bilinear_sampler<MAXV, true> {};

template <int MAXV, bool CLIP> struct rw_biquadratic_sampler { // :392-405, 429-437
	static constexpr int MAXP = CLIP ? MAXV + 1 : MAXV;
	biquadratic_hart<MAXP> polygon;
	rw_frame frame;
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3, const rw_frame& f) {
		frame = f;
		f3 v[MAXP];
		const int vc = rw_shading_space_polygon<MAXV, MAXP>(v, l, f, false);
		if (vc == 0) return false;
		prepare_biquadratic_hart<MAXP>(polygon, vc, v);
		return true;
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const { return rw_to_world(frame, sample_biquadratic_hart<MAXP>(density, polygon, rnd), false); }
	VKR_DEV float ggx_density_factor() const { return 0.0f; }
};
template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_BIQUADRATIC_COSINE_WARP_HART, MAXV> : rw_biquadratic_sampler<MAXV, false> {};
template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_BIQUADRATIC_COSINE_WARP_CLIPPING_HART, MAXV> : rw_biquadratic_sampler<MAXV, true> {};

template <int MAXV> struct rw_sampler<VKR_TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO, MAXV> { // :439-481
	psa_arvo_polygon<MAXV + 1> polygon;
	rw_frame frame;
	bool flip;   // the shading point lies behind the light's plane: the winding is restored by mirroring the y-axis (:444-449)
	VKR_DEV bool prepare(const rw_light<MAXV>& l, f3 position, const rw_frame& f) {
		frame = f;
		flip = fmaf(l.plane_w, 1.0f, fmaf(l.plane_normal.z, position.z, fmaf(l.plane_normal.y, position.y, l.plane_normal.x * position.x))) < 0.0f;
		f3 v[MAXV + 1];
		const int vc = rw_shading_space_polygon<MAXV, MAXV + 1>(v, l, f, flip);
		if (vc == 0) return false;
		prepare_psa_arvo<MAXV + 1>(polygon, vc, v);
		return !(polygon.psa <= 0.0f);
	}
	VKR_DEV f3 sample(f2 rnd, float* density) const {
		const f3 d = sample_psa_arvo<MAXV + 1>(polygon, rnd, 3);
		*density = d.z / polygon.psa;
		return rw_to_world(frame, d, flip);
	}
	VKR_DEV float ggx_density_factor() const { return 1.0f / polygon.psa; }
};

} // namespace vkr
