// vkr_shade_light.cuh -- one polygonal light for one pixel of the shading pass with projected solid angle sampling: the five sampling strategies of
// evaluate_polygonal_light_shading() (src/shaders/shading_pass.frag.glsl:329-711) in the form the megakernel needs -- every candidate sample goes
// through submit() (vkr_ray_stream.cuh), which either adds it in place (TRACE = false) or hands it to the trace warps.
// Written for a warp (control flow is warp-uniform, `on` masks lanes), but without shadow rays nothing in here is a warp-level operation, so
// tests/device_on_host.cpp runs it on the CPU one pixel at a time against the reference-shader fixtures. Compile with -fmad=false.
#pragma once
#include "vkr_shade_common.cuh"
#include "vkr_ray_stream.cuh"

namespace vkr {

// One polygonal light for the warp's 32 pixels (shading_pass.frag.glsl:329-711, projected solid angle technique).
// Control flow is warp-uniform; `on` masks lanes whose pixel is not shaded by this light.
template <int STRATEGY, int MAXP, bool BIASED, bool OPTIMAL, bool TRACE, bool LIGHT_TEXTURES = false>
VKR_DEV void shade_light(bool on, const shading_point& sp, const ltc_state& l, const unsigned char* light, noise_stream& ns,
	const shading_kernel_params& p, const unsigned char* cb, uint32_t px, uint32_t py, ray_producer& q, pixel_sum& result, int lane)
{
	const int S = p.sample_count;
	const bool flip = dot4_point(light + L_PLANE, sp.position) < 0.0f;
	const f3 zero = make3(0.0f, 0.0f, 0.0f);
	psa_polygon<MAXP> pd;
	pd.psa = 0.0f; pd.inner_ellipse_0 = make2(0.0f, 0.0f); pd.vertex_count = 0;
	if (on) {
		f3 v[MAXP];
		const int vc = transform_and_clip<MAXP>(v, light, l.rx, l.ry, sp.normal, l.t, flip);
		if (vc == 0) on = false;
		else prepare_psa<MAXP, BIASED>(pd, vc, v);
	}
	if (STRATEGY == VKR_STRATEGY_DIFFUSE_ONLY || STRATEGY == VKR_STRATEGY_DIFFUSE_GGX_MIS) {
		if (on && pd.psa <= 0.0f) on = false;
#pragma unroll 1
		for (int s = 0; s != S; ++s) {
			bool has = false, pre_vis = false; f3 w = zero, c = zero; float tmax = 0.0f;
			if (on) {
				const f3 d = sample_psa<MAXP, BIASED>(pd, next_noise_2(ns, p, cb, px, py));
				const float density = d.z / pd.psa;
				w = shading_to_world(l, sp.normal, flip, d);
				const float lambert = dot(sp.normal, w);
				pre_vis = lambert > 0.0f;
				// What the shader multiplies radiance * BRDF with -- which is ZERO, not absent, for a sample that is not visible (:203-231, 305-323).
				// If that factor is not finite (degenerate polygon, NaN direction) the product is NaN either way and the pixel turns pink (:862-864):
				// such a sample goes out as a certain miss (tmax = 0) that carries NaN.
				float wgt = 0.0f; bool poisoned;
				if (STRATEGY == VKR_STRATEGY_DIFFUSE_ONLY) {
					has = density > 0.0f;
					wgt = lambert / density;
					poisoned = has && !is_finite(wgt);
				}
				else {
					has = true;
					const float ggx_density = ggx_reflected_direction_density(sp.lambert_outgoing, sp.outgoing, w, sp.normal, sp.roughness);
					wgt = (p.mis_heuristic == VKR_MIS_BALANCE) ? (1.0f / (density + ggx_density)) : (density / (density * density + ggx_density * ggx_density));
					poisoned = !is_finite(lambert) || !is_finite(wgt);
				}
				if (poisoned) { pre_vis = true; tmax = 0.0f; w = zero; c = not_a_number3(); }
				else if (pre_vis) {
					tmax = light_plane_distance(sp, light, w);
					const f3 rtb = light_radiance<LIGHT_TEXTURES>(p, light, sp.position, w) * evaluate_brdf<true, true>(sp, w);
					if (STRATEGY == VKR_STRATEGY_DIFFUSE_ONLY) c = rtb * wgt;
					else c = make3(rtb.x * lambert * wgt, rtb.y * lambert * wgt, rtb.z * lambert * wgt);
				}
			}
			submit<TRACE, false>(q, lane, has && pre_vis, pre_vis, w, tmax, c, zero, result, false);
		}
		if (STRATEGY == VKR_STRATEGY_DIFFUSE_GGX_MIS) {
			const f3 o_ss = make3(
				fmaf(l.t.x, 0.0f, fmaf(l.rx.z, sp.outgoing.z, fmaf(l.rx.y, sp.outgoing.y, l.rx.x * sp.outgoing.x))),
				0.0f,
				fmaf(l.t.z, 0.0f, fmaf(sp.normal.z, sp.outgoing.z, fmaf(sp.normal.y, sp.outgoing.y, sp.normal.x * sp.outgoing.x))));
			const float density_factor = 1.0f / pd.psa;
#pragma unroll 1
			for (int s = 0; s != S; ++s) {
				bool has = false; f3 w = zero, c = zero; float tmax = 0.0f;
				if (on) {
					float ggx_density;
					const f3 d = sample_ggx_reflected_direction(&ggx_density, o_ss, sp.roughness, next_noise_2(ns, p, cb, px, py));
					w = shading_to_world(l, sp.normal, flip, d);
					if (d.z > 0.0f && light_ray_intersection<MAXP - 1>(light, sp.position, w, 0.0f)) {
						const float lambert = dot(sp.normal, w);
						const float polygon_density = lambert * density_factor;
						const float wgt = (p.mis_heuristic == VKR_MIS_BALANCE) ? (1.0f / (ggx_density + polygon_density)) : (ggx_density / (ggx_density * ggx_density + polygon_density * polygon_density));
						if (!is_finite(lambert) || !is_finite(wgt)) { has = true; tmax = 0.0f; w = zero; c = not_a_number3(); } // 0 * inf, see above
						else if (lambert > 0.0f) {
							has = true;
							tmax = light_plane_distance(sp, light, w);
							const f3 rtb = light_radiance<LIGHT_TEXTURES>(p, light, sp.position, w) * evaluate_brdf<true, true>(sp, w);
							c = make3(rtb.x * lambert * wgt, rtb.y * lambert * wgt, rtb.z * lambert * wgt);
						}
					}
				}
				submit<TRACE, false>(q, lane, has, true, w, tmax, c, zero, result, false);
			}
		}
	}
	else {
		psa_polygon<MAXP> ps;
		ps.psa = 0.0f; ps.inner_ellipse_0 = make2(0.0f, 0.0f); ps.vertex_count = 0;
		if (on) {
			f3 v[MAXP];
			const int vc = transform_and_clip<MAXP>(v, light, l.cx, l.cy, l.cz, l.ct, flip);
			if (vc != 0) prepare_psa<MAXP, BIASED>(ps, vc, v);
			if (pd.psa == 0.0f) on = false;
		}
		const float specular_albedo = l.albedo;
		const float specular_weight = specular_albedo * ps.psa;
		const bool has_specular = on && ps.psa > 0.0f;
		if (STRATEGY == VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY) {
#pragma unroll 1
			for (int s = 0; s != S; ++s) {
				bool has = false; f3 w = zero, c = zero; float tmax = 0.0f;
				if (on) {
					const f3 dd = sample_psa<MAXP, BIASED>(pd, next_noise_2(ns, p, cb, px, py));
					w = shading_to_world(l, sp.normal, flip, dd);
					if (dot(sp.normal, w) > 0.0f) {
						has = true;
						tmax = light_plane_distance(sp, light, w);
						c = (light_radiance<LIGHT_TEXTURES>(p, light, sp.position, w) * evaluate_brdf<true, false>(sp, w)) * pd.psa;
					}
				}
				submit<TRACE, false>(q, lane, has, true, w, tmax, c, zero, result, false);
				has = false;
				if (has_specular) {
					const f3 dc = sample_psa<MAXP, BIASED>(ps, next_noise_2(ns, p, cb, px, py));
					const f3 dsh = normalize(c2s_mul(l, dc));
					const float ltc_density = evaluate_ltc_density(l, dsh, 1.0f);
					w = shading_to_world(l, sp.normal, flip, dsh);
					if (!(dsh.z <= 0.0f || dc.z <= 0.0f)) { // :587; true for NaN directions
						const float hidden = 0.0f * dsh.z * ps.psa / ltc_density; // what one channel of the shader's expression is for a sample that is not visible
						if (hidden != hidden) { has = true; tmax = 0.0f; w = zero; c = not_a_number3(); } // NaN either way, see above
						else if (dot(sp.normal, w) > 0.0f) {
							has = true;
							tmax = light_plane_distance(sp, light, w);
							const f3 rtb2 = light_radiance<LIGHT_TEXTURES>(p, light, sp.position, w) * evaluate_brdf<false, true>(sp, w);
							c = make3(rtb2.x * dsh.z * ps.psa / ltc_density, rtb2.y * dsh.z * ps.psa / ltc_density, rtb2.z * dsh.z * ps.psa / ltc_density);
						}
					}
				}
				submit<TRACE, false>(q, lane, has, true, w, tmax, c, zero, result, false);
			}
		}
		else if (STRATEGY == VKR_STRATEGY_DIFFUSE_SPECULAR_MIS) {
			f3 diffuse_weight = make3(max_glsl(sp.diffuse_albedo.x, 0.01f), max_glsl(sp.diffuse_albedo.y, 0.01f), max_glsl(sp.diffuse_albedo.z, 0.01f)) * pd.psa;
			const float rcp_d = 1.0f / pd.psa;
			const float rcp_s = 1.0f / ps.psa;
			f3 specular_weight_rgb = make3(specular_weight, specular_weight, specular_weight);
			if (OPTIMAL) {
				const f3 radiance_over_pi = light_radiance(light) * kInvPi;
				diffuse_weight = diffuse_weight * radiance_over_pi;
				specular_weight_rgb = specular_weight_rgb * radiance_over_pi;
			}
			const float v_est = ldf(cb, OFF_MIS_VIS);
#pragma unroll 1
			// The reference draws the diffuse and the specular sample first and then evaluates both (:610-636); drawing
			// each sample right before its evaluation consumes the noise stream in the same order. One loop body serves
			// both techniques and the end-of-light flush (s == S), so the kernel holds one copy of sample_psa and drain.
			for (int s = 0; s <= S; ++s) {
#pragma unroll 1
				for (int j = 0; j != 2; ++j) {
					bool has = on && s != S && (j == 0 || has_specular);
					bool pre_vis = false; f3 w = zero, c = zero, c_occ = zero; float tmax = 0.0f;
					if (has) {
						f3 d = sample_psa<MAXP, BIASED>(select_polygon(j != 0, pd, ps), next_noise_2(ns, p, cb, px, py));
						if (j != 0) d = normalize(c2s_mul(l, d));
						has = !(d.z <= 0.0f); // as the shader writes it (:619): a NaN direction (degenerate, nearly edge-on polygon) is not skipped, it poisons the pixel
						if (has) {
							const float diffuse_density = d.z * rcp_d;
							const float specular_density = evaluate_ltc_density(l, d, rcp_s);
							w = shading_to_world(l, sp.normal, flip, d);
							pre_vis = dot(sp.normal, w) > 0.0f;
							f3 integrand = zero;
							if (pre_vis) {
								tmax = light_plane_distance(sp, light, w);
								integrand = (light_radiance<LIGHT_TEXTURES>(p, light, sp.position, w) * evaluate_brdf<true, true>(sp, w)) * d.z;
							}
							if (j == 0 && !has_specular) { // one technique only: no MIS (:629-631)
								c = integrand * (1.0f / diffuse_density);
								has = pre_vis;
							}
							else {
								const f3 w_own = (j == 0) ? diffuse_weight : specular_weight_rgb, w_other = (j == 0) ? specular_weight_rgb : diffuse_weight;
								const float p_own = (j == 0) ? diffuse_density : specular_density, p_other = (j == 0) ? specular_density : diffuse_density;
								c = mis_estimate(p.mis_heuristic, integrand, w_own, p_own, w_other, p_other, v_est);
								if (OPTIMAL) c_occ = mis_estimate(p.mis_heuristic, zero * d.z, w_own, p_own, w_other, p_other, v_est);
								else if (!pre_vis || !is_finite(c)) {
									// The shader multiplies a ZERO integrand by the MIS weights when the sample is not visible (:633-636); with degenerate
									// densities the weights are not finite and 0 * inf = NaN turns the pixel pink whatever the shadow ray says. Such a sample
									// is pushed as a certain miss (tmax = 0) carrying NaN. Found by tools/fuzz_parity.py; about one pixel in a million.
									const f3 c_hidden = pre_vis ? mis_estimate(p.mis_heuristic, zero, w_own, p_own, w_other, p_other, v_est) : c;
									if (c_hidden.x != c_hidden.x || c_hidden.y != c_hidden.y || c_hidden.z != c_hidden.z) {
										pre_vis = true; tmax = 0.0f; w = zero;
										c = make3(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
									}
								}
							}
						}
					}
					submit<TRACE, OPTIMAL>(q, lane, has, pre_vis, w, tmax, c, c_occ, result, s == S);
				}
			}
			return;
		}
		else { // VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM
			const float diffuse_albedo = max_glsl(dot(sp.diffuse_albedo, make3(0.21263901f, 0.71516868f, 0.07219232f)), 0.01f);
			const float diffuse_weight = diffuse_albedo * pd.psa;
			const float diffuse_ratio = diffuse_weight / (diffuse_weight + specular_weight);
#pragma unroll 1
			for (int s = 0; s != S; ++s) {
				bool has = false; f3 w = zero, c = zero; float tmax = 0.0f;
				if (on) {
					f2 rnd = next_noise_2(ns, p, cb, px, py);
					const bool specular_selected = rnd.x >= diffuse_ratio;
					const float offset = specular_selected ? 1.0f : 0.0f;
					rnd.x = (rnd.x - offset) / (diffuse_ratio - offset);
					f3 d = specular_selected ? sample_psa<MAXP, BIASED>(ps, rnd) : sample_psa<MAXP, BIASED>(pd, rnd);
					if (specular_selected) d = normalize(c2s_mul(l, d));
					const float diffuse_density = d.z * diffuse_albedo;
					const float specular_density = evaluate_ltc_density(l, d, specular_albedo);
					const float density = (diffuse_density + specular_density) / (diffuse_weight + specular_weight);
					w = shading_to_world(l, sp.normal, flip, d);
					if (!(d.z <= 0.0f)) { // :669; true for a NaN direction
						const float hidden = 0.0f * d.z / density; // what one channel of the shader's expression is for a sample that is not visible
						if (hidden != hidden) { has = true; tmax = 0.0f; w = zero; c = not_a_number3(); } // NaN either way, see above
						else if (dot(sp.normal, w) > 0.0f) {
							has = true;
							tmax = light_plane_distance(sp, light, w);
							const f3 rtb = light_radiance<LIGHT_TEXTURES>(p, light, sp.position, w) * evaluate_brdf<true, true>(sp, w);
							c = make3(rtb.x * d.z / density, rtb.y * d.z / density, rtb.z * d.z / density);
						}
					}
				}
				submit<TRACE, false>(q, lane, has, true, w, tmax, c, zero, result, false);
			}
		}
	}
	submit<TRACE, OPTIMAL>(q, lane, false, false, zero, 0.0f, zero, zero, result, true);
}

// The light shader of this translation unit: projected solid angle sampling with the five sampling strategies
template <int STRATEGY, int MAXP, bool BIASED, bool OPTIMAL, bool TRACE, bool LIGHT_TEXTURES = false>
struct psa_light_shader {
	VKR_DEV void operator()(bool on, const shading_point& sp, const ltc_state& l, const unsigned char* light, noise_stream& ns,
		const shading_kernel_params& p, const unsigned char* cb, uint32_t px, uint32_t py, ray_producer& q, pixel_sum& result, int lane) const
	{
		shade_light<STRATEGY, MAXP, BIASED, OPTIMAL, TRACE, LIGHT_TEXTURES>(on, sp, l, light, ns, p, cb, px, py, q, result, lane);
	}
};

} // namespace vkr
