// vkr_anchor.cuh -- anchored shadow rays: what all shadow rays of one pixel, and of one (pixel, light) pair, have in common is done once.
//
// Every shadow ray of a pixel starts at the same surface point o, inside the same chain of nested boxes from the root of the BVH down to the leaf
// that holds the surface. A plain any-hit traversal re-discovers that chain for each of the ~10^3 rays of the pixel (about 20 of the ~40 node
// visits per ray in the benchmark scene) only to learn what was known beforehand: a ray leaves every box that contains its origin.
//
//   origin path   per pixel, once: the root-to-leaf chain of node pairs along the child whose box contains o (any chain would be correct: the
//                 SIBLINGS hanging off a root-to-leaf chain plus the node at its end partition the triangles). Entry k = pair index * 2 + the
//                 child that continues the chain; the chain is cut after kPathLevels pairs, its end ("tail") is then an inner node.
//   light cone    per (pixel, light), once: a cone with apex o around the light polygon and the distance of its farthest vertex. A sibling whose
//                 box (its bounding sphere, to be exact) lies outside the cone cannot be hit by a ray to this light: one bit per path level.
//   the ray       starts with the tail and the surviving siblings instead of the root: a sibling step is an ordinary
//                 node visit with the chain's child masked out.
// Soundness does not rest on the sampler: every ray is checked against the cone when it is submitted (ray_in_cone, with the thresholds the
// cone was built from; the culling uses a slightly wider and longer cone), and a ray that is not inside keeps all siblings. Hit / miss stays
// the OR over all triangles the predicate accepts, so frames are bit-identical to the plain traversal.
// No shading kernel starts its rays this way (DESIGN.md section 3, editions of the trace warps that were removed); the CPU tests run these pieces.
#pragma once
#include "vkr_trace.cuh"

namespace vkr {

constexpr int kPathLevels = 20;              // chain pairs remembered per pixel (one bit each in the sibling masks); deeper trees continue in the tail
constexpr uint32_t kAllSiblings = 0xffffffffu;

VKR_DEV bool box_contains(float cx, float cy, float cz, float hx, float hy, float hz, f3 o) {
	return fabsf(o.x - cx) <= hx && fabsf(o.y - cy) <= hy && fabsf(o.z - cz) <= hz;
}

// Walks from the root along the child whose box contains o (both: the smaller box; neither, which only rounding at a box face can cause: the
// nearer centre). store(k, entry) receives the chain, *tail the reference (inner node or leaf) the chain ends in. Returns the number of entries.
template <class Store>
VKR_DEV int find_origin_path(const float4* __restrict__ nodes, f3 o, int* tail, Store&& store) {
	int node = 0, count = 0;
	while (true) {
		const float4* nd = nodes + 4 * (size_t) node;
		const float4 q0 = __ldg(nd), q1 = __ldg(nd + 1), q2 = __ldg(nd + 2), q3 = __ldg(nd + 3);
		const bool in0 = box_contains(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, o), in1 = box_contains(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, o);
		int child;
		if (in0 != in1) child = in1 ? 1 : 0;
		else if (in0) child = (q2.y + q2.z + q2.w < q0.w + q1.x + q1.y) ? 1 : 0;
		else {
			const float d0 = fabsf(o.x - q0.x) + fabsf(o.y - q0.y) + fabsf(o.z - q0.z), d1 = fabsf(o.x - q1.z) + fabsf(o.y - q1.w) + fabsf(o.z - q2.x);
			child = (d1 < d0) ? 1 : 0;
		}
		store(count, (uint32_t) node * 2u + (uint32_t) child);
		++count;
		const int ref = __float_as_int(child ? q3.y : q3.x);
		if (ref < 0 || count == kPathLevels) { *tail = ref; return count; }
		node = ref;
	}
}

// Cone around the light as seen from o. `valid` quantities are what a ray is checked against, `cull` quantities (a little wider, a little longer)
// what boxes are culled against; enabled = false (light too close or too big to be worth it, degenerate numbers): all siblings stay.
struct light_cone {
	f3 axis;                       // unit
	float cos2_valid, len2_valid;  // ray inside: axis.w > 0, (axis.w)^2 >= cos2_valid * w.w, tmax^2 * w.w <= len2_valid
	float cos_cull, sin_cull, len_cull;
	bool enabled;
};

// vertices: world-space vertices of the light polygon, 16 bytes apart (the constant block's layout), count of them
VKR_DEV light_cone make_light_cone(f3 o, const unsigned char* vertices, int count) {
	light_cone c;
	f3 sum = make3(0.0f, 0.0f, 0.0f);
	float len2 = 0.0f;
	for (int i = 0; i != count; ++i) {
		const float* v = reinterpret_cast<const float*>(vertices + 16 * i);
		const f3 e = make3(v[0] - o.x, v[1] - o.y, v[2] - o.z);
		const float l2 = dot(e, e);
		len2 = fmaxf(len2, l2);
		sum = sum + e * (1.0f / sqrtf(l2));
	}
	c.axis = sum * (1.0f / sqrtf(dot(sum, sum)));
	float cos_min = 1.0f;
	for (int i = 0; i != count; ++i) {
		const float* v = reinterpret_cast<const float*>(vertices + 16 * i);
		const f3 e = make3(v[0] - o.x, v[1] - o.y, v[2] - o.z);
		cos_min = fminf(cos_min, dot(c.axis, e) * (1.0f / sqrtf(dot(e, e))));
	}
	// What makes the cone valid is the per-ray check (ray_in_cone); the vertices only make it tight. A little slack keeps samples on the border inside.
	const float cos_valid = cos_min * 0.999f - 1.0e-3f;
	c.cos2_valid = cos_valid * cos_valid;
	c.len2_valid = len2 * 1.002f;
	c.cos_cull = cos_valid * 0.999f - 1.0e-4f;
	c.sin_cull = sqrtf(fmaxf(0.0f, 1.0f - c.cos_cull * c.cos_cull)) * 1.001f + 1.0e-4f;
	c.len_cull = sqrtf(c.len2_valid) * 1.001f;
	// NaN or inf anywhere (a vertex at o, an overflow) fails the comparisons and disables the cone
	c.enabled = cos_valid > 0.25f && c.cos_cull > 0.0f && c.len_cull < 3.0e37f && c.sin_cull < 2.0f && dot(c.axis, c.axis) > 0.5f;
	return c;
}

// Is the segment {o + t w : 0 < t < tmax} inside the cone? Decided in the cone's own (valid) numbers; NaN says no.
VKR_DEV bool ray_in_cone(const light_cone& c, f3 w, float tmax) {
	const float aw = dot(c.axis, w), ww = dot(w, w);
	return c.enabled && aw > 0.0f && aw * aw >= c.cos2_valid * ww && tmax * tmax * ww <= c.len2_valid;
}

// Can a point of the cull cone lie in the sphere around centre c with radius r (+ slack)? Distance from the sphere's centre to the infinite cone
// (apex o, axis a, half angle theta): |v| behind the apex's normal cone, else |v| sin(phi - theta); plus the cap at len_cull along the axis.
VKR_DEV bool sphere_may_touch_cone(const light_cone& c, f3 v, float r) {
	const float slack = r * 1.001f + 1.0e-5f * (fabsf(v.x) + fabsf(v.y) + fabsf(v.z) + r);
	const float along = dot(v, c.axis);
	const float vv = dot(v, v);
	const float perp = sqrtf(fmaxf(0.0f, vv - along * along));
	if (along - slack > c.len_cull) return false;                         // beyond the far end of every ray
	const float outside = perp * c.cos_cull - along * c.sin_cull;          // |v| sin(phi - theta): > 0 outside the cone
	if (!(outside > 0.0f)) return true;                                   // centre inside the cone (or NaN)
	const float behind = along * c.cos_cull + perp * c.sin_cull;           // |v| cos(phi - theta): < 0 where the apex is the nearest point
	const float distance = (behind < 0.0f) ? sqrtf(vv) : outside;
	return !(distance > slack);
}

// One bit per path level: may the sibling of that level be hit by a ray inside the cone? load(k) returns entry k of the path.
template <class Load>
VKR_DEV uint32_t cull_siblings(const float4* __restrict__ nodes, f3 o, const light_cone& c, int count, Load&& load) {
	if (!c.enabled) return kAllSiblings;
	uint32_t mask = 0u;
	for (int k = 0; k != count; ++k) {
		const uint32_t entry = load(k);
		const float4* nd = nodes + 4 * (size_t) (entry >> 1);
		float cx, cy, cz, hx, hy, hz;
		if (entry & 1u) { const float4 q0 = __ldg(nd), q1 = __ldg(nd + 1); cx = q0.x; cy = q0.y; cz = q0.z; hx = q0.w; hy = q1.x; hz = q1.y; }   // the chain goes on in child 1: the sibling is child 0
		else { const float4 q1 = __ldg(nd + 1), q2 = __ldg(nd + 2); cx = q1.z; cy = q1.w; cz = q2.x; hx = q2.y; hy = q2.z; hz = q2.w; }
		const float r = sqrtf(fmaf(hz, hz, fmaf(hy, hy, hx * hx)));
		if (sphere_may_touch_cone(c, make3(cx - o.x, cy - o.y, cz - o.z), r)) mask |= 1u << k;
	}
	return mask;
}

// One visit of node pair `pair` with child `skip` (0, 1; anything else: none) left out: returns the nearer child that the ray hits (the other one goes to
// push()), kTraversalDone if none.
template <class Push>
VKR_DEV int visit_pair(const float4* __restrict__ nodes, int pair, int skip, const ray_slabs& r, float tmin, float tmax, Push&& push) {
	const float4* nd = nodes + 4 * (size_t) pair;
	float4 q0, q1, q2, q3;
	ldg_32_bytes(nd, q0, q1); ldg_32_bytes(nd + 2, q2, q3);
	const int ref0 = __float_as_int(q3.x), ref1 = __float_as_int(q3.y);
	float tn0, tn1;
	const bool h0 = ray_box(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, r, tmin, tmax, &tn0) && skip != 0;
	const bool h1 = ray_box(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, r, tmin, tmax, &tn1) && skip != 1;
	if (h0 && h1) {
		const bool swap = tn1 < tn0;
		push(swap ? ref0 : ref1);
		return swap ? ref1 : ref0;
	}
	return h0 ? ref0 : (h1 ? ref1 : kTraversalDone);
}

// Per-thread any-hit query of an anchored ray, run on the CPU against occluded() by
// tests/test_device_on_host.py. path / count / tail: find_origin_path(o); mask: cull_siblings() for a cone the ray is inside of, or kAllSiblings.
VKR_DEV bool occluded_anchored(const bvh_view& bvh, f3 o, f3 d, float tmin, float tmax, const uint32_t* path, int count, int tail, uint32_t mask, int* stack, int stride, int* visits) {
	if (!(tmax > tmin)) return false;
	const ray_slabs r = make_slabs(o, d);
	int sp = 0;
	auto push = [&](int ref) { stack[sp * stride] = ref; ++sp; };
	uint32_t pending = (count >= 32) ? mask : (mask & ((1u << count) - 1u));
	int node = tail;
	float t;
	while (true) {
		if (node < 0) { // a leaf
			const int first = (node & 0x7fffffff) >> 4, n = node & 15;
			for (int i = 0; i != n; ++i)
				if (ray_triangle(bvh.tris + 3 * (size_t) (first + i), o, d, tmin, tmax, &t)) return true;
			node = kTraversalDone;
		}
		else if (node != kTraversalDone) {
			if (visits) ++*visits;
			node = visit_pair(bvh.nodes, node, 2, r, tmin, tmax, push);
		}
		else if (sp) { --sp; node = stack[sp * stride]; }
		else if (pending) { // the deepest sibling left: the nearest to the origin
			const int k = 31 - __clz((int) pending);
			pending &= ~(1u << k);
			if (visits) ++*visits;
			node = visit_pair(bvh.nodes, (int) (path[k] >> 1), (int) (path[k] & 1u), r, tmin, tmax, push);
		}
		else return false;
	}
}

} // namespace vkr
