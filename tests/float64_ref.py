"""Plain float64 references for the two primitives every frame rests on, projected-solid-angle (PSA) sampling of a horizon-clipped polygon
(vkr_psa.cuh) and the any-hit shadow query (vkr_trace.cuh), and for what a frame estimates: the BRDF (brdfs.glsl) and the direct lighting, the
BRDF times the cosine integrated over the lights minus what occluders cover (direct_lighting). numpy only; nothing here shares code or operation
order with the oracle or the kernels.

Polygons are (n, 3) arrays of vertices seen from the origin, the shading normal is +z. Rays are rows {ox, oy, oz, dx, dy, dz, tmin, tmax}.
"""
import math

import numpy as np


def _clip_halfspace(poly, normal):
	"""Sutherland-Hodgman: the part of the polygon (list of 3-tuples) where dot(normal, p) > 0, with the crossing points on the plane."""
	out = []
	n = len(poly)
	for i in range(n):
		a, b = poly[i], poly[(i + 1) % n]
		sa = normal[0] * a[0] + normal[1] * a[1] + normal[2] * a[2]
		sb = normal[0] * b[0] + normal[1] * b[1] + normal[2] * b[2]
		if sa > 0.0:
			out.append(a)
		if (sa > 0.0) != (sb > 0.0):
			w = sa / (sa - sb)
			out.append((a[0] + w * (b[0] - a[0]), a[1] + w * (b[1] - a[1]), a[2] + w * (b[2] - a[2])))
	return out


def vector_irradiance(poly):
	"""The integral of the direction w over a spherical polygon (smaller than a hemisphere), half the sum over its edges of the arc length times the
	edge plane's unit normal (Lambert), oriented towards the polygon. Edges of length zero (a clip crossing that coincides with a vertex) contribute
	nothing."""
	total = np.zeros(3)
	n = len(poly)
	unit = []
	for p in poly:
		r = math.sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2])
		unit.append((p[0] / r, p[1] / r, p[2] / r))
	for i in range(n):
		a, b = unit[i], unit[(i + 1) % n]
		cx, cy, cz = a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]
		s = math.sqrt(cx * cx + cy * cy + cz * cz)
		if s == 0.0:
			continue
		total += math.atan2(s, a[0] * b[0] + a[1] * b[1] + a[2] * b[2]) / s * np.array([cx, cy, cz])
	total *= 0.5
	return -total if total @ np.sum(unit, axis=0) < 0.0 else total


def lambert_psa(poly):
	"""Projected solid angle of a spherical polygon in the upper hemisphere: the z component of its vector irradiance."""
	return abs(float(vector_irradiance(poly)[2]))


def solid_angle(poly):
	"""Solid angle of a convex polygon seen from the origin: a fan of triangles around vertex 0, each by Van Oosterom and Strackee (1983),
	tan(omega / 2) = |det(a, b, c)| / (|a||b||c| + (a.b)|c| + (b.c)|a| + (c.a)|b|). The determinant is taken over the edges from a, which keeps
	its relative accuracy for distant specks."""
	P = np.asarray(poly, dtype=np.float64)
	r = np.linalg.norm(P, axis=1)
	total = 0.0
	for k in range(1, len(P) - 1):
		a, b, c = P[0], P[k], P[k + 1]
		det = abs(float(np.dot(a, np.cross(b - a, c - a))))
		total += 2.0 * math.atan2(det, r[0] * r[k] * r[k + 1] + (a @ b) * r[k + 1] + (b @ c) * r[0] + (c @ a) * r[k])
	return total


def clip_and_psa(pts, horizon_eps=1.0e-6):
	"""Clip at z = 0 (a vertex is kept when z > 0, as in the kernel's case table) and return (psa, clipped vertex count, ill_conditioned, clipped
	polygon). ill_conditioned: a vertex lies within horizon_eps (relative to its distance) of the horizon, where the vertex count can go either way."""
	poly = [tuple(float(c) for c in p) for p in np.asarray(pts, dtype=np.float64)]
	clipped = _clip_halfspace(poly, (0.0, 0.0, 1.0))
	near = any(abs(p[2]) <= horizon_eps * math.sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]) for p in poly)
	return (lambert_psa(clipped) if len(clipped) >= 3 else 0.0), len(clipped), near, clipped


def psa_of_region(pts, normals):
	"""PSA of the part of the z-clipped polygon on the positive side of every plane through the origin with the given normals."""
	region = clip_and_psa(pts)[3]
	for nrm in normals:
		if len(region) < 3:
			return 0.0
		region = _clip_halfspace(region, tuple(float(c) for c in nrm))
	return lambert_psa(region) if len(region) >= 3 else 0.0


def _edge_normals(pts):
	"""Unit normals of the planes through the origin and each edge, oriented so that the polygon's cone lies on their positive side."""
	P = np.asarray(pts, dtype=np.float64)
	N = np.cross(P, np.roll(P, -1, axis=0))
	length = np.linalg.norm(N, axis=1)
	N = N[length > 0] / length[length > 0, None]
	centre = (P / np.linalg.norm(P, axis=1, keepdims=True)).mean(0)
	return N if (N @ centre).sum() >= 0 else -N


def in_polygon_cone(dirs, pts, margin):
	"""1 where a direction lies inside the cone over the polygon by more than `margin` (sine of the angle to every edge plane), 0 where it lies
	outside one edge plane by more than `margin`, -1 (undecided) otherwise."""
	s = np.asarray(dirs, dtype=np.float64) @ _edge_normals(pts).T
	out = np.full(len(s), -1, dtype=np.int8)
	out[(s > margin).all(axis=1)] = 1
	out[(s < -margin).any(axis=1)] = 0
	return out


def sample_cdf_position(pts, first_vertex, central, d):
	"""Where a sample direction d sits in the sampler's order of the polygon, as a fraction of its PSA: the PSA of the part swept before d,
	over the PSA of the whole (z-clipped) polygon. The sampler sweeps azimuth: counter-clockwise from the most clockwise vertex when the zenith is
	outside the polygon, from the first clipped vertex in the order of the clipped vertices when it is inside (`first_vertex`, `central`:
	the second vertex of that order decides the sense of rotation, pass (v0, v1))."""
	total = clip_and_psa(pts)[0]
	if not central:
		return psa_of_region(pts, [(d[1], -d[0], 0.0)]) / total
	v0, v1 = first_vertex
	sense = 1.0 if v0[0] * v1[1] - v0[1] * v1[0] >= 0.0 else -1.0
	def wedge(a, b):   # the part between azimuths a and b, swept in `sense` (at most half a turn)
		return psa_of_region(pts, [(-sense * a[1], sense * a[0], 0.0), (sense * b[1], -sense * b[0], 0.0)])
	if sense * (v0[0] * d[1] - v0[1] * d[0]) >= 0.0:
		return wedge(v0, d) / total
	return 1.0 - wedge(d, v0) / total


def shadow_truth(tris, rays, rel_margin=2.0 ** -20, chunk_elements=1 << 21):
	"""float64 Moeller-Trumbore of every ray against every triangle. Returns (hit, decided) as bool arrays.

	The triangles are the fp32 vertex triples (9 floats per row, taken as exact). In the fp32 predicate each numerator is a cross product and a dot
	product of inputs that were rounded once (o - p0, the edges): fewer than 8 roundings of 2^-24 relative to the product of the norms involved. The
	default rel_margin, 2^-20, is 16 of them, and the margins below are twice the resulting bounds. Each quantity gets an error bound rel_margin times
	the product of the norms it is made of (numerator of u: |o - p0| |d| |e2|,
	of v: |d| |o - p0| |e1|, of t: |e2| |o - p0| |e1|, the determinant: |e1| |d| |e2|). A triangle is a clear hit when u, v, 1 - u - v and the
	distances of t to tmin and tmax all exceed their bounds, a clear miss when one of them is below minus its bound, or when the segment
	[tmin, tmax] stays on one side of the triangle's plane by more than the bound of that distance (this decides near-parallel triangles, whose
	small determinant leaves u, v and t unbounded). A ray is decided when one triangle is a clear hit or every triangle is a clear miss; an empty
	or NaN interval is a decided miss (the predicate's definition)."""
	T = np.asarray(tris, dtype=np.float32).reshape(-1, 3, 3).astype(np.float64)
	R = np.asarray(rays, dtype=np.float32).reshape(-1, 8).astype(np.float64)
	p0 = T[:, 0]; e1 = T[:, 1] - T[:, 0]; e2 = T[:, 2] - T[:, 0]
	n1 = np.linalg.norm(e1, axis=1); n2 = np.linalg.norm(e2, axis=1)
	hit = np.zeros(len(R), dtype=bool); decided = np.zeros(len(R), dtype=bool)
	step = max(1, chunk_elements // max(len(T), 1))
	E = rel_margin
	with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
		for s in range(0, len(R), step):
			r = R[s:s + step]
			o = r[:, None, 0:3]; d = r[:, None, 3:6]; tmin = r[:, 6:7]; tmax = r[:, 7:8]
			nd = np.linalg.norm(r[:, 3:6], axis=1)[:, None]
			pv = np.cross(d, e2[None]); det = (e1[None] * pv).sum(-1)
			tv = o - p0[None]; nt = np.linalg.norm(tv, axis=2)
			qv = np.cross(tv, e1[None])
			num_u = (tv * pv).sum(-1); num_v = (d * qv).sum(-1); num_t = (e2[None] * qv).sum(-1)
			e_det = E * n1[None] * nd * n2[None]; e_u = E * nt * nd * n2[None]; e_v = E * nd * nt * n1[None]; e_t = E * n2[None] * nt * n1[None]
			# the segment's plane distances (times |n|): g(t) = num_t - t det vanishes at the hit distance
			finite_max = np.isfinite(tmax)
			tmax_f = np.where(finite_max, tmax, 0.0)
			g0 = num_t - tmin * det; b0 = e_t + np.abs(tmin) * e_det
			g1 = np.where(finite_max, num_t - tmax_f * det, -det); b1 = np.where(finite_max, e_t + np.abs(tmax_f) * e_det, e_det)
			plane_miss = (np.abs(g0) > b0) & (np.abs(g1) > b1) & (np.sign(g0) == np.sign(g1))
			well = np.abs(det) > 2.0 * e_det
			adet = np.abs(det)
			u = num_u / det; v = num_v / det; t = num_t / det
			mu = 2.0 * (e_u + np.abs(u) * e_det) / adet; mv = 2.0 * (e_v + np.abs(v) * e_det) / adet; mt = 2.0 * (e_t + np.abs(t) * e_det) / adet
			clear_hit = well & (u > mu) & (v > mv) & (1.0 - u - v > mu + mv) & (t - tmin > mt) & (tmax - t > mt)
			clear_miss = plane_miss | (well & ((u < -mu) | (v < -mv) | (u + v > 1.0 + mu + mv) | (t < tmin - mt) | (t > tmax + mt)))
			empty = ~(r[:, 7] > r[:, 6])
			any_hit = clear_hit.any(axis=1) & ~empty
			hit[s:s + step] = any_hit
			decided[s:s + step] = any_hit | clear_miss.all(axis=1) | empty
	return hit, decided


# ---- the shading pass's integral: BRDF times cosine times radiance over the lights, with occluders ------------------------------------------

def brdf(wi, wo, n, albedo, f0, roughness):
	"""The BRDF of brdfs.glsl (diffuse and specular lobes, each on or off), in world space, for unit incoming directions wi [m, 3] and one unit
	outgoing direction wo and normal n: Frostbite's diffuse term albedo / pi * F_D(n.wo) * F_D(n.wi) with F_D(c) = 1 + (F90 - 1) (1 - c)^5,
	F90 = 0.5 + 2 roughness (wo.h)^2, plus GGX with alpha = roughness, height-correlated Smith and Schlick's Fresnel per channel of f0
	(ltc_fit.specular_brdf). Returns (diffuse [m, 3], specular [m, 3])."""
	from vulkan_renderer_b200.ltc_fit import specular_brdf
	wi = np.asarray(wi, dtype=np.float64); wo = np.asarray(wo, dtype=np.float64); n = np.asarray(n, dtype=np.float64)
	t, b = _tangent_frame(n)
	local = np.stack([wi @ t, wi @ b, wi @ n], axis=-1)
	wo_local = np.array([wo @ t, wo @ b, wo @ n])
	h = local + wo_local
	h /= np.linalg.norm(h, axis=-1, keepdims=True)
	oh = h @ wo_local
	f90 = 0.5 + 2.0 * roughness * oh * oh
	schlick = lambda c: 1.0 + (f90 - 1.0) * (1.0 - c) ** 5
	diffuse = (schlick(wo_local[2]) * schlick(local[:, 2]))[:, None] * np.asarray(albedo, dtype=np.float64)[None] / math.pi
	specular = np.stack([specular_brdf(wo_local, local, roughness, float(f)) for f in f0], axis=-1)
	return diffuse, specular


def _tangent_frame(n):
	n = np.asarray(n, dtype=np.float64)
	a = np.array([1.0, 0.0, 0.0]) if abs(n[0]) < 0.8 else np.array([0.0, 1.0, 0.0])
	t = a - (a @ n) * n; t /= np.linalg.norm(t)
	return t, np.cross(n, t)


_GAUSS_NODES, _GAUSS_WEIGHTS = np.polynomial.legendre.leggauss(8)
_GAUSS_NODES = 0.5 * (_GAUSS_NODES + 1.0); _GAUSS_WEIGHTS = 0.5 * _GAUSS_WEIGHTS


def _triangle_rule(tris, g):
	"""Gauss-Legendre 8 x 8 through the Duffy map (s, t) -> a + s (b - a) + s t (c - b), Jacobian 2 area s, for triangles [T, 3, 3]: [T, c]."""
	s = _GAUSS_NODES[:, None]; t = _GAUSS_NODES[None, :]
	a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
	p = a[:, None, None] + s[None, :, :, None] * (b - a)[:, None, None] + (s * t)[None, :, :, None] * (c - b)[:, None, None]
	w = (_GAUSS_WEIGHTS[:, None] * _GAUSS_WEIGHTS[None, :] * s)[None] * np.linalg.norm(np.cross(b - a, c - b), axis=-1)[:, None, None]
	values = g(p.reshape(-1, 3)).reshape(len(tris), len(_GAUSS_NODES), len(_GAUSS_NODES), -1)
	return (values * w[..., None]).sum(axis=(1, 2))


def integrate_polygon(poly, g, rtol=1e-10, atol=0.0, max_levels=40, max_triangles=1 << 16):
	"""The integral of g (points [m, 3] -> values [m, c]) over a planar convex polygon [k, 3]: a fan of triangles, each refined 4 ways (midpoints of
	the edges) until the rule on a triangle and the sum of the rule on its four children agree to rtol of the whole (or to atol, if larger), with
	each triangle's share of the tolerance in proportion to its area. Returns (integral [c], levels used)."""
	P = np.asarray(poly, dtype=np.float64)
	tris = np.stack([np.broadcast_to(P[0], (len(P) - 2, 3)), P[1:-1], P[2:]], axis=1)
	area_of = lambda T: 0.5 * np.linalg.norm(np.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0]), axis=-1)
	total_area = float(area_of(tris).sum())
	if total_area == 0.0:
		return 0.0, 0
	parent = _triangle_rule(tris, g)
	result = np.zeros(parent.shape[1])
	scale = None
	for level in range(max_levels):
		m = (tris + np.roll(tris, -1, axis=1)) * 0.5      # midpoints of the edges ab, bc, ca
		kids = np.stack([np.stack([tris[:, 0], m[:, 0], m[:, 2]], 1), np.stack([m[:, 0], tris[:, 1], m[:, 1]], 1),
			np.stack([m[:, 2], m[:, 1], tris[:, 2]], 1), np.stack([m[:, 0], m[:, 1], m[:, 2]], 1)], axis=1)
		child = _triangle_rule(kids.reshape(-1, 3, 3), g).reshape(len(tris), 4, -1)
		fine = child.sum(axis=1)
		if scale is None:
			scale = max(float(np.abs(fine.sum(axis=0)).max()), atol / rtol, 1e-300)
		done = np.abs(fine - parent).max(axis=1) <= rtol * scale * area_of(tris) / total_area
		result += fine[done].sum(axis=0)
		if done.all():
			return result, level + 1
		tris = kids[~done].reshape(-1, 3, 3); parent = child[~done].reshape(-1, child.shape[2])
		if len(tris) > max_triangles:
			break
	raise RuntimeError("integrate_polygon: no convergence to %g after %d levels, %d triangles left" % (rtol, level + 1, len(tris)))


def _plane_normal(poly):
	P = np.asarray(poly, dtype=np.float64)
	nrm = sum(np.cross(P[i] - P[0], P[i + 1] - P[0]) for i in range(1, len(P) - 1))
	return nrm / np.linalg.norm(nrm)


def light_integral(x, n, poly, g, occluders=(), planes=(), rtol=1e-10):
	"""The integral over directions w of g(w) [m, c] where the light polygon [k, 3] (world space, emitting on both faces) lies above x's tangent
	plane (n . w > 0) and on the positive side of the extra planes through x (normals `planes`), minus the part whose segment to x crosses one of
	the occluder triangles [3, 3]. Integrated over the polygon's area with dw = |n_L . (p - x)| / |p - x|^3 dA. Each occluder must lie strictly
	between x and the light's plane, their central projections onto it must not overlap (the two halves of a quad do not)."""
	x = np.asarray(x, dtype=np.float64); n = np.asarray(n, dtype=np.float64)
	P = np.asarray(poly, dtype=np.float64) - x
	nl = _plane_normal(P); height = float(P[0] @ nl)
	def integrand(p):
		r = np.linalg.norm(p, axis=-1)
		return g(p / r[:, None]) * (abs(height) / r ** 3)[:, None]
	def region_integral(region, atol=0.0):
		return integrate_polygon(np.array(region), integrand, rtol, atol)[0] if len(region) >= 3 else 0.0
	region = _clip_halfspace([tuple(p) for p in P], tuple(n))
	atol = 0.0
	if len(planes):   # a sliver cut off by the extra planes is integrated to rtol of the whole light, not of itself
		atol = rtol * float(np.abs(region_integral(region)).max())
	for normal in planes:
		region = _clip_halfspace(region, tuple(normal)) if len(region) >= 3 else region
	total = unshadowed = region_integral(region, atol)
	for tri in occluders:
		T = np.asarray(tri, dtype=np.float64) - x
		depth = (T @ nl) / height                        # 0 at x, 1 on the light's plane
		if (depth <= 0.0).all() or (depth >= 1.0).all():
			continue
		if not ((depth > 0.0) & (depth < 1.0)).all():
			raise ValueError("an occluder crosses x's plane or the light's plane: %s" % tri)
		shadow = region
		centre = T.mean(axis=0)
		for i in range(3):
			e = np.cross(T[i], T[(i + 1) % 3])
			e = e if e @ centre > 0.0 else -e
			shadow = _clip_halfspace(shadow, tuple(e)) if len(shadow) >= 3 else shadow
		total = total - region_integral(shadow, atol)
	# a fully shadowed light leaves the quadrature's rounding, not light
	return np.where(np.abs(total) <= 10.0 * rtol * np.abs(unshadowed), 0.0, np.atleast_1d(total))


def direct_lighting(x, n, wo, albedo, f0, roughness, lights, occluders=(), lobes=(True, True), planes=(), rtol=1e-10):
	"""Sum over lights (vertices [k, 3], radiance [3]) of L_e times the integral of f(w) (n . w) over the visible part of the light above x's
	tangent plane: the outgoing radiance the shading pass estimates, in float64. lobes: (diffuse, specular) of the BRDF; planes, occluders: see
	light_integral. Returns [3]."""
	n = np.asarray(n, dtype=np.float64)
	def g(w):
		diffuse, specular = brdf(w, wo, n, albedo, f0, roughness)
		f = (diffuse if lobes[0] else 0.0) + (specular if lobes[1] else 0.0)
		return f * np.maximum(w @ n, 0.0)[:, None]
	total = np.zeros(3)
	for poly, radiance in lights:
		total += np.asarray(radiance, dtype=np.float64) * light_integral(x, n, poly, g, occluders, planes, rtol)
	return total
