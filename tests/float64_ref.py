"""Plain float64 references for the two primitives every frame rests on: projected-solid-angle (PSA) sampling of a horizon-clipped polygon
(vkr_psa.cuh) and the any-hit shadow query (vkr_trace.cuh). numpy only; nothing here shares code or operation order with the oracle or the kernels.

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


def lambert_psa(poly):
	"""Projected solid angle of a spherical polygon in the upper hemisphere (Lambert: half the z-weighted sum of the edges' arc lengths). Edges of
	length zero (a clip crossing that coincides with a vertex) contribute nothing."""
	total = 0.0
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
		total += math.atan2(s, a[0] * b[0] + a[1] * b[1] + a[2] * b[2]) * cz / s
	return abs(0.5 * total)


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
