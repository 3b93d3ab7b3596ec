"""The polygon sampler and the shadow predicate against plain float64 references (tests/float64_ref.py), on the CPU: the oracle's sampler
(oracle.psa_sample_batch), the oracle's any-hit query (oracle.trace_any, brute force and its own BVH) and the device's traversal compiled for the
CPU (vkr_device_on_host_trace_any over the node pairs of each builder). tests/test_gpu_zzzzzy_float64_probes.py feeds the same polygons, random
numbers and rays to the GPU's probes.

The polygons cover what a shading point sees of a light: horizon-crossing polygons (also with vertices exactly at z = 0), polygons over the
zenith, slivers, distant specks (PSA about 1e-8), nearly hemisphere-filling polygons and polygons entirely below the horizon. The random numbers are
i.i.d. uniforms, the corners of the 16-bit lattice the noise table feeds the sampler (u16 / 65535: 0, 1/65535, 1 - 1/65535 and 1.0), and u.x exactly at
the cumulative sector fractions.
"""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import binding as oracle
from tests import float64_ref as R

VERTEX_COUNTS = [3, 4, 5, 6, 7]
SHADOW_SCENES = ["cornell", "mini_city", "mini_room", "roughness_planes"]

# Largest error of the biased variant's arctangent (fast_positive_atan, polygon_sampling.glsl:83-97) over all float32 tangents, measured in float64
# by test_fast_positive_atan_error_envelope: 1.17e-5 rad. Each sector's PSA is half a difference of two rsqrt(det) * atan terms with rsqrt(det) <= 1,
# so the biased PSA is off by at most the vertex count times this.
FAST_ATAN_MAX_ERROR = 1.2e-5


def psa_tolerance(ref, vertex_count, biased):
	"""|PSA - float64 PSA|. Unbiased: 2e-5 relative above 1e-3 and 2e-7 absolute, the bound of the sector-area arithmetic in fp32 that
	test_oracle_kats.py holds polygons above the horizon to; clipped, sliver and speck polygons meet it too. Biased: plus the arctangent's error
	once per sector (FAST_ATAN_MAX_ERROR)."""
	return 2e-5 * max(ref, 1e-3) + 2e-7 + (vertex_count * FAST_ATAN_MAX_ERROR if biased else 0.0)


# ---- polygons ----------------------------------------------------------------------------------------------------------------------------

def _clockwise(pts):
	"""The sampler wants the vertices clockwise as seen from the origin: the polygon's normal (sum of edge cross products) points away from it."""
	c = pts.mean(axis=0)
	w = sum(np.cross(pts[i] - c, pts[(i + 1) % len(pts)] - c) for i in range(len(pts)))
	return pts if w.dot(c) > 0 else pts[::-1].copy()


def _ring(rng, n, centre, radius, tilt=0.6, squash=1.0):
	"""n vertices on an ellipse (radius, radius * squash) around centre in a random plane facing the origin roughly."""
	centre = np.asarray(centre, dtype=np.float64)
	z = centre / np.linalg.norm(centre)
	t = rng.normal(size=3); t -= t.dot(z) * z; t /= np.linalg.norm(t)
	b = np.cross(z, t)
	nrm = z + tilt * (rng.uniform(-1, 1) * t + rng.uniform(-1, 1) * b); nrm /= np.linalg.norm(nrm)
	u = np.cross(nrm, t); u /= np.linalg.norm(u); v = np.cross(nrm, u)
	angles = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 2 * np.pi) + rng.uniform(-0.25, 0.25, n) * (2 * np.pi / n)
	return centre[None] + radius * (np.cos(angles)[:, None] * u[None] + squash * np.sin(angles)[:, None] * v[None])


def _on_horizon(rng, n):
	"""A planar polygon through a horizontal line: vertices 0 and k lie exactly at z = 0, the others above it, or (half of the time) some below."""
	azimuth = rng.uniform(0, 2 * np.pi)
	p = np.array([math.cos(azimuth), math.sin(azimuth), 0.0]) * rng.uniform(1.0, 3.0)
	u = np.array([-math.sin(azimuth), math.cos(azimuth), 0.0])
	w = np.array([0.0, 0.0, 1.0]) * rng.uniform(0.5, 1.5) + p / np.linalg.norm(p) * rng.uniform(-0.5, 0.8)
	below = rng.uniform() < 0.5
	theta = np.sort(np.concatenate([[0.0, np.pi], rng.uniform(0.2, 2 * np.pi - 0.2 if below else np.pi - 0.2, n - 2)]))
	s = np.cos(theta); t = np.sin(theta); t[(theta == 0.0) | (theta == np.pi)] = 0.0
	r = rng.uniform(0.3, 1.0)
	pts = p[None] + r * s[:, None] * u[None] + r * t[:, None] * w[None]
	pts[t == 0.0, 2] = 0.0
	return pts


def polygon_families(seed=2024):
	"""[(family, vertex count, float32 vertices)], clockwise as seen from the origin."""
	rng = np.random.default_rng(seed)
	out = []
	def add(family, n, pts):
		out.append((family, n, _clockwise(np.asarray(pts, dtype=np.float32))))
	for n in VERTEX_COUNTS:
		for _ in range(3):
			c = rng.normal(size=3); c[2] = abs(c[2]) + 0.3; c *= rng.uniform(1.0, 4.0) / np.linalg.norm(c)
			add("above", n, _ring(rng, n, c, rng.uniform(0.2, 0.9)))
		k = 0
		while k < 4:
			c = rng.normal(size=3); c[2] = rng.uniform(-0.3, 0.3); c *= rng.uniform(1.0, 3.0) / np.linalg.norm(c)
			pts = _ring(rng, n, c, rng.uniform(0.4, 1.5))
			if pts[:, 2].min() < -1e-3 and pts[:, 2].max() > 1e-3:
				add("horizon", n, pts); k += 1
		for _ in range(2):
			add("on_horizon", n, _on_horizon(rng, n))
		for _ in range(2):
			add("zenith", n, _ring(rng, n, [rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.8, 2.0)], rng.uniform(0.8, 1.5), tilt=0.3))
		add("zenith_horizon", n, _ring(rng, n, [rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 0.5], 3.0, tilt=0.8))
		add("hemisphere", n, _ring(rng, n, [0.0, 0.0, rng.uniform(0.05, 0.2)], 40.0, tilt=0.0))
		for _ in range(2):
			c = rng.normal(size=3); c[2] = abs(c[2]) + 0.2; c *= rng.uniform(1.0, 3.0) / np.linalg.norm(c)
			add("sliver", n, _ring(rng, n, c, rng.uniform(0.5, 1.0), squash=1e-3))
		c = rng.normal(size=3); c[2] = abs(c[2]) + 0.3; c *= rng.uniform(8.0, 12.0) / np.linalg.norm(c)
		add("speck", n, _ring(rng, n, c, 1e-3))
		c = rng.normal(size=3); c[2] = -abs(c[2]) - 0.5; c *= 2.0 / np.linalg.norm(c)
		add("below", n, _ring(rng, n, c, 0.4))
	return out


LATTICE = (np.array([0, 1, 65534, 65535], dtype=np.float32) / np.float32(65535.0)).astype(np.float32)


def random_numbers(seed, info, iid=256):
	"""(u [n, 2] float32, kind [n]): i.i.d. uniforms, all pairs of lattice corners, and u.x exactly at (and one float beside) the cumulative sector
	fractions of the polygon the oracle prepared."""
	rng = np.random.default_rng(seed)
	u = [rng.uniform(0, 1, (iid, 2)).astype(np.float32)]; kind = ["iid"] * iid
	grid = np.stack(np.meshgrid(LATTICE, LATTICE, indexing="ij"), axis=-1).reshape(-1, 2)
	u.append(grid); kind += ["lattice"] * len(grid)
	vc, psa = info["vc"], info["psa"]
	if vc and psa > 0:
		cum = np.cumsum(info["sectors"][:vc].astype(np.float64))[:-1] / psa
		edges = np.float32(np.clip(cum, 0, 1))
		xs = np.concatenate([edges, np.nextafter(edges, np.float32(0)), np.nextafter(edges, np.float32(1))]).astype(np.float32)
		u.append(np.stack([xs, rng.uniform(0, 1, len(xs)).astype(np.float32)], axis=1)); kind += ["sector"] * len(xs)
	return np.concatenate(u).astype(np.float32), np.array(kind)


def sampling_case(family, n, pts, biased, index):
	"""Inputs and the oracle's outputs of one (polygon, variant): (u, kind, dirs, info)."""
	_, _, info = oracle.psa_sample_batch(pts, n + 1, np.zeros((1, 2), dtype=np.float32), biased=biased)
	u, kind = random_numbers(1000 + index, info)
	dirs, _, info = oracle.psa_sample_batch(pts, n + 1, u, biased=biased)
	return u, kind, dirs, info


def check_sampling_against_float64(family, n, pts, biased, u, kind, dirs, info, stats):
	"""The float64 checks of one (polygon, variant) whose samples `dirs` and `info` came from the oracle or from the GPU. Collects the largest
	relative PSA error and the worst backward error into `stats`."""
	psa_ref, vc_ref, ill, clipped = R.clip_and_psa(pts.astype(np.float64))
	label = (family, n, biased, pts.tolist())
	assert abs(info["psa"] - psa_ref) <= psa_tolerance(psa_ref, n, biased), (label, info["psa"], psa_ref)
	if psa_ref > 0:
		stats["psa_rel"] = max(stats.get("psa_rel", 0.0), abs(info["psa"] - psa_ref) / psa_ref)
	if not ill:
		assert info["vc"] == vc_ref, (label, info["vc"], vc_ref)
	if info["vc"] == 0:
		assert info["psa"] == 0.0 and not info["sectors"].any() and not dirs.any()
		return
	assert vc_ref >= 3
	assert abs(float(np.sum(info["sectors"].astype(np.float64))) - info["psa"]) <= 1e-6 * max(info["psa"], 1e-3)
	assert info["central"] == (R.in_polygon_cone(np.array([[0.0, 0.0, 1.0]]), pts, 0.0)[0] == 1) or R.in_polygon_cone(np.array([[0.0, 0.0, 1.0]]), pts, 1e-6)[0] == -1
	d = dirs.astype(np.float64)
	finite = np.isfinite(d).all(axis=1)
	# Recorded finding: the biased variant returns NaN for u.x = 1.0 on a horizon-clipped sliver (V = 3, clipped to 4 vertices, PSA 1.2e-4; the
	# polygon is POLYGONS[13]). The oracle computes the reference shader's arithmetic bit for bit, so this is the reference's behaviour; the noise
	# table does hand the sampler u = 1.0 (u16 = 65535). Only that case may be non-finite.
	assert finite[u[:, 0] != 1.0].all() and (finite | (biased and family == "sliver")).all(), (label, u[~finite])
	stats["nan"] = stats.get("nan", 0) + int((~finite).sum())
	d = d[finite]; u = u[finite]; kind = kind[finite]
	assert (d[:, 2] >= 0.0).all()
	assert np.abs(np.linalg.norm(d, axis=1) - 1.0).max() < 1e-6, label
	where = R.in_polygon_cone(d, pts, CONTAINMENT_MARGIN[family])
	assert (where != 0).all(), (label, u[where == 0], d[where == 0])
	# the inverse CDF: the sample's position in the sampler's sweep, as a fraction of the float64 PSA, is u.x
	if psa_ref < 1e-6 or family == "sliver":
		return   # the fraction's float64 sub-region areas are themselves ill-conditioned for specks and slivers; their PSA checks above stand
	first = (tuple(float(c) for c in _clipped_vertex(pts, n, 0)), tuple(float(c) for c in _clipped_vertex(pts, n, 1)))
	# the swept part and the whole are each off by the PSA tolerance. The biased variant stops at the initial guess (no refinement steps), so its
	# samples follow the PSA only to its envelope, measured 2.6e-2 (a horizon-crossing quad).
	tol = BIASED_BACKWARD_ENVELOPE if biased else BACKWARD_TOLERANCE + 2.0 * psa_tolerance(psa_ref, n, False) / psa_ref
	sel = np.nonzero(kind == "iid")[0][:48]
	for i in sel:
		f = R.sample_cdf_position(pts.astype(np.float64), first, info["central"], d[i])
		stats["backward"] = max(stats.get("backward", 0.0), abs(f - float(u[i, 0])))
		assert abs(f - float(u[i, 0])) <= tol, (label, u[i], f)


def _clipped_vertex(pts, n, k):
	vc, v = oracle.clip(n, pts, n + 1)
	return v[k].astype(np.float64)


# Containment: how far (sine of the angle to an edge plane) a sample may lie outside the polygon, per family. Samples sit on the boundary when u.y = 0
# (inner edge) or u.x is 0 or 1 (first or last sector), and the recipe skips the refinement for |u.x - 0.5| > 0.5 - 1e-5, so at the lattice ends the
# initial guess stands. These are the recipe's own errors, not the port's: the oracle computes the reference shader's arithmetic bit for bit (its
# frames equal the reference's, tests/golden/ref_shader.npz). Measured worst cases over all variants and random-number kinds, about half of each:
#   above 5.5e-5 (u = (1/65535, 1 - 1/65535), no refinement), zenith 6e-6, hemisphere 2.2e-5, zenith_horizon 5.2e-5,
#   on_horizon 2.4e-4 (u = (0, 0): the corner on the horizon), horizon 3.6e-3 (u.x = 1 - 1/65535, u.y = 0; i.i.d. u: 5.5e-4),
#   sliver 5.6e-3 (u.x = 1 - 1/65535; i.i.d. u: inside), speck 2.3e-2 (a speck 2e-4 wide: its fp32 ellipses have no significant digits left).
CONTAINMENT_MARGIN = dict(above=1e-4, zenith=1e-5, hemisphere=5e-5, zenith_horizon=1e-4, on_horizon=5e-4, horizon=8e-3, sliver=1e-2, speck=5e-2, below=0.0)
# The inverse-CDF check: two refinement steps leave a backward error around 1e-5 (test_oracle_kats.py); 1e-4 leaves room for the fp32 sector areas.
BACKWARD_TOLERANCE = 1e-4
BIASED_BACKWARD_ENVELOPE = 5e-2


POLYGONS = polygon_families()


@pytest.mark.parametrize("biased", [False, True])
@pytest.mark.parametrize("n", VERTEX_COUNTS)
def test_oracle_sampler_meets_the_float64_references(n, biased):
	stats = {}
	for index, (family, nv, pts) in enumerate(POLYGONS):
		if nv != n:
			continue
		u, kind, dirs, info = sampling_case(family, n, pts, biased, index)
		check_sampling_against_float64(family, n, pts, biased, u, kind, dirs, info, stats)
	print("V=%d biased=%d: largest relative PSA error %.2e, worst backward error %.2e, %d NaN samples" % (n, biased, stats.get("psa_rel", 0), stats.get("backward", 0), stats.get("nan", 0)))
	assert (stats.get("nan", 0) > 0) == ((n, biased) == (3, True))


def test_fast_positive_atan_error_envelope():
	"""FAST_ATAN_MAX_ERROR: the biased variant's arctangent against float64 over a dense sweep of float32 tangents of both signs (all magnitudes from
	1e-6 to 1e6, and around 1, where the reflection switches)."""
	mags = np.concatenate([np.geomspace(1e-6, 1e6, 400001), np.linspace(0.9, 1.1, 200001)]).astype(np.float32)
	t = np.concatenate([mags, -mags, np.float32([0.0, 1.0, -1.0])])
	ref = np.arctan(t.astype(np.float64)); ref = np.where(t < 0, ref + np.pi, ref)
	err = np.abs(oracle.elementary("fast_positive_atan", t).astype(np.float64) - ref).max()
	print("fast_positive_atan: largest error %.3e rad" % err)
	assert 1.0e-5 < err <= FAST_ATAN_MAX_ERROR


def test_the_references_on_known_answers():
	# a square over the zenith, z = 1, half side a: PSA = 4 a / sqrt(1 + a^2) * atan(a / sqrt(1 + a^2)) (Lambert, four equal edges)
	a = 0.7
	sq = np.array([[-a, -a, 1.0], [a, -a, 1.0], [a, a, 1.0], [-a, a, 1.0]])
	psa, vc, ill, _ = R.clip_and_psa(sq)
	assert vc == 4 and not ill and abs(psa - 4 * a / math.sqrt(1 + a * a) * math.atan(a / math.sqrt(1 + a * a))) < 1e-13
	assert R.in_polygon_cone(np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [a, 0.0, 1.0]]) , sq, 1e-9).tolist() == [1, 0, -1]
	# a triangle cut by the horizon: in the plane x = 1, from (1, -1, -1), (1, 1, -1) to (1, 0, 1); above z = 0 the triangle (1, -1/2, 0), (1, 1/2, 0),
	# (1, 0, 1). Its PSA by hand: the horizon edge has z = 0 and contributes nothing; the two slanted edges from (1, +-1/2, 0) to (1, 0, 1) each
	# contribute half of angle * (a x b).z / |a x b|
	tri = np.array([[1.0, -1.0, -1.0], [1.0, 1.0, -1.0], [1.0, 0.0, 1.0]])
	p, q = np.array([1.0, 0.5, 0.0]), np.array([1.0, 0.0, 1.0])
	cr = np.cross(p / np.linalg.norm(p), q / np.linalg.norm(q))
	slanted = math.acos(p.dot(q) / np.linalg.norm(p) / np.linalg.norm(q)) * abs(cr[2]) / np.linalg.norm(cr)   # each slanted edge
	horizon = 2.0 * math.atan(0.5)                       # the edge on the horizon: its plane's normal is z, its arc counts in full
	psa, vc, ill, clipped = R.clip_and_psa(tri)
	assert vc == 3 and not ill and abs(psa - 0.5 * (horizon - 2.0 * slanted)) < 1e-13 and abs(psa - 0.10190813799333487) < 1e-12
	# the same through the half-space clip: the right half (y > 0) has half of it, and the wedge fractions are monotone
	assert abs(R.psa_of_region(tri, [(0.0, 1.0, 0.0)]) - 0.5 * psa) < 1e-13
	assert R.clip_and_psa(-tri)[1] == 4 and R.clip_and_psa(tri - np.array([0.0, 0.0, 2.0]))[:2] == (0.0, 0)
	# a ray through a triangle's centroid hits; beyond tmax, behind tmin, beside it or parallel to it, it misses -- all decided
	t3 = np.array([[0.0, 0.0, 5.0, 3.0, 0.0, 5.0, 0.0, 3.0, 5.0]], dtype=np.float32)
	rays = np.array([[1, 1, 0, 0, 0, 1, 1e-3, 10], [1, 1, 0, 0, 0, 1, 1e-3, 4.9], [1, 1, 0, 0, 0, 1, 5.1, 10], [4, 4, 0, 0, 0, 1, 1e-3, 10],
		[1, 1, 0, 1, 0, 0, 1e-3, 10], [1, 1, 0, 0, 0, 1, 1e-3, np.inf], [1, 1, 0, 0, 0, 1, 1e-3, np.nan], [1, 1, 0, 0, 0, 1, 7.0, 7.0]], dtype=np.float32)
	hit, decided = R.shadow_truth(t3, rays)
	assert decided.all() and hit.tolist() == [True, False, False, False, False, True, False, False]
	assert np.array_equal(oracle.trace_any(t3, rays)[1].astype(bool), hit)
	# through a vertex or along an edge the float64 predicate cannot decide
	edge_rays = np.array([[0, 0, 0, 0, 0, 1, 1e-3, 10], [1.5, 0, 0, 0, 0, 1, 1e-3, 10]], dtype=np.float32)
	assert not R.shadow_truth(t3, edge_rays)[1].any()


# ---- shadow rays -------------------------------------------------------------------------------------------------------------------------

SPECIAL_COMPONENTS = np.float32([0.0, -0.0, 1e-40, -1e-40, 1e-45, -1e-45, np.finfo(np.float32).tiny, -np.finfo(np.float32).tiny])


def light_polygons(constants, light_count):
	"""World-space vertices of the lights, read from the constant block (256-byte header, then one block per light; vertex count at word 20,
	world-space vertices as float4 at byte 160 + 16 maxv)."""
	stride = (len(constants) - 256) // light_count
	maxv = (stride - 128) // 48
	out = []
	for i in range(light_count):
		block = constants[256 + i * stride: 256 + (i + 1) * stride]
		count = int(np.frombuffer(block, dtype=np.uint32)[20])
		out.append(np.frombuffer(block, dtype=np.float32)[40 + 4 * maxv: 40 + 8 * maxv].reshape(maxv, 4)[:count, :3].astype(np.float64))
	return out


def _rays(o, d, tmin, tmax):
	n = len(o)
	return np.concatenate([o, d, np.broadcast_to(np.asarray(tmin, dtype=np.float64).reshape(-1, 1), (n, 1)), np.broadcast_to(np.asarray(tmax, dtype=np.float64).reshape(-1, 1), (n, 1))], axis=1).astype(np.float32)


def first_hit_distance(tris, rays, iterations=40):
	"""The fp32 distance the predicate accepts first on each ray (bisection over the float32 bit patterns of tmax with the oracle's brute force:
	the ray is occluded on (tmin, tmax) exactly when that distance is below tmax). Rays must hit and have tmin > 0."""
	lo = rays[:, 6].copy().view(np.int32).astype(np.int64); hi = rays[:, 7].copy().view(np.int32).astype(np.int64)
	for _ in range(iterations):
		if (hi - lo <= 1).all():
			break
		mid = (lo + hi) // 2
		probe = rays.copy(); probe[:, 7] = mid.astype(np.int32).view(np.float32)
		h = oracle.trace_any(tris, probe)[1].astype(bool)
		hi = np.where(h, mid, hi); lo = np.where(h, lo, mid)
	return (hi - 1).astype(np.int32).view(np.float32)   # the largest tmax that still misses


def shadow_ray_families(tris, seed, n=600, nodes=None, surface=None, lights=None, families=None):
	"""{family: rays [m, 8] float32}. surface: G-buffer positions of lit pixels, lights: world-space light polygons (family "light"); nodes: node
	pairs of a BVH (family "box_faces")."""
	rng = np.random.default_rng(seed)
	T = tris.reshape(-1, 3, 3).astype(np.float64)
	lo = tris.reshape(-1, 3).min(0).astype(np.float64); hi = tris.reshape(-1, 3).max(0).astype(np.float64)
	diag = float(np.linalg.norm(hi - lo))
	def targets(m):
		return np.einsum("nk,nkj->nj", rng.dirichlet([1, 1, 1], m), T[rng.integers(0, len(T), m)])
	def unit(v):
		return v / np.linalg.norm(v, axis=1, keepdims=True)
	out = {}
	want = lambda f: families is None or f in families
	if want("light") and surface is not None:
		o = surface[rng.integers(0, len(surface), n)].astype(np.float64)
		rays = []
		for k, poly in enumerate(lights):
			m = n // len(lights)
			w = rng.dirichlet(np.ones(len(poly)), m)
			centre = poly.mean(0)
			pts = centre + (w @ poly - centre) * rng.choice([1.0, 1.0, 1.08, 1.2], (m, 1))   # some points beyond the light's rim
			e = pts - o[k * m:(k + 1) * m]; dist = np.linalg.norm(e, axis=1)
			rays.append(_rays(o[k * m:(k + 1) * m], e / dist[:, None], 1e-3, dist))
		out["light"] = np.concatenate(rays)
	if want("random"):
		o = rng.uniform(lo, hi, (n, 3)); tg = T[rng.integers(0, len(T), n)].mean(1) + rng.normal(scale=0.05, size=(n, 3))
		d = tg - o; length = np.linalg.norm(d, axis=1)
		out["random"] = _rays(o, d / length[:, None], 1e-3, length * rng.uniform(0.3, 1.5, n))
	if want("unusual"):
		o = rng.uniform(lo, hi, (n, 3))
		d = unit(targets(n) - o)
		axes = np.eye(3)[rng.integers(0, 3, n // 4)] * rng.choice([-1.0, 1.0], (n // 4, 1))
		d[: n // 4] = axes
		d = d.astype(np.float32)
		for k in range(n // 4, n):
			for a in rng.choice(3, rng.integers(1, 3), replace=False):
				d[k, a] = SPECIAL_COMPONENTS[rng.integers(0, len(SPECIAL_COMPONENTS))]
		out["unusual"] = _rays(o, d, 1e-3, 2.0 * diag)
	if want("box_faces") and nodes is not None:
		k = rng.integers(0, len(nodes), n); child = rng.integers(0, 2, n)
		c = nodes[k[:, None], 6 * child[:, None] + np.arange(3)[None]]; h = nodes[k[:, None], 6 * child[:, None] + 3 + np.arange(3)[None]]
		ok = (h >= 0).all(1)
		c, h, child = c[ok], h[ok], child[ok]
		m = len(c); axis = rng.integers(0, 3, m); side = rng.choice(np.float32([-1.0, 1.0]), m)
		o = (c + h * rng.uniform(-1, 1, (m, 3)).astype(np.float32)).astype(np.float32)
		o[np.arange(m), axis] = (c[np.arange(m), axis] + side * h[np.arange(m), axis]).astype(np.float32)   # exactly on the face
		d = rng.normal(size=(m, 3)); d[np.arange(m), axis] = 0.0; d = unit(d)                           # along the face
		out["box_faces"] = _rays(o, d, 1e-3, 2.0 * diag)
	if want("corners"):
		m = n // 3
		ti = rng.integers(0, len(T), m); corner = rng.integers(0, 3, m)
		mid = ((tris.reshape(-1, 3, 3)[ti, corner] + tris.reshape(-1, 3, 3)[ti, (corner + 1) % 3]) * np.float32(0.5)).astype(np.float32)
		o = np.concatenate([T[ti, corner], mid.astype(np.float64)])
		d = unit(rng.normal(size=(2 * m, 3)))
		r1 = _rays(o, d, rng.choice([1e-3, -1e-3], 2 * m), diag)
		o2 = rng.uniform(lo, hi, (m, 3)); tg = np.where(rng.uniform(size=(m, 1)) < 0.5, T[ti, corner], mid.astype(np.float64))
		e = tg - o2; length = np.linalg.norm(e, axis=1)
		r2 = _rays(o2, e / length[:, None], 1e-3, length * 1.5)                                           # through shared vertices and edges
		out["corners"] = np.concatenate([r1, r2])
	if want("interval"):
		base = shadow_ray_families(tris, seed + 1, n=n, families=["random"])["random"]
		base[:, 7] = 2.0 * diag
		hits = base[oracle.trace_any(tris, base)[1].astype(bool)][: n // 3]
		t = first_hit_distance(tris, hits)
		at_tmax = hits.copy(); at_tmax[:, 7] = t                                                         # open interval: misses the first triangle
		past = hits.copy(); past[:, 7] = np.nextafter(t, np.float32(np.inf))
		at_tmin = hits.copy(); at_tmin[:, 6] = t; at_tmin[:, 7] = np.nextafter(t, np.float32(np.inf))    # nothing lies strictly between
		equal = hits.copy(); equal[:, 6] = equal[:, 7] = t
		reverse = hits.copy(); reverse[:, 6] = 1.5 * t; reverse[:, 7] = t
		infinite = hits.copy(); infinite[:, 7] = np.inf
		nan = hits.copy(); nan[:, 7] = np.nan
		negative = base[: n // 3].copy(); negative[:, 6] = -0.5 * diag
		out["interval"] = np.concatenate([at_tmax, past, at_tmin, equal, reverse, infinite, nan, negative])
	if want("long"):
		corners = np.array([[lo[0] if i & 1 else hi[0], lo[1] if i & 2 else hi[1], lo[2] if i & 4 else hi[2]] for i in range(8)])
		o = corners[rng.integers(0, 8, n)].astype(np.float32).astype(np.float64)
		tg = np.where(rng.uniform(size=(n, 1)) < 0.5, targets(n), rng.uniform(lo, hi, (n, 3)))
		e = tg - o; length = np.linalg.norm(e, axis=1)
		out["long"] = _rays(o, e / length[:, None], 1e-3, np.where(rng.uniform(size=n) < 0.5, length * 1.001, 2.0 * diag))
	return out


# Families whose rays meet an edge, a vertex or a plane only by accident, and the undecided fraction they must stay below. Exception: roughness_planes
# is flat (its bounding box is a few centimetres thick), so its random origins lie next to the planes and the segments graze them: 4.3 % measured.
# The long rays start at the corners of the bounding box, which lie on the walls of the closed scenes (cornell: 12 % undecided), so they are not
# counted among these; the fp32 equalities hold on all of them.
RANDOM_FAMILIES = ("light", "random")
UNDECIDED_LIMIT = 0.01
UNDECIDED_LIMIT_FLAT = 0.1


def check_shadow_answers(name, family, rays, got, brute, truth, decided, what):
	"""got (fp32 traversal) == brute (the oracle's brute force) on every ray, == truth on every decided ray. Returns the undecided fraction."""
	bad = np.nonzero(got.astype(bool) != brute.astype(bool))[0]
	assert len(bad) == 0, (what, name, family, len(bad), rays[bad[:5]].tolist())
	bad = np.nonzero(decided & (got.astype(bool) != truth))[0]
	assert len(bad) == 0, (what, name, family, "float64", len(bad), rays[bad[:5]].tolist())
	undecided = 1.0 - decided.mean()
	if family in RANDOM_FAMILIES:
		assert undecided < (UNDECIDED_LIMIT_FLAT if name == "roughness_planes" else UNDECIDED_LIMIT), (name, family, undecided)
	return undecided


def scene_inputs(name, width=96, height=64):
	"""(triangles, G-buffer surface points of lit pixels, light polygons) of a data set, all from the oracle's side."""
	from tests import harness as H
	from tests.ref_frames import host_constants
	info = H.dataset(name); oi = H.OracleInputs(info)
	lights = len(info["lights"])
	constants = host_constants(info, width, height, lights)
	gb = oi.gbuffer(width, height, constants, oi.visibility(width, height, constants))
	valid = np.argwhere(gb[1, :, :, 3] != 0)
	return oi.shadow_tris, np.ascontiguousarray(gb[0, valid[:, 0], valid[:, 1], :3], dtype=np.float32), light_polygons(constants, lights)


@pytest.mark.parametrize("name", SHADOW_SCENES)
def test_shadow_predicate_meets_the_float64_truth(name):
	"""The oracle's brute force and its own BVH, and the device's traversal compiled for the CPU over the node pairs of both host builders, against
	shadow_truth on every decided ray and against the oracle's brute force on every ray. The undecided fraction of the random families (shadow rays
	to the lights, random segments) stays below 1 % (RANDOM_FAMILIES). The other families aim at edges, vertices, box faces, walls and interval ends
	on purpose; float64 leaves many of their rays undecided, the fp32 equality holds on all."""
	from tests.test_device_on_host import _lib
	from tests.test_host_logic import _probe_bvh, BUILDERS
	from vulkan_renderer_b200 import api
	dev = _lib(); lib = api.load_library()
	tris, surface, lights = scene_inputs(name)
	built = {b: _probe_bvh(lib, tris, BUILDERS[b]) for b in sorted(BUILDERS)}
	families = shadow_ray_families(tris, 7, nodes=built["sah"][0], surface=surface, lights=lights)
	for family, rays in families.items():
		bvh, brute = oracle.trace_any(tris, rays)
		truth, decided = R.shadow_truth(tris, rays)
		check_shadow_answers(name, family, rays, bvh, brute, truth, decided, "oracle BVH")
		for builder, (nodes, slots, ids, depth) in built.items():
			out = np.zeros(len(rays), dtype=np.uint8)
			nodes = np.ascontiguousarray(nodes, dtype=np.float32); slots = np.ascontiguousarray(slots, dtype=np.float32)
			dev.vkr_device_on_host_trace_any(nodes.ctypes.data_as(C.c_void_p), slots.ctypes.data_as(C.c_void_p), C.c_uint32(len(slots)), C.c_uint32(len(rays)),
				rays.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), None)
			undecided = check_shadow_answers(name, family, rays, out, brute, truth, decided, "device traversal, " + builder)
		print("%s %-9s %5d rays, %5.1f %% occluded, undecided %.2f %%" % (name, family, len(rays), 100.0 * brute.mean(), 100.0 * undecided))
