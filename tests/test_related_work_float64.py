"""The related-work sampling techniques 1..10 (csrc/vkr_related_work.cuh) against plain float64 references (tests/float64_ref.py), on the CPU: the oracle
(oracle.related_work_batch) and the device code compiled for the CPU (the same call on tests/build/libdevice_on_host.so) go through the same checks.
tests/test_gpu_zzzzzzzzzz_related_work_float64.py feeds the same cases to the GPU's probe (vkr_sample_related_work_batch) and reuses these checks.

The device code equals the oracle bit for bit (tests/test_device_on_host.py) and the oracle equals the reference shader (the "_q<technique>" fixtures), but
two restatements of the same GLSL can be wrong together. These checks know nothing of the GLSL:
  A. culling: the clipping techniques (5, 7, 9, 10) cull a light exactly when nothing of it is left above the horizon; the others never cull.
  B. containment: every direction is a finite unit vector inside the cone over the technique's support (light polygon, Urena's rectangle or the
     polygon clipped at the horizon). Where a technique's own fp32 recipe fails, the case is recorded as an exception with the reference's lines
     that fail the same way (LATTICE_END_EXCEPTIONS, recorded_failures).
  C. pointwise densities: 1 / solid angle (2, 3, 4, 5), Turk's area density from the direction's hit point on the light's plane (1), cosine over the
     projected solid angle (10), and the GGX density factor.
  D. quadrature identities on a K x K midpoint grid: mean(g(w) / p(w)) equals the float64 integral of g over the support, for g = 1 and g = w where
     p times the solid angle stays bounded away from 0, for g = max(cos, 0) everywhere, and for half-space indicators (also times the cosine). These
     hold for the pushforward of the sampler as a whole: a wrong sector, a wrong fan triangle or a warp that reports another density fails them.
  E. Jacobian: |dw/du.x x dw/du.y| p = 1 from central differences of the fp32 outputs, the pointwise check of Hart's densities (6..9).
  F. sector boundaries: at u.x exactly on a boundary of Turk's area fan the sample continues the sector below; the other techniques are continuous
     there. Hart's warps return the polygon's vertices 0, 1 and the last one at the corners of the unit square, with densities in the ratio of their
     cosines (the cosine fit that defines the warps).
"""
import math

import numpy as np
import pytest

from oracle import binding as O
from tests import float64_ref as R
from tests.test_device_on_host import DATASETS, MIXED, TECHNIQUES, _lib, _light_blocks, _scenarios

K = 64                       # midpoint grid of the quadrature identities
JACOBIAN_STEP = 2.0 ** -8    # central differences of the Jacobian check
JACOBIAN_STRIDE = 4          # every 4th grid point in each direction carries a stencil
LATTICE = (np.array([0, 1, 65534, 65535], dtype=np.float32) / np.float32(65535.0)).astype(np.float32)
DATA_SETS = [(name, maxv) for maxv, name in sorted(DATASETS.items())] + [(name, maxv) for maxv, name in sorted(MIXED.items())]
CLIPPING = (5, 7, 9, 10)
HART = (6, 7, 8, 9)

# ---- tolerances and the recipes' own failures -------------------------------------------------------------------------------------------------
# Measured worst cases over all data sets, families and random numbers are in brackets; each tolerance leaves a margin of 2 to 10 over them.

# The techniques' own failures, all of them the reference shader's arithmetic: the oracle equals the reference's frames bit for bit
# (tests/golden/ref_shader.npz), and the lines below of /src/shaders/polygon_sampling_related_work.glsl (PSRW) and cubic_solver.glsl do the same.
# Each is allowed only on the inputs that trigger it, the other samples of the case go through every check that still applies, and
# test_related_work_samplers_meet_the_float64_references asserts that each one is still seen where EXPECTED_FAILURES says.
#  * Random numbers at the ends of the noise table's lattice (u16 = 0 or 65535, u = 0 or 1) -- the table does hand these out:
#    - 6, 7 (bilinear): linear_warp() (PSRW:360-361) returns 0 / 0 when u = 0 and the corner density is 0, i.e. a vertex below the horizon.
#      Its own comment (PSRW:358-359) names the case. Only NaN is allowed; finite lattice samples must lie in the light.
#    - 8, 9 (biquadratic): quadratic_warp() keeps roots[0] when neither of the other roots lies in [0, 1] (PSRW:468-471); at u = 1 that
#      root lies far outside, and so does the direction (45 degrees beside the light, u = (0, 1)); at u = 0 the same 0 / 0 as above.
#    - 10 (Arvo): NaN at some lattice corners of edge-on, hemisphere-filling and horizon-clipped lights, and a direction 10 degrees outside the
#      light at u = (1 - 1/65535, 0) on a light of mini_mixed.
#    For 8, 9 and 10 finite lattice samples must still be unit vectors.
LATTICE_END_EXCEPTIONS = (6, 7, 8, 9, 10)
LATTICE_END_OUTSIDE = (8, 9, 10)
# The recorded failures each data set shows (a NaN, a zero density or a flagged case); a fix of the recipe has to update this list
EXPECTED_FAILURES = {2: ["Urena's solid angle cancels"], 3: ["Arvo's triangle sampling cancels"],
	8: ["biquadratic warp with a zero row", "biquadratic warp of a speck", "biquadratic warp with a linear marginal"],
	9: ["biquadratic warp of a speck", "biquadratic warp with a linear marginal"],
	10: ["Arvo's edges of a speck", "Arvo's edge at the normal", "Arvo's samples on the horizon"]}


def recorded_failures(technique, case):
	"""{name: what it allows} of the technique's own failures on this case. Allowances: "nan" (samples may be non-finite), "length" (finite
	directions may have any length), "outside" (they may leave the support), "density" (the densities follow no float64 reference: checks C, D and E are skipped), "pushforward" (the
	samples do not follow the densities: D and E are skipped), "jacobian" (E is skipped)."""
	family = case["family"]; poly = case["polygon"]
	unit = poly / np.linalg.norm(poly, axis=1, keepdims=True)
	out = {}
	if technique == 2 and family in ("speck", "centred_speck", "grazing"):
		# Urena's solid angle is 2 pi subtracted from a sum of four arc cosines of dot products of edge normals (PSRW:152-162). For a small or
		# edge-on rectangle the difference cancels, and acos near -1 or 1 has lost half of its digits: the solid angle is off by more than 100 %,
		# and where it cancels to 0 the density is inf and every direction NaN (a NaN, pink, pixel in the shader).
		out["Urena's solid angle cancels"] = {"nan", "density"}
	if technique == 3 and family in ("speck", "centred_speck", "grazing"):
		# Arvo's spherical triangle sampling takes s as a ratio of differences (PSRW:283) and normalises differences of nearly parallel
		# directions (PSRW:286, 291): for a speck or an edge-on light these lose all their digits, and directions come back NaN or with a length
		# up to 54.
		out["Arvo's triangle sampling cancels"] = {"nan", "length", "outside", "density"}
	if technique == 8 and unit[0, 2] <= 0.0:
		# quadratic_warp() divides by the cubic's leading coefficient (cubic_solver.glsl:31), (d0 - 2 d1 + d2) / 3, which is exactly 0 when the
		# three densities it warps with are equal. With vertex 0 below the horizon (8 does not clip) the row of corner densities at u.y = 0 is
		# all 0, and so are those near it in fp32: a row of NaN samples; with no vertex above the horizon every density takes the uniform fallback
		# (PSRW:445-448) and every sample is NaN.
		out["biquadratic warp with a zero row"] = {"nan"}
	if technique in (8, 9) and R.solid_angle(poly) < 1e-6:
		# The same division for a light below 1e-6 sr, whose cosines are equal or nearly so in fp32: NaN samples, and directions that are not
		# unit vectors (|w| off by up to 0.05) or leave the speck.
		out["biquadratic warp of a speck"] = {"nan", "length", "outside"}
	if technique in (8, 9) and biquadratic_marginal_is_linear(unit):
		# The same division by a leading coefficient that is not 0 but tiny: when the marginal density in u.y is nearly linear (|c3 / c1| below
		# 1e-4 in float64; 1.1e-5 for a horizon-crossing quad of mini_city), the normalised cubic's coefficients reach 1e5 and solve_cubic()
		# returns u.y on a grid of 2^-9 (cubic_solver.glsl:31-72). The warp follows its density on average (checks D hold) but not pointwise:
		# |J p - 1| oscillates by 30 % along u.y.
		out["biquadratic warp with a linear marginal"] = {"jacobian"}
	if technique == 10 and R.clip_and_psa(poly)[0] < 1e-6:
		# prepare_edge_arvo() scales each edge's length coefficients by the cosecants of its vertex's elevation and of the angle between the edge
		# and the meridian (PSRW:574-581); for a light below 1e-6 sr these grow without bound: the projected solid angle is off by up to 20 %
		# (a speck of mini_v7) and directions leave a speck on the normal.
		out["Arvo's edges of a speck"] = {"density", "outside"}
	if technique == 10 and (1.0 - unit[:, 2] < 2.0 ** -21).any():
		# A vertex within a few ulps of the normal normalises to z = 1 in fp32, and prepare_edge_arvo() takes inversesqrt(0) (PSRW:577, 581): the
		# length coefficients, the projected solid angle and every sample are NaN. prepare() does not cull then (NaN <= 0 is false): with the
		# diffuse-only strategy the light contributes nothing, with GGX MIS a GGX sample that hits it makes a NaN (pink) pixel.
		out["Arvo's edge at the normal"] = {"nan"}
	if technique == 10 and (poly[:, 2] <= 0.0).any():
		# Arvo's projected solid angle sampling of a light that crosses the horizon puts part of its samples on the horizon (up to 22 % of the
		# grid for a triangle of mini_mixed): the Newton steps are clamped to the sector (PSRW:918) and at its ends the outer edge's elevation is
		# that of a vertex on the horizon, so z = sqrt(mix(inner_z^2, outer_z^2, u.y)) = 0 (PSRW:924-926) and the reported density z / PSA is 0.
		# The shader skips such samples (density > 0 fails), so the estimator loses that share of the light; B and C hold for every sample.
		out["Arvo's samples on the horizon"] = {"pushforward"}
	return out


def biquadratic_marginal_is_linear(unit):
	"""Whether the marginal density of Hart's biquadratic warp in u.y is nearly linear: its three control values are 3 d0, the sum of the middle
	row and the sum of the far row of target densities (max(0, cosine) at vertex 0, at the last vertices and at the points the sampler reaches
	halfway), evaluated in float64 as PSRW:417-448 defines them."""
	def middle(v0, far):
		s2 = min(float(v0 @ far), 1.0)
		if s2 >= 1.0:
			return max(0.0, float(v0[2]))
		s = 0.5 * s2 + 0.5
		return max(0.0, s * v0[2] + math.sqrt(max(0.0, 1.0 - s * s)) / math.sqrt(2.0 * (1.0 - s2 * s2)) * (far[2] - s2 * v0[2]))
	fan = [R.solid_angle(unit[[0, k, k + 1]]) for k in range(1, len(unit) - 1)]
	target = 0.5 * sum(fan); k = 1
	while target > fan[k - 1] and k < len(fan):
		target -= fan[k - 1]; k += 1
	a, b = unit[k], unit[k + 1]; lo, hi = 0.0, 1.0
	for _ in range(60):   # the point of the far edges at half the fan's solid angle
		m = 0.5 * (lo + hi); q = _unit((1.0 - m) * a + m * b)
		lo, hi = (m, hi) if R.solid_angle(np.stack([unit[0], a, q])) < target else (lo, m)
	halfway = _unit((1.0 - lo) * a + lo * b)
	v0, last = unit[0], unit[-1]
	y = (3.0 * max(0.0, v0[2]), middle(v0, v0) + middle(v0, halfway) + middle(v0, last), max(0.0, unit[1, 2]) + max(0.0, halfway[2]) + max(0.0, last[2]))
	c1, c3 = y[0], (y[0] - 2.0 * y[1] + y[2]) / 3.0
	return c1 > 0.0 and abs(c3) < 1e-4 * c1


# Unit length of the directions [1.4e-6; hemisphere-filling lights ("close"): 5.9e-4, solid angle sampling leaves its last step unnormalised]
UNIT_TOLERANCE = dict(close=2e-3)
UNIT_DEFAULT = 1e-5
# Containment: how far (sine of the angle to an edge plane) a direction may lie outside the support [4.7e-5 on an edge-on rectangle, else 3.6e-5]
CONTAINMENT_MARGIN = 2e-4
# |p / p64 - 1| of the pointwise densities and the GGX density factor. Lights in front of the point [8e-6] hold 1e-4, 2x tighter than the
# known-answer test of techniques 3 and 4; specks [6.1e-4, the fp32 unit vectors of a 1e-8 sr light], hemisphere-filling lights [3.2e-4],
# edge-on lights [3.2e-3] and the random points, which come near both [3.4e-3], get what the fp32 inputs allow.
DENSITY_TOLERANCE = dict(random=6e-3, front=1e-4, behind=1e-4, grazing=1e-2, speck=3e-3, close=5e-3, horizon=1e-4, below=1e-4, centred=1e-4, centred_speck=3e-3)
# Quadrature identities at K = 64, |mean - integral| over the integral (over the solid angle for g = w). The midpoint rule's error on a
# piecewise smooth pushforward [4.2e-3, hemisphere-filling lights]; Turk's warp has a square root at the fan vertex, which the midpoint rule
# integrates to O(K^-1.5) [9.3e-3]; Hart's warps clamp corner densities to 0 [2.6e-2 for g = 1 with p SA >= 0.25, 1.4e-2 for the cosine].
QUADRATURE_TOLERANCE = 1e-2
QUADRATURE_TOLERANCE_TURK = 3e-2
QUADRATURE_TOLERANCE_HART = 6e-2
# Arvo's projected solid angle sampling inverts its CDF with a cubic guess and three clamped Newton steps (PSRW:872-968); its samples follow the
# density it reports only up to the residual of that inversion [1.6e-2 for g = w on a triangle of mini_tri; g = cos holds by construction].
QUADRATURE_TOLERANCE_ARVO = 5e-2
BOUNDED = 0.25               # g = 1 and g = w where p times the solid angle stays above this on the grid
# Half-space indicators: the boundary cuts grid cells, O(1 / K) [1.6e-2]
HALF_SPACE_TOLERANCE = 3.0 / K
# Jacobian: a stencil is used when its forward and backward estimates agree to JACOBIAN_SMOOTHNESS; then |J p - 1| per point [0.33, a stencil
# across a kink of a biquadratic warp] and its median [1.2e-3; random and hemisphere-filling points 1.3e-2]. Edge-on lights and specks leave too
# few significant digits in the fp32 differences and are not held to it. Turk's square root makes most stencils near the fan vertex disagree
# [skipped over a data set: 15 %; the other techniques 2.5 %].
JACOBIAN_SMOOTHNESS = 0.1
JACOBIAN_TOLERANCE = 0.5
JACOBIAN_MEDIAN_TOLERANCE = dict(random=5e-2, close=5e-2)
JACOBIAN_MEDIAN_DEFAULT = 5e-3
# Arvo's clamped Newton steps hold the azimuth at a sector's end over a patch of u (J = 0 there) [per point 1.0, median 3.4e-2]: its median only.
JACOBIAN_MEDIAN_ARVO = 0.1
JACOBIAN_SKIP_LIMIT = {1: 0.3}
JACOBIAN_SKIP_DEFAULT = 0.08
# Turk on an exact fan boundary against the float below, over the square root of the solid angle [2.8e-4 for a 1e-8 sr speck]
EDGE_TOLERANCE = 2e-3
# Bilinear warps: corner densities against the corner cosines [6.7e-7]
HART_CORNER_TOLERANCE = 1e-4

# ---- cases ---------------------------------------------------------------------------------------------------------------------------------

def _light(block, maxv):
	"""World-space geometry of one light block (float64 of its floats): vertices, plane normal and offset, Urena's rectangle."""
	b = np.frombuffer(block, dtype=np.float32).astype(np.float64)
	count = int(np.frombuffer(block, dtype=np.int32)[20])
	vertices = b[40 + 4 * maxv: 40 + 8 * maxv].reshape(maxv, 4)[:count, :3]
	translation, r0, r1 = b[4:7], b[[24, 28, 32]], b[[25, 29, 33]]
	ex, ey = r0 * b[3], r1 * b[7]
	rectangle = np.stack([translation, translation + ex, translation + ex + ey, translation + ey])
	return dict(vertices=vertices, plane=b[16:20], rectangle=rectangle)


def _area(V):
	return 0.5 * float(np.linalg.norm(sum(np.cross(V[k] - V[0], V[k + 1] - V[0]) for k in range(1, len(V) - 1))))


def _frame(position, normal, rng):
	"""Rows x, y, z of world_to_shading_space (z = the normal) and its translation, as the 12 floats the samplers take."""
	n = np.asarray(normal, dtype=np.float64); n = n / np.linalg.norm(n)
	x = np.cross(n, rng.normal(size=3)); x /= np.linalg.norm(x)
	rows = np.stack([x, np.cross(n, x), n]).astype(np.float32)
	t = -(rows.astype(np.float64) @ np.asarray(position, dtype=np.float32).astype(np.float64))
	return np.concatenate([rows.reshape(9), t.astype(np.float32)])


def _unit(v):
	return v / np.linalg.norm(v)


def _shading_points(block, maxv, rng):
	"""[(family, position, frame)] around one light: one point per family (two random ones)."""
	light = _light(block, maxv)
	V = light["vertices"]; c = V.mean(0); nrm = light["plane"][:3]
	size = math.sqrt(_area(V))
	tangent = _unit(np.cross(nrm, rng.normal(size=3)))
	out = [("random", p, f) for p, f in _scenarios(block, rng, 2)]
	def toward(p, jitter):
		return _unit(_unit(c - p) + jitter * rng.normal(size=3))
	def add(family, p, normal):
		p = np.asarray(p, dtype=np.float32)
		out.append((family, p, _frame(p, normal, rng)))
	p = c + nrm * size * rng.uniform(0.5, 2.0) + tangent * size * rng.uniform(-0.5, 0.5)
	add("front", p, toward(p, 0.3))
	p = c - nrm * size * rng.uniform(0.5, 2.0) + tangent * size * rng.uniform(-0.5, 0.5)
	add("behind", p, toward(p, 0.3))
	p = c + tangent * size * rng.uniform(1.5, 3.0) + nrm * size * 1e-3
	add("grazing", p, _unit(_unit(c - p) + nrm))
	distance = size / math.sqrt(10.0 ** -rng.uniform(6.0, 8.0))
	p = c + _unit(nrm + 0.5 * tangent) * distance
	add("speck", p, toward(p, 0.3))
	p = c + nrm * size * 1e-2 + tangent * size * 0.1
	add("close", p, _unit(-nrm + 0.1 * rng.normal(size=3)))   # the light fills most of the hemisphere above the point
	p = c + _unit(nrm + 0.5 * tangent) * size * rng.uniform(0.8, 2.0)
	add("horizon", p, _unit(np.cross(c - p, rng.normal(size=3))))
	p = c + _unit(nrm - 0.5 * tangent) * size * rng.uniform(1.5, 3.0)
	normal = -_unit(c - p)
	assert ((V - p) @ normal).max() < 0.0
	add("below", p, normal)
	p = c + _unit(nrm + 0.3 * tangent) * size * rng.uniform(0.8, 2.0)
	add("centred", p, _unit(c - p))
	p = c + nrm * size / math.sqrt(10.0 ** -rng.uniform(6.0, 8.0))
	add("centred_speck", p, _unit(c - p))
	return out


_CASES = {}


def cases(dataset, maxv):
	"""[case] of one data set: every light of its constant block seen from every shading point of _shading_points. A case holds the inputs and the
	float64 geometry in shading space: the light polygon, Urena's rectangle and the light clipped at the horizon."""
	key = (dataset, maxv)
	if key not in _CASES:
		rng = np.random.default_rng(sum(map(ord, dataset)) * 10 + maxv)
		out = []
		for index, block in enumerate(_light_blocks(dataset, maxv)):
			light = _light(block, maxv)
			for family, position, frame in _shading_points(block, maxv, rng):
				rows = frame[:9].astype(np.float64).reshape(3, 3)
				p = position.astype(np.float64)
				polygon = (light["vertices"] - p) @ rows.T
				_, _, near, clipped = R.clip_and_psa(polygon)
				out.append(dict(dataset=dataset, maxv=maxv, light=index, family=family, block=block, position=position, frame=frame, rows=rows,
					plane=light["plane"], area=_area(light["vertices"]), polygon=polygon, rectangle=(light["rectangle"] - p) @ rows.T,
					clipped=np.array(clipped) if len(clipped) >= 3 else None, near_horizon=near))
		_CASES[key] = out
	return _CASES[key]


def support(case, technique):
	"""The set a technique samples, as a polygon in shading space seen from the shading point (None: empty or, for the baseline, none defined)."""
	if technique == 0:
		return None
	if technique == 2:
		return case["rectangle"]
	return case["clipped"] if technique in CLIPPING else case["polygon"]


def _turk_edges(block, maxv):
	"""u.x in float32 for which the fp32 target area (total area * u.x) lands exactly on a cumulative fan area of the block, one per inner boundary."""
	b = np.frombuffer(block, dtype=np.float32)
	count = int(np.frombuffer(block, dtype=np.int32)[20])
	fan = b[40 + 8 * maxv: 40 + 8 * maxv + 4 * (maxv - 2)].reshape(maxv - 2, 4)[:, 1]
	total = fan[maxv - 3]
	out = []
	for i in range(count - 3):
		u = np.float32(float(fan[i]) / float(total))
		for step in range(-8, 9):
			v = np.nextafter(u, np.float32(np.inf if step > 0 else -np.inf)) if step else u
			for _ in range(abs(step) - 1):
				v = np.nextafter(v, np.float32(np.inf if step > 0 else -np.inf))
			if np.float32(total * v) == fan[i]:
				out.append(v)
				break
	return out


def random_numbers(case, technique):
	"""(u [n, 2] float32, kind [n]): the K x K midpoint grid, the Jacobian stencils around every JACOBIAN_STRIDE-th grid point (kinds jx+, jx-, jy+, jy-,
	in that order per point), all pairs of the noise lattice's corners, u.x at the float64 cumulative fan fractions of the support and one float to
	either side, and for Turk u.x exactly on the fp32 boundaries of the light's area fan next to the float below it."""
	g = ((np.arange(K) + 0.5) / K).astype(np.float32)
	grid = np.stack(np.meshgrid(g, g, indexing="ij"), axis=-1).reshape(-1, 2)
	u = [grid]; kind = ["grid"] * len(grid)
	centres = grid.reshape(K, K, 2)[JACOBIAN_STRIDE // 2::JACOBIAN_STRIDE, JACOBIAN_STRIDE // 2::JACOBIAN_STRIDE].reshape(-1, 2).astype(np.float64)
	h = JACOBIAN_STEP
	stencil = np.stack([centres + [h, 0], centres - [h, 0], centres + [0, h], centres - [0, h]], axis=1).reshape(-1, 2).astype(np.float32)
	u.append(stencil); kind += ["jx+", "jx-", "jy+", "jy-"] * len(centres)
	lattice = np.stack(np.meshgrid(LATTICE, LATTICE, indexing="ij"), axis=-1).reshape(-1, 2)
	u.append(lattice); kind += ["lattice"] * len(lattice)
	poly = support(case, technique)
	if poly is not None:
		fan = np.cumsum([R.solid_angle(poly[[0, k, k + 1]]) for k in range(1, len(poly) - 1)])
		edges = np.float32(np.clip(fan[:-1] / fan[-1], 0.0, 1.0)) if fan[-1] > 0 else np.zeros(0, dtype=np.float32)
		xs = np.concatenate([edges, np.nextafter(edges, np.float32(0)), np.nextafter(edges, np.float32(1))])
		for y in (0.3, 0.7):
			u.append(np.stack([xs, np.full(len(xs), y, dtype=np.float32)], axis=1)); kind += ["fan"] * len(xs)
	if technique == 1:
		for x in _turk_edges(case["block"], case["maxv"]):
			for y in (0.3, 0.7):
				u.append(np.float32([[x, y], [np.nextafter(x, np.float32(0)), y]])); kind += ["edge", "edge-"]
	return np.concatenate(u).astype(np.float32), np.array(kind)


def run(technique, case, u, library=None):
	"""The oracle's samples (library None) or those of the device code on the CPU: None if culled, else (dirs, densities, GGX density factor)."""
	if library is None:
		return O.related_work_batch(technique, case["maxv"], case["block"], case["position"], case["frame"], u)
	return O.related_work_batch(technique, case["maxv"], case["block"], case["position"], case["frame"], u, symbol_library=library, symbol="vkr_device_on_host_related_work_batch")


def _note(stats, name, family, value):
	key = (name, family)
	if not np.isnan(value) and value > stats.get(key, -1.0):
		stats[key] = float(value)


def _half_spaces(poly):
	"""Normals of three planes through the centre direction of the polygon, 60 degrees apart."""
	P = np.asarray(poly, dtype=np.float64)
	m = _unit((P / np.linalg.norm(P, axis=1, keepdims=True)).sum(0))
	a = _unit(np.cross(m, [1.0, 0.0, 0.0] if abs(m[0]) < 0.9 else [0.0, 1.0, 0.0])); b = np.cross(m, a)
	return [math.cos(t) * a + math.sin(t) * b for t in (0.0, math.pi / 3.0, 2.0 * math.pi / 3.0)]


def _jacobian(W, kind):
	"""Central, forward and backward estimates of |dw/du.x x dw/du.y| at the stencil centres (in the order random_numbers made them), and their grid
	indices."""
	S = W[np.isin(kind, ["jx+", "jx-", "jy+", "jy-"])].reshape(-1, 4, 3)
	grid = W[kind == "grid"].reshape(K, K, 3)
	c = grid[JACOBIAN_STRIDE // 2::JACOBIAN_STRIDE, JACOBIAN_STRIDE // 2::JACOBIAN_STRIDE].reshape(-1, 3)
	h = JACOBIAN_STEP
	central = np.linalg.norm(np.cross((S[:, 0] - S[:, 1]) / (2 * h), (S[:, 2] - S[:, 3]) / (2 * h)), axis=1)
	forward = np.linalg.norm(np.cross((S[:, 0] - c) / h, (S[:, 2] - c) / h), axis=1)
	backward = np.linalg.norm(np.cross((c - S[:, 1]) / h, (c - S[:, 3]) / h), axis=1)
	return central, forward, backward


def check_case(technique, case, u, kind, out, stats):
	"""The float64 checks A..F of one (technique, case) whose samples `out` (None if culled, else dirs, densities, GGX factor) came from the oracle, the
	device code on the CPU or the GPU's probe. Records the worst errors in `stats` under (check, family)."""
	family = case["family"]; label = (TECHNIQUES[technique], case["dataset"], case["light"], family)
	poly = support(case, technique)
	# A. culling
	if technique in CLIPPING:
		if not case["near_horizon"]:
			assert (out is not None) == (poly is not None), (label, "culled" if out is None else "not culled")
	else:
		assert out is not None, (label, "culled")
	if out is None:
		return
	dirs, dens, ggx = out
	d = dirs.astype(np.float64); p = dens.astype(np.float64)
	finite = np.isfinite(d).all(axis=1) & np.isfinite(p)
	failures = recorded_failures(technique, case)
	allowed = set().union(*failures.values()) if failures else set()
	lattice = (kind == "lattice") & (technique in LATTICE_END_EXCEPTIONS)
	# B. finite unit vectors inside the support
	assert (finite | lattice).all() or "nan" in allowed, (label, "non-finite", u[~(finite | lattice)][:4])
	for name, what in failures.items():
		if (("nan" in what and not finite.all()) or ("pushforward" in what and (p[finite] == 0.0).any())
				or what & {"length", "outside", "density", "jacobian"}):
			stats[("seen", name)] = stats.get(("seen", name), 0) + 1
	stats[("non-finite", family)] = stats.get(("non-finite", family), 0) + int((~finite).sum())
	if not finite.any():
		return
	if "length" not in allowed:
		norm_error = np.abs(np.linalg.norm(d[finite], axis=1) - 1.0).max()
		_note(stats, "unit", family, norm_error)
		assert norm_error <= UNIT_TOLERANCE.get(family, UNIT_DEFAULT), (label, "unit length", norm_error)
	if technique == 0:
		return
	inside = finite & ~((kind == "lattice") & (technique in LATTICE_END_OUTSIDE)) & ("outside" not in allowed)
	W = d @ case["rows"].T   # shading space
	cos = W[:, 2]
	Wu = W[inside] / np.linalg.norm(W[inside], axis=1, keepdims=True)
	_note(stats, "outside", family, max(0.0, -float((Wu @ R._edge_normals(poly).T).min(initial=0.0))))
	where = R.in_polygon_cone(Wu, poly, CONTAINMENT_MARGIN)
	assert (where != 0).all(), (label, "outside the support", u[inside][where == 0][:4])
	if "density" in allowed:
		return
	sa = R.solid_angle(poly)
	psa = R.clip_and_psa(poly)[0]
	# C. pointwise densities and the GGX density factor
	tol = DENSITY_TOLERANCE[family]
	if technique in (2, 3, 4, 5):
		e = np.abs(p[finite] * sa - 1.0).max(); _note(stats, "density", family, e)
		assert e <= tol, (label, "density", e)
		e = abs(ggx * sa - 1.0); _note(stats, "ggx", family, e)
		assert e <= tol, (label, "GGX density factor", e)
	elif technique == 1:
		nrm, w = case["plane"][:3], case["plane"][3]
		dw = d / np.linalg.norm(d, axis=1, keepdims=True)
		facing = dw @ nrm
		t = -(nrm @ case["position"].astype(np.float64) + w) / facing
		ref = t * t / (np.abs(facing) * case["area"])
		e = np.abs(p / ref - 1.0).max(); _note(stats, "density", family, e)
		assert e <= tol, (label, "Turk density", e)
		assert ggx == 0.0
	elif technique == 10:
		e = (np.abs(p * psa - np.maximum(cos, 0.0))[finite] / np.maximum(cos[finite], 1e-3)).max(); _note(stats, "density", family, e)
		assert e <= tol, (label, "cosine / projected solid angle", e)
		e = abs(ggx * psa - 1.0); _note(stats, "ggx", family, e)
		assert e <= tol, (label, "GGX density factor", e)
	else:
		assert ggx == 0.0
	# F. sector boundaries, the bilinear warps' corners
	if technique == 1:
		a, b = d[kind == "edge"], d[kind == "edge-"]
		e = np.linalg.norm(a - b, axis=1).max() / math.sqrt(sa) if len(a) else 0.0; _note(stats, "edge", family, e)
		assert e <= EDGE_TOLERANCE, (label, "sample on a fan boundary leaves the sector below", e)
	if technique in (6, 7):
		corner = lambda x, y: np.nonzero((u[:, 0] == x) & (u[:, 1] == y))[0][0]
		c00, c01, c11 = corner(0, 0), corner(0, 1), corner(1, 1)
		if np.isfinite(p[[c00, c01, c11]]).all() and min(cos[c00], cos[c01], cos[c11]) > 0.05:
			for c in (c01, c11):
				e = abs(p[c] * cos[c00] / (p[c00] * cos[c]) - 1.0); _note(stats, "hart corners", family, e)
				assert e <= HART_CORNER_TOLERANCE, (label, "corner densities against the cosines", e)
	# D. quadrature identities on the midpoint grid (a row of NaN samples leaves no mean to compare). Turk's 1 / p of a light 0.01 of its size
	# away, cos A / d^2, peaks at the point's foot on the light over a width the 64 x 64 grid does not resolve [18 %]; its pointwise density
	# and Jacobian checks hold there.
	g = kind == "grid"
	if "pushforward" in allowed or not finite[g].all() or (technique == 1 and family == "close"):
		return
	Wg, pg, cg = W[g], p[g], np.maximum(cos[g], 0.0)
	inv = 1.0 / pg
	qtol = {1: QUADRATURE_TOLERANCE_TURK, 10: QUADRATURE_TOLERANCE_ARVO}.get(technique, QUADRATURE_TOLERANCE_HART if technique in HART else QUADRATURE_TOLERANCE)
	scale = max(psa, 0.1 * sa)
	e = abs(np.mean(cg * inv) - psa) / scale; _note(stats, "quad cos", family, e)
	assert e <= qtol, (label, "mean(cos / p)", e)
	bounded = (pg * sa).min() >= BOUNDED
	if bounded:
		e = abs(np.mean(inv) / sa - 1.0); _note(stats, "quad 1", family, e)
		assert e <= qtol, (label, "mean(1 / p)", e)
		e = np.linalg.norm(np.mean(Wg * inv[:, None], axis=0) - R.vector_irradiance(poly)) / sa; _note(stats, "quad w", family, e)
		assert e <= qtol, (label, "mean(w / p)", e)
	if family not in ("speck", "centred_speck"):   # the fp32 directions of a speck do not resolve a plane through it
		for m in _half_spaces(poly):
			inside = (Wg @ m) > 0.0
			region = R._clip_halfspace([tuple(v) for v in poly], tuple(m))
			e = abs(np.mean(inside * cg * inv) - (R.clip_and_psa(region)[0] if len(region) >= 3 else 0.0)) / scale; _note(stats, "half-space cos", family, e)
			assert e <= HALF_SPACE_TOLERANCE, (label, "mean(indicator cos / p)", e)
			if bounded:
				e = abs(np.mean(inside * inv) - (R.solid_angle(region) if len(region) >= 3 else 0.0)) / sa; _note(stats, "half-space", family, e)
				assert e <= HALF_SPACE_TOLERANCE, (label, "mean(indicator / p)", e)
	# E. Jacobian
	if family not in ("speck", "centred_speck", "grazing") and "jacobian" not in allowed and finite[np.isin(kind, ["jx+", "jx-", "jy+", "jy-"])].all():
		central, forward, backward = _jacobian(W, kind)
		pc = p[g].reshape(K, K)[JACOBIAN_STRIDE // 2::JACOBIAN_STRIDE, JACOBIAN_STRIDE // 2::JACOBIAN_STRIDE].reshape(-1)
		smooth = np.abs(forward - backward) <= JACOBIAN_SMOOTHNESS * central
		stats[("stencils", "all")] = stats.get(("stencils", "all"), 0) + len(smooth)
		stats[("stencils", "skipped")] = stats.get(("stencils", "skipped"), 0) + int((~smooth).sum())
		e = np.abs(central[smooth] * pc[smooth] - 1.0)
		if len(e):
			_note(stats, "jacobian", family, e.max()); _note(stats, "jacobian median", family, np.median(e))
			if technique == 10:
				assert np.median(e) <= JACOBIAN_MEDIAN_ARVO, (label, "Jacobian median", np.median(e))
			else:
				assert e.max() <= JACOBIAN_TOLERANCE, (label, "Jacobian", e.max())
				assert np.median(e) <= JACOBIAN_MEDIAN_TOLERANCE.get(family, JACOBIAN_MEDIAN_DEFAULT), (label, "Jacobian median", np.median(e))


def check_totals(technique, stats):
	"""The fraction of Jacobian stencils skipped over all cases of a test."""
	if stats.get(("stencils", "all")):
		skipped = stats[("stencils", "skipped")] / stats[("stencils", "all")]
		assert skipped <= JACOBIAN_SKIP_LIMIT.get(technique, JACOBIAN_SKIP_DEFAULT), ("Jacobian stencils skipped", skipped)


def report(title, stats):
	"""Prints the worst error of each check over each scenario family, and the counts."""
	print(title)
	for name in sorted({k[0] for k in stats}):
		print("  %-16s %s" % (name, "  ".join(("%s %d" if isinstance(v, int) else "%s %.2e") % (f, v) for (n, f), v in sorted(stats.items()) if n == name)))


@pytest.mark.parametrize("technique", sorted(TECHNIQUES))
@pytest.mark.parametrize("dataset,maxv", DATA_SETS)
def test_related_work_samplers_meet_the_float64_references(technique, dataset, maxv):
	"""The oracle and the device code on the CPU through checks A..F on every case of a data set."""
	lib = _lib()
	stats = {}; lit = 0
	for case in cases(dataset, maxv):
		u, kind = random_numbers(case, technique)
		for library in (None, lib):
			out = run(technique, case, u, library)
			check_case(technique, case, u, kind, out, stats)
		lit += out is not None
	report("technique %d (%s), %s (V = %d): %d of %d cases lit" % (technique, TECHNIQUES[technique], dataset, maxv, lit, len(cases(dataset, maxv))), stats)
	check_totals(technique, stats)
	for name in EXPECTED_FAILURES.get(technique, ()):
		assert stats.get(("seen", name), 0) > 0, ("the recorded failure no longer occurs", name)
	assert lit > 0
