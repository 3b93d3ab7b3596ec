"""The shading pass's per-pixel estimator against a float64 integral of the direct lighting (tests/float64_ref.direct_lighting), on the CPU through
the oracle. tests/test_gpu_zzzzzzzzzzzzz_estimator_float64.py runs the same cases through the GPU's shading pass.

The frames, the oracle and the device code agree bit for bit, and the polygon sampler and the shadow query each meet their own float64 references
(tests/test_float64_references.py), but a pair that agrees bit for bit can still be wrong together, and nothing else checks what the pieces add up
to: the BRDF, the LTC set-up and density, the GGX sampler and its density, the ray / light test of GGX MIS, the five MIS weightings with the
visibility estimate of the optimal heuristics, and the shadow rays. Their expectation must be the integral of L f cos V over the lights.

One piece is out of reach of any expectation: the value an occluded sample adds under the optimal heuristic, v W_own - v (sum of W p) / (sum of p)
per technique. Summed over the two techniques and integrated over the occluded directions it is v (W_d P_d + W_s P_s) - v (W_d P_d + W_s P_s) = 0
(P: each technique's probability of landing there), so a zero in its place changes the variance, not the mean. The frames' bit-for-bit
comparison with the oracle under the optimal heuristic with shadow rays (tests/test_gpu_parity.py) is what holds it.

Method. A synthetic G-buffer holds one shading point per aligned block of pixels (BLOCK x BLOCK, a multiple of the 16 x 8 tile). Every pixel of a
block reads other noise texels, so one frame gives BLOCK^2 x spp samples of one estimator; frames with animated noise give more. The mean over a
block and over K frames estimates the pixel's value, and its standard error comes from batch means: the spread of the K per-frame block means
(pixels of different frames can reuse noise texels, so the pixel variance would understate it). The frames read one fixed table, so their
expectation is the table's own quadrature of the integral, off by its variance over the texels; relative to the batch means' variance that
adds the ratio of the samples a case takes to the table's texels (each sample reads one texel: a diffuse and a specular pair, or a pair and
the next sample's pair). The table is sized so that this ratio stays at a few percent (NOISE). Each case must meet |mean - I| <= SIGMAS SE + EPS I
per colour channel, the mean of z^2 over a configuration must stay below the chi-square bound at p = 1e-6, and every case must resolve a bias
smaller than RESOLUTION of I (SIGMAS SE + EPS I <= RESOLUTION I), so that a bias of a percent cannot pass.

EPS. The estimators are exact only for uniform random numbers; the noise table hands out u16 / 65535, and the sampler works in fp32. The sizes
test_float64_references accepts for the sampler bound what that leaves: the projected solid angle to 2e-5 relative (psa_tolerance), which enters
each estimate as its reciprocal; the 16-bit lattice, a quadrature of 65536 points per dimension, off the integral by about 1 / 65536 = 1.5e-5 per
dimension of the random numbers (two per sample); the fp32 sums of spp samples and of the lights, a few 1e-7. Together less than 1e-4.

Random numbers. The estimators are unbiased for uniform random pairs (u.x, u.y). The white noise table of the reference's loader
(src/noise_table.c:73-75: the low 16 bits of wang_hash of consecutive integers, one per channel) is not uniform in two dimensions: its channel
pairs (R, G) and (B, A), which get_noise_2 hands out as one pair, correlate (-0.058) and fail a 64 x 64 chi-square test by a factor of 650
(test_the_white_noise_table_is_not_uniform_in_two_dimensions). Frames that use it converge a percent or more away from the integral where the
integrand is sharp (the diffuse-only estimator on a mirror-like surface: -1.5 %, behind a light: -6 %), in the reference as here. That is the
noise table's bias, not the estimator's, so these tests upload a table of independent uniform 16-bit texels (uniform_noise_table) through the
same loader entry point the blue-noise and Ahmed tables use.

Known bias. Sampling diffuse and specular separately (strategy 2) draws specular samples from the LTC distribution, which is zero where the
direction lies below the horizon of the cosine space (z_c = (M w).z <= 0) although the BRDF is not: the part of the specular integral over those
directions is never sampled. The reference does the same (the oracle equals its frames bit for bit), so this is the estimator's definition, not a
port error: the expectation asserted for strategy 2 is the integral minus that part, computed in float64 from the same LTC texels
(expected_bias_of_separate_sampling). The other strategies cover the whole light with the diffuse technique and are unbiased.
"""
import ctypes as C
import math
import os
import tempfile
import time

import numpy as np
import pytest
from scipy import stats as scipy_stats

from tests import float64_ref as R
from tests.test_float64_references import light_polygons
from vulkan_renderer_b200 import api, synth

BLOCK = 32            # pixels of a block edge on the CPU (the GPU file uses its own)
NOISE = (512, 512, 64)   # 16.8 M texels, 40 times the 0.4 M samples a case takes on the CPU
SIGMAS = 6.0
EPS = 1.0e-4
CHI_SQUARE_P = 1.0e-6
CAMERA = (0.3, -1.0, 1.5)          # below the light and the points behind it, above the others: every case faces it
VERTEX_COUNTS = [3, 4, 5, 6, 7]
LIGHT_SETS = ["v%d" % n for n in VERTEX_COUNTS] + ["mixed"]
# (strategy, heuristic, MIS visibility estimate): every heuristic the C-ABI accepts for each strategy
CONFIGURATIONS = [(api.STRATEGY_DIFFUSE_ONLY, 0, 0.5), (api.STRATEGY_DIFFUSE_GGX_MIS, api.MIS_BALANCE, 0.5), (api.STRATEGY_DIFFUSE_GGX_MIS, api.MIS_POWER, 0.5),
	(api.STRATEGY_DIFFUSE_SPECULAR_SEPARATELY, 0, 0.5)] + [(api.STRATEGY_DIFFUSE_SPECULAR_MIS, h, 0.5) for h in (api.MIS_BALANCE, api.MIS_POWER, api.MIS_WEIGHTED)] \
	+ [(api.STRATEGY_DIFFUSE_SPECULAR_MIS, h, v) for h in (api.MIS_OPTIMAL_CLAMPED, api.MIS_OPTIMAL) for v in (0.0, 0.5, 1.0)] + [(api.STRATEGY_DIFFUSE_SPECULAR_RANDOM, 0, 0.5)]


def config_name(config):
	strategy, heuristic, visibility = config
	return "s%d_h%d_v%.1f" % (strategy, heuristic, visibility)


# ---- the scene: lights, an occluder halfway between a row of points and the light, far ground -----------------------------------------------

LIGHT_CENTRE = np.array([0.0, 0.0, 2.0])
OCCLUDER = dict(x=(-0.45, 0.45), y=(-2.5, -1.7), z=1.0)      # the row of shading points at y = -4.2, z = 0 sees light 0 across it


def _regular(n, phase):
	return [(0.5 + 0.5 * math.cos(phase + 2.0 * math.pi * k / n), 0.5 + 0.5 * math.sin(phase + 2.0 * math.pi * k / n)) for k in range(n)]


def _lights(light_set):
	"""Light 0 faces down over LIGHT_CENTRE (plane space [0, 1]^2 scaled by 1.2, centred); the mixed set adds a pentagon and a heptagon beside it,
	tilted, so that triangles run in the heptagon kernel."""
	def at(centre, n, angles, scale, flux):
		return synth.make_light((centre[0] - 0.5 * scale, centre[1] + 0.5 * scale, centre[2]), angles, (scale, scale), flux, _regular(n, 0.3 * n))
	if light_set == "mixed":
		return [at(LIGHT_CENTRE, 3, (math.pi, 0.0, 0.0), 1.2, (8.0, 10.0, 12.0)), at((2.6, 0.5, 2.4), 5, (math.pi + 0.2, 0.1, 0.0), 0.8, (6.0, 5.0, 4.0)),
			at((-2.4, 1.0, 2.2), 7, (math.pi - 0.15, -0.15, 0.0), 1.0, (4.0, 5.0, 6.0))]
	return [at(LIGHT_CENTRE, int(light_set[1:]), (math.pi, 0.0, 0.0), 1.2, (8.0, 10.0, 12.0))]


def scene_mesh():
	"""The occluder (a quad, two triangles) and ground far below (8 x 8 quads), so that the shadow BVH has more than one leaf."""
	m = synth.Mesh()
	(x0, x1), (y0, y1), z = OCCLUDER["x"], OCCLUDER["y"], OCCLUDER["z"]
	m.add(synth._grid_quad([x0, y0, z], [x1 - x0, 0, 0], [0, y1 - y0, 0], 1, 1), 0)
	m.add(synth._grid_quad([-40.0, -40.0, -60.0], [80.0, 0, 0], [0, 80.0, 0], 8, 8), 0)
	return m.finish()


def dataset(directory=None):
	"""Writes the scene, its material textures, the synthetic LTC fits and one quicksave per light set. Returns {light set: info}."""
	directory = directory or os.path.join(os.environ.get("VKR_TEST_DATA", os.path.join(tempfile.gettempdir(), "vkr_b200_data")), "estimator_float64")
	os.makedirs(directory, exist_ok=True)
	materials = [dict(name="grey", base=(0.5, 0.5, 0.5), roughness=0.5, metal=0.0)]
	vks = os.path.join(directory, "scene.vks"); tex = os.path.join(directory, "textures"); ltc = os.path.join(directory, "ggx_ltc_fit")
	synth.write_vks(vks, scene_mesh(), materials)
	synth.write_material_textures(tex, materials)
	if not os.path.exists(os.path.join(ltc, "fit50.dat")):
		synth.write_ltc_fits(ltc)
	camera = synth.look_at_camera(CAMERA, (0.0, 0.0, 0.5))
	out = {}
	for light_set in LIGHT_SETS:
		save = os.path.join(directory, light_set + ".save")
		synth.write_quicksave(save, camera, _lights(light_set))
		out[light_set] = dict(vks=vks, textures=tex, save=save, ltc=ltc, materials=materials, material_params=synth.material_params(materials), lights=_lights(light_set))
	return out


# ---- the shading points ------------------------------------------------------------------------------------------------------------------

def _unit(v):
	v = np.asarray(v, dtype=np.float64)
	return v / np.linalg.norm(v)


def _toward(a, b, angle):
	"""The unit vector at `angle` from a, rotated towards b."""
	a = _unit(a); b = _unit(b)
	u = _unit(b - (b @ a) * a)
	return math.cos(angle) * a + math.sin(angle) * u


ROUGHNESS = [0.05, 0.2, 0.5, 1.0]
F0 = [0.0, 0.04, 1.0]
ALBEDO = [0.0, 0.5, 1.0]


def cases(polygon, seed=17):
	"""[(family, position, normal, albedo, f0, roughness)], fixed up front: light 0 over the zenith (all roughnesses x F0 at albedo 0.5, albedo 0 and
	1, coloured albedo and F0), crossing the horizon (also with a vertex within 1e-6 of the tangent plane), grazing views (theta_o 60 and 85 degrees),
	a small distant light, points behind the light's plane, and a row of points in front of, in the penumbra of and behind the occluder.
	polygon: light 0's world-space vertices (the horizon cases are built on them)."""
	rng = np.random.default_rng(seed)
	centre = polygon.mean(axis=0)
	out = []
	def add(family, x, n, albedo, f0, roughness):
		albedo = albedo if np.ndim(albedo) else (albedo,) * 3
		f0 = f0 if np.ndim(f0) else (f0,) * 3
		assert _unit(n) @ _unit(np.asarray(CAMERA) - x) >= math.cos(math.radians(85.01)), (family, x, n)
		out.append((family, np.asarray(x, dtype=np.float64), _unit(n), np.asarray(albedo, dtype=np.float64), np.asarray(f0, dtype=np.float64), float(roughness)))
	jitter = lambda: rng.normal(scale=0.03, size=3)
	x = np.array([1.2, 1.4, 0.2])
	for r in ROUGHNESS:
		for f in F0:
			add("zenith", x, centre - x + jitter(), 0.5, f, r)
	add("zenith", x, centre - x + jitter(), 0.0, 0.04, 0.5)
	add("zenith", x, centre - x + jitter(), 1.0, 0.04, 0.5)
	add("zenith", x, centre - x + jitter(), (1.0, 0.5, 0.0), (0.04, 1.0, 0.5), 0.2)
	x = np.array([-1.6, 1.0, 0.0])
	wo = _unit(np.asarray(CAMERA) - x)
	add("horizon", x, _toward(centre - x, wo, math.radians(80.0)), 0.5, 0.04, 0.2)
	add("horizon", x, _toward(centre - x, wo + (0.0, 0.0, 0.5), math.radians(72.0)), 0.0, 1.0, 1.0)
	# a vertex of light 0 on the tangent plane: the normal is perpendicular to it, tipped towards the light's centre
	e = _unit(polygon[1] - x)
	tipped = (centre - x) + 0.5 * np.linalg.norm(centre - x) * _unit(np.asarray(CAMERA) - x)
	add("horizon_vertex", x, _unit(tipped - (tipped @ e) * e), 0.5, 0.04, 0.5)
	x = np.array([1.5, -1.0, 0.0])
	wo = _unit(np.asarray(CAMERA) - x)
	add("grazing", x, _toward(wo, centre - x, math.radians(60.0)), 0.5, 1.0, 0.2)
	add("grazing", x, _toward(wo, centre - x, math.radians(85.0)), 1.0, 0.04, 0.5)
	x = centre + np.array([-7.0, 5.0, -2.0])
	add("distant", x, centre - x, 0.5, 1.0, 0.2)
	add("distant", x, centre - x + jitter(), 1.0, 0.04, 1.0)
	x = centre + np.array([0.25, -0.2, 0.7])
	add("behind", x, (0.1, 0.05, -1.0), 0.5, 0.04, 0.5)
	add("behind", x, (-0.2, 0.1, -1.0), 0.0, 1.0, 0.5)
	for dx in (-2.0, -1.1, -0.9, -0.75, 0.0):     # visible fraction of light 0: 1, 0.77, 0.51, 0.31, 0 (v4)
		x = np.array([dx, -4.2, 0.0])
		add("occluder", x, centre - x + jitter(), 0.5, 0.04, 0.5)
	return out


def uniform_noise_table(shape, seed=2718):
	"""[layers, height, width, 4] uint16 of independent uniform texels (numpy's PCG64), shape = (width, height, layers)."""
	width, height, layers = shape
	return np.random.default_rng(seed).integers(0, 65536, size=(layers, height, width, 4), dtype=np.uint16)


def synthetic_gbuffer(case_list, block, columns=8):
	"""[4, H, W, 4] float32: case k fills block (k // columns, k % columns); blocks without a case are invalid (valid = 0)."""
	rows = (len(case_list) + columns - 1) // columns
	gb = np.zeros((4, rows * block, columns * block, 4), dtype=np.float32)
	for k, (_, x, n, albedo, f0, roughness) in enumerate(case_list):
		r, c = divmod(k, columns)
		sl = (slice(r * block, (r + 1) * block), slice(c * block, (c + 1) * block))
		gb[0][sl] = [x[0], x[1], x[2], roughness]
		gb[1][sl] = [n[0], n[1], n[2], 1.0]
		gb[2][sl] = [albedo[0], albedo[1], albedo[2], 0.0]
		gb[3][sl] = [f0[0], f0[1], f0[2], 0.0]
	return gb


def block_means(frame, count, block, columns=8):
	"""Per-case means of one frame [count, 3], float64."""
	rows = frame.shape[0] // block
	m = np.asarray(frame[..., :3], dtype=np.float64).reshape(rows, block, columns, block, 3).mean(axis=(1, 3)).reshape(-1, 3)
	return m[:count]


# ---- float64 truth -----------------------------------------------------------------------------------------------------------------------

def lights_from_constants(constants, light_count):
	"""[(world-space vertices [k, 3], surface radiance [3])] as the kernel reads them (radiance at byte 48 of each light block)."""
	polys = light_polygons(constants, light_count)
	stride = (len(constants) - 256) // light_count
	radiance = [np.frombuffer(constants[256 + i * stride + 48: 256 + i * stride + 60], dtype=np.float32).astype(np.float64) for i in range(light_count)]
	return list(zip(polys, radiance))


def ltc_coefficients(constants, ltc0, ltc1, f0, roughness, n, wo):
	"""(d0 [4], d1 [2]) of get_ltc_coefficients in float64: the LTC texture coordinates from the constant block (6 floats at byte 224), a bilinear,
	clamp-to-edge fetch of the UNORM16 texels, the layer rounded to nearest."""
	c = np.frombuffer(constants[224:248], dtype=np.float32).astype(np.float64)
	res = ltc0.shape[1]; layers = ltc0.shape[0]
	f0_luminance = float(np.dot(f0, [0.2126, 0.7152, 0.0722]))
	u = math.sqrt(min(max(roughness, 0.0), 1.0)) * c[2] + c[3]
	v = math.acos(min(max(float(n @ wo), 0.0), 1.0)) * c[4] + c[5]
	layer = int(min(max(np.rint(min(max(f0_luminance, 0.0), 1.0) * c[0] + c[1]), 0), layers - 1))
	def fetch(table):
		x = u * res - 0.5; y = v * res - 0.5
		x0 = math.floor(x); y0 = math.floor(y); fx = x - x0; fy = y - y0
		cl = lambda i: min(max(i, 0), res - 1)
		t = table[layer].astype(np.float64) / 65535.0
		a = t[cl(y0), cl(x0)] * (1 - fx) + t[cl(y0), cl(x0 + 1)] * fx
		b = t[cl(y0 + 1), cl(x0)] * (1 - fx) + t[cl(y0 + 1), cl(x0 + 1)] * fx
		return a * (1 - fy) + b * fy
	return fetch(ltc0), fetch(ltc1)


def expected_bias_of_separate_sampling(case, lights, occluders, constants, ltc0, ltc1):
	"""The part of the specular integral strategy 2 never samples: directions above the tangent plane where the LTC's cosine-space z,
	-d0[1] (w . x_axis) + d1[0] (w . n) with x_axis the outgoing direction's tangent part, is not positive. Returns [3] (to subtract)."""
	_, x, n, albedo, f0, roughness, wo = case
	d0, d1 = ltc_coefficients(constants, ltc0, ltc1, f0, roughness, n, wo)
	x_axis = _unit(wo - (wo @ n) * n)
	below = -(-d0[1] * x_axis + d1[0] * n)
	return R.direct_lighting(x, n, wo, albedo, f0, roughness, lights, occluders, lobes=(False, True), planes=[below])


def truth(case_list, constants, light_count, occluders, strategy, ltc0, ltc1):
	"""[count, 3] float64 expectations, from the float32 inputs the kernel reads: the G-buffer values, the camera at byte 144, the lights' vertices
	and radiance from the constant block."""
	camera = np.frombuffer(constants[144:156], dtype=np.float32).astype(np.float64)
	lights = lights_from_constants(constants, light_count)
	out = []
	for family, x, n, albedo, f0, roughness in case_list:
		x = x.astype(np.float32).astype(np.float64); n = _unit(n.astype(np.float32).astype(np.float64))
		albedo = albedo.astype(np.float32).astype(np.float64); f0 = f0.astype(np.float32).astype(np.float64); roughness = float(np.float32(roughness))
		wo = _unit(camera - x)
		value = R.direct_lighting(x, n, wo, albedo, f0, roughness, lights, occluders)
		if strategy == api.STRATEGY_DIFFUSE_SPECULAR_SEPARATELY:
			value = value - expected_bias_of_separate_sampling((family, x, n, albedo, f0, roughness, wo), lights, occluders, constants, ltc0, ltc1)
		out.append(value)
	return np.array(out)


# ---- statistics ----------------------------------------------------------------------------------------------------------------------------

def check(name, case_list, frame_means, expected, resolution, stats_out=None):
	"""frame_means [K, count, 3]: batch means. Asserts every case and the configuration's chi-square; prints the worst |z|, the worst relative
	error and the worst achieved resolution. Returns the per-case (z, relative error, resolution)."""
	K = frame_means.shape[0]
	mean = frame_means.mean(axis=0)
	se = frame_means.std(axis=0, ddof=1) / math.sqrt(K)
	scale = np.maximum(expected, 1e-30)
	achieved = (SIGMAS * se + EPS * scale) / scale
	# z in units of the whole allowance: EPS I stands for a systematic error of up to SIGMAS deviations (PSA sampling of a nearly Lambertian lobe has
	# almost no variance, so there EPS decides)
	z = (mean - expected) / np.maximum(np.sqrt(se * se + (EPS * scale / SIGMAS) ** 2), 1e-300)
	rel = np.abs(mean - expected) / scale
	lit = expected > 0
	failures = []
	for k, case in enumerate(case_list):
		for ch in range(3):
			if not lit[k, ch]:
				# unlit (albedo and F0 zero, or the light fully occluded): a ray that slips through the crack between the occluder's two
				# triangles is a tiny, legitimate leak (the GPU shows 1e-6 of the unshadowed value); EPS of the brightest case bounds it
				if abs(mean[k, ch]) > EPS * float(expected.max()):
					failures.append("%s case %d (%s) channel %d: %.3e where nothing is lit" % (name, k, case[0], ch, mean[k, ch]))
				continue
			if abs(mean[k, ch] - expected[k, ch]) > SIGMAS * se[k, ch] + EPS * expected[k, ch]:
				failures.append("%s case %d (%s, roughness %g, f0 %s, albedo %s) channel %d: mean %.6e, float64 %.6e, rel %.2e, z %.1f"
					% (name, k, case[0], case[5], case[4].tolist(), case[3].tolist(), ch, mean[k, ch], expected[k, ch], rel[k, ch], z[k, ch]))
			if achieved[k, ch] > resolution:
				failures.append("%s case %d (%s, roughness %g, f0 %s, albedo %s) channel %d: resolution %.2e > %.2e"
					% (name, k, case[0], case[5], case[4].tolist(), case[3].tolist(), ch, achieved[k, ch], resolution))
	cases_lit = int(lit.any(axis=1).sum())
	mean_z2 = float((z[lit] ** 2).mean())
	bound = scipy_stats.chi2.ppf(1.0 - CHI_SQUARE_P, cases_lit) / cases_lit   # the channels of a case are correlated: count cases, not channels
	print("%-34s K=%3d worst |z| %4.1f, mean z^2 %.2f (bound %.2f), worst rel. error %.2e, worst resolution %.2e"
		% (name, K, float(np.abs(z[lit]).max()), mean_z2, bound, float(rel[lit].max()), float(achieved[lit].max())))
	if mean_z2 > bound:
		failures.append("%s: mean z^2 %.2f over %d cases above the chi-square bound %.2f" % (name, mean_z2, cases_lit, bound))
	assert not failures, "\n".join(failures)
	if stats_out is not None:
		stats_out.append((name, z, rel, achieved))


# ---- the CPU leg: the oracle on the synthetic G-buffer -----------------------------------------------------------------------------------

class HostConstants:
	"""The constant block as vkr_write_constants writes it without a device, with animated noise: each call is the next frame."""

	def __init__(self, info, noise_shape=NOISE):
		self.lib = lib = api.load_library()
		self.scene = api.Scene(); self.ltc = api.LtcTable(); self.noise = api.NoiseTable(); self.spec = api.SceneSpecification(); self.settings = api.RenderSettings()
		assert lib.vkr_load_scene(C.byref(self.scene), None, info["vks"].encode(), info["textures"].encode(), 0) == 0
		assert lib.vkr_load_ltc_table(C.byref(self.ltc), None, info["ltc"].encode(), 51) == 0
		assert lib.vkr_load_noise_table(C.byref(self.noise), None, noise_shape[0], noise_shape[1], noise_shape[2], api.NOISE_WHITE) == 0
		assert lib.vkr_quick_load(C.byref(self.spec), info["save"].encode()) == 0
		assert lib.vkr_create_and_assign_light_textures(None, None, C.byref(self.spec)) == 0
		lib.vkr_specify_default_render_settings(C.byref(self.settings))
		self.settings.animate_noise = 1; self.settings.exposure_factor = 1.0
		self.light_count = self.spec.polygonal_light_count
		self.vertex_counts = [self.spec.polygonal_lights[i].vertex_count for i in range(self.light_count)]

	def __call__(self, width, height, mis_visibility_estimate):
		self.settings.mis_visibility_estimate = mis_visibility_estimate
		size = self.lib.vkr_get_constants_size(C.byref(self.spec)); buf = (C.c_uint8 * size)()
		assert self.lib.vkr_write_constants(buf, C.byref(self.spec), C.byref(self.settings), C.byref(self.scene), C.byref(self.ltc), C.byref(self.noise), width, height) == size
		return bytes(buf)

	def close(self):
		lib = self.lib
		lib.vkr_destroy_scene_specification(C.byref(self.spec)); lib.vkr_destroy_noise_table(C.byref(self.noise), None)
		lib.vkr_destroy_ltc_table(C.byref(self.ltc), None); lib.vkr_destroy_scene(C.byref(self.scene), None)


# The CPU leg runs every configuration once, each on one of the light sets in turn and with shadow rays off and on in turn, at a lower resolution
# than the GPU leg; the oracle equals the device code and the GPU bit for bit, so this checks the same arithmetic. GGX MIS also runs on the mixed
# set: only a light with fewer vertices than the frame's largest one reaches the padded edges the ray / light test of GGX MIS skips.
CPU_FRAMES = 32
CPU_SAMPLES = 12
CPU_RESOLUTION = 0.02


def _cpu_plan():
	plan = [(config, LIGHT_SETS[i % len(LIGHT_SETS)], i % 2 == 1) for i, config in enumerate(CONFIGURATIONS)]
	return plan + [(config, "mixed", False) for config in CONFIGURATIONS if config[0] == api.STRATEGY_DIFFUSE_GGX_MIS]


@pytest.fixture(scope="module")
def cpu_inputs():
	from tests import harness as H
	infos = dataset()
	oi = H.OracleInputs(infos["v4"])
	oi.noise = uniform_noise_table(NOISE)
	return infos, oi


def run_oracle(info, oi, config, shadows, frames, samples, block):
	from oracle import binding as oracle
	strategy, heuristic, visibility = config
	constants_of = HostConstants(info)
	try:
		polygon = light_polygons(constants_of(8, 8, visibility), constants_of.light_count)[0]
		case_list = cases(polygon)
		gb = synthetic_gbuffer(case_list, block)
		height, width = gb.shape[1:3]
		counts = constants_of.vertex_counts
		cfg = dict(width=width, height=height, light_count=constants_of.light_count, max_light_vertex_count=max(counts), min_light_vertex_count=min(counts),
			sample_count=samples, sampling_strategies=strategy, mis_heuristic=heuristic, biased_sampling=0, trace_shadow_rays=int(shadows), show_polygonal_lights=0,
			row_begin=0, row_end=0, output_srgb=0, polygon_sampling_technique=api.TECHNIQUE_PSA, error_display=0)
		tris = oi.shadow_tris if shadows else np.zeros((0, 9), dtype=np.float32)
		means = []
		for f in range(frames):
			constants = constants_of(width, height, visibility)
			out, _ = oracle.shade(cfg, constants, gb, oi.noise, oi.ltc0, oi.ltc1, tris)
			means.append(block_means(out, len(case_list), block))
		occluders = oi.shadow_tris.reshape(-1, 3, 3) if shadows else ()
		expected = truth(case_list, constants, constants_of.light_count, occluders, strategy, oi.ltc0, oi.ltc1)
		return case_list, np.array(means), expected
	finally:
		constants_of.close()


def test_estimators_converge_to_the_float64_integral_on_the_cpu(cpu_inputs):
	infos, oi = cpu_inputs
	start = time.time()
	stats = []
	for config, light_set, shadows in _cpu_plan():
		case_list, means, expected = run_oracle(infos[light_set], oi, config, shadows, CPU_FRAMES, CPU_SAMPLES, BLOCK)
		check("%s %s shadows %d" % (config_name(config), light_set, shadows), case_list, means, expected, CPU_RESOLUTION, stats)
	print("CPU leg: %d configurations, %.1f s" % (len(stats), time.time() - start))


def test_the_white_noise_table_is_not_uniform_in_two_dimensions():
	"""The finding above: the reference's white noise table, as the oracle reads it, fails a chi-square test of its random pairs by far; the table
	these tests use passes it."""
	from tests import harness as H
	def chi_square_per_bin(table):
		t = table.reshape(-1, 4).astype(np.float64) / 65535.0
		h, _, _ = np.histogram2d(t[:, 0], t[:, 1], bins=64, range=[[0.0, 1.0], [0.0, 1.0]])
		expected = len(t) / 64.0 ** 2
		return float(((h - expected) ** 2 / expected).sum() / (64 * 64 - 1))
	white = chi_square_per_bin(H.white_noise_table(256, 256, 64)); uniform = chi_square_per_bin(uniform_noise_table((256, 256, 64)))
	print("chi-square per degree of freedom of the (R, G) pairs: white noise table %.1f, uniform table %.3f" % (white, uniform))
	assert white > 100.0 and uniform < 1.2


# ---- the float64 reference itself --------------------------------------------------------------------------------------------------------

def _local(P, x, n):
	t, b = R._tangent_frame(n)
	return np.stack([(P - x) @ t, (P - x) @ b, (P - x) @ n], axis=-1)


def test_the_float64_integral_on_known_answers():
	"""With f = 1 / pi the integral is the projected solid angle over pi (Lambert), above and across the horizon, on either side of the light;
	refining further changes nothing; a speck of a light is the point-light limit; an occluder that covers the light's cone leaves nothing and one
	that covers half of a square light leaves half of what a plane through x and the occluder's edge leaves."""
	rng = np.random.default_rng(5)
	lambert = lambda n: (lambda w: np.maximum(w @ n, 0.0)[:, None] / math.pi)
	for k in range(12):
		x = rng.normal(size=3); n = _unit(rng.normal(size=3))
		centre = x + _unit(n + rng.normal(scale=0.9, size=3)) * rng.uniform(0.5, 3.0)
		u = _unit(rng.normal(size=3)); v = _unit(np.cross(u, rng.normal(size=3)))
		count = 3 + k % 5
		angles = np.sort(rng.uniform(0, 2 * math.pi, count))
		poly = centre + rng.uniform(0.3, 1.5) * (np.cos(angles)[:, None] * u + np.sin(angles)[:, None] * v)
		got = float(R.light_integral(x, n, poly, lambert(n))[0])
		ref = R.clip_and_psa(_local(poly, x, n))[0] / math.pi
		assert abs(got - ref) <= 1e-10 * max(ref, 1e-3), (k, got, ref)
		# the same light seen from its other side: both faces emit
		mirror = x + 2.0 * ((centre - x) @ _unit(np.cross(poly[1] - poly[0], poly[2] - poly[0]))) * _unit(np.cross(poly[1] - poly[0], poly[2] - poly[0]))
		got = float(R.light_integral(mirror, n, poly, lambert(n))[0])
		assert abs(got - R.clip_and_psa(_local(poly, mirror, n))[0] / math.pi) <= 1e-10 * max(got, 1e-3)
	# refinement converges: a sharp lobe at rtol 1e-6 and 1e-10 agree to 1e-6
	x = np.zeros(3); n = np.array([0.0, 0.0, 1.0]); wo = _unit([0.4, 0.0, 1.0])
	poly = np.array([[-1.0, -1.0, 1.0], [1.0, -1.0, 1.0], [1.0, 1.0, 1.0], [-1.0, 1.0, 1.0]])
	fine = R.direct_lighting(x, n, wo, [0.5] * 3, [1.0] * 3, 0.05, [(poly, [1.0, 1.0, 1.0])])
	coarse = R.direct_lighting(x, n, wo, [0.5] * 3, [1.0] * 3, 0.05, [(poly, [1.0, 1.0, 1.0])], rtol=1e-6)
	assert np.abs(fine - coarse).max() <= 1e-6 * fine.max()
	# a speck: L A f cos(theta) cos(theta_L) / r^2
	p = np.array([0.3, -0.2, 2.0]); size = 1e-4
	speck = p + size * np.array([[-1.0, -1.0, 0.0], [1.0, -1.0, 0.0], [1.0, 1.0, 0.0], [-1.0, 1.0, 0.0]])
	w = _unit(p); d = float(np.linalg.norm(p))
	f = sum(R.brdf(w[None], wo, n, [0.5] * 3, [0.04] * 3, 0.3))[0]
	limit = f * w[2] * abs(w[2]) * (4.0 * size * size) / (d * d)
	got = R.direct_lighting(x, n, wo, [0.5] * 3, [0.04] * 3, 0.3, [(speck, [1.0, 1.0, 1.0])])
	assert np.abs(got - limit).max() <= 1e-6 * limit.max()
	# occluders: one covering the whole cone leaves nothing; one covering the half x > 0 of a centred square leaves the half x < 0
	big = [np.array([[-5.0, -5.0, 0.5], [5.0, -5.0, 0.5], [0.0, 5.0, 0.5]])]
	assert np.abs(R.direct_lighting(x, n, wo, [0.5] * 3, [0.04] * 3, 0.3, [(poly, [1.0] * 3)], occluders=big)).max() <= 1e-12
	half = [np.array([[0.0, -2.0, 0.5], [2.0, -2.0, 0.5], [2.0, 2.0, 0.5]]), np.array([[0.0, -2.0, 0.5], [2.0, 2.0, 0.5], [0.0, 2.0, 0.5]])]
	shadowed = R.direct_lighting(x, n, wo, [0.5] * 3, [0.04] * 3, 0.3, [(poly, [1.0] * 3)], occluders=half)
	left = R.direct_lighting(x, n, wo, [0.5] * 3, [0.04] * 3, 0.3, [(poly, [1.0] * 3)], planes=[(-1.0, 0.0, 0.0)])
	assert np.abs(shadowed - left).max() <= 1e-9 * left.max()
	# the BRDF: the diffuse lobe of a rough, white, non-metallic surface at normal incidence, F_D(1) F_D(1) / pi = 1 / pi
	diffuse, specular = R.brdf(np.array([[0.0, 0.0, 1.0]]), np.array([0.0, 0.0, 1.0]), n, [1.0] * 3, [0.0] * 3, 1.0)
	assert np.allclose(diffuse, 1.0 / math.pi, rtol=1e-14)
	# with f0 = 1 the specular lobe at the mirror direction is D G / (4 cos cos) with D = 1 / (pi alpha^2), G = 1 / (1 + Lambda(o) + Lambda(i))
	a = 0.3
	_, specular = R.brdf(np.array([[0.0, 0.0, 1.0]]), np.array([0.0, 0.0, 1.0]), n, [0.0] * 3, [1.0] * 3, a)
	assert np.allclose(specular, 1.0 / (math.pi * a * a) / 4.0, rtol=1e-12)
