"""The product's device sampling code, compiled for the CPU, against the oracle (bit for bit).

vulkan_renderer_b200/csrc/vkr_related_work.cuh (with vkr_psa.cuh and vkr_device_math.cuh underneath) uses no warp intrinsics, so
tests/device_on_host.cpp compiles the same source with g++ -ffp-contract=off. The oracle side (oracle/related_work_oracle.h) is
pinned against the reference shader (tests/test_ref_shader.py, fixtures "_q<technique>"); this test closes the chain to the
code the GPU runs for SURVEY 8 row f4 -- the -m gpu tests then exercise it inside the kernel.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import harness as H
from tests.ref_frames import assert_matches_fixture, host_constants
from oracle import binding as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libdevice_on_host.so")
TECHNIQUES = {0: "baseline", 1: "area (Turk)", 2: "rectangle solid angle (Urena)", 3: "solid angle (Arvo)", 4: "solid angle", 5: "clipped solid angle",
	6: "bilinear warp (Hart)", 7: "bilinear warp, clipped (Hart)", 8: "biquadratic warp (Hart)", 9: "biquadratic warp, clipped (Hart)", 10: "projected solid angle (Arvo)"}
DATASETS = {3: "mini_tri", 4: "mini_city", 5: "mini_v5", 6: "mini_v6", 7: "mini_v7"}
MIXED = {4: "mini_mixed", 7: "mini_poly"}   # lights with fewer vertices than the bound


def _lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	return C.CDLL(LIB_PATH)


def _light_blocks(name, maxv):
	info = H.dataset(name)
	constants = host_constants(info, 64, 48, 3)
	stride = 160 + 16 * maxv * 2 + 16 * (maxv - 2)
	assert len(constants) == 256 + 3 * stride
	return [constants[256 + i * stride: 256 + (i + 1) * stride] for i in range(3)]


def _scenarios(block, rng, count):
	"""Shading points around the light with random shading frames: position, rows x/y/z of world_to_shading_space, translation."""
	b = np.frombuffer(block, dtype=np.float32)
	centre = b[4:7]
	out = []
	for _ in range(count):
		position = (centre + rng.uniform(-3.0, 3.0, 3)).astype(np.float32)
		n = rng.normal(size=3); n /= np.linalg.norm(n)
		x = np.cross(n, rng.normal(size=3)); x /= np.linalg.norm(x)
		y = np.cross(n, x)
		rows = np.stack([x, y, n]).astype(np.float32)
		t = -(rows.astype(np.float64) @ position.astype(np.float64))
		out.append((position, np.concatenate([rows.reshape(9), t.astype(np.float32)])))
	return out


def _compare(technique, maxv, dataset, seed, points=24, samples=16):
	lib = _lib()
	rng = np.random.default_rng(seed)
	checked = culled = 0
	for block in _light_blocks(dataset, maxv):
		for position, frame in _scenarios(block, rng, points):
			rnd = rng.random((samples, 2)).astype(np.float32)
			rnd[0] = (0.0, 0.0); rnd[1] = (np.float32(1.0) - np.float32(2.0 ** -24), 0.5)   # the ends of the unit interval
			ref = O.related_work_batch(technique, maxv, block, position, frame, rnd)
			dev = O.related_work_batch(technique, maxv, block, position, frame, rnd, symbol_library=lib, symbol="vkr_device_on_host_related_work_batch")
			assert (ref is None) == (dev is None), "culling differs"
			if ref is None:
				culled += 1
				continue
			for a, b, what in zip(ref[:2], dev[:2], ("direction", "density")):
				same = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))   # sign and payload of a NaN are the host compiler's business (x86: 0 / 0 is -NaN)
				assert same.all(), "%s differs: technique %d (%s), %s" % (what, technique, TECHNIQUES[technique], dataset)
			assert np.float32(ref[2]).view(np.uint32) == np.float32(dev[2]).view(np.uint32)
			checked += 1
	return checked, culled


@pytest.mark.parametrize("technique", sorted(TECHNIQUES))
@pytest.mark.parametrize("maxv", sorted(DATASETS))
def test_device_sampler_matches_oracle(technique, maxv):
	checked, _ = _compare(technique, maxv, DATASETS[maxv], seed=100 * technique + maxv)
	assert checked > 0


@pytest.mark.parametrize("technique", [3, 4, 5, 7, 9, 10])
@pytest.mark.parametrize("maxv", sorted(MIXED))
def test_device_sampler_matches_oracle_with_mixed_vertex_counts(technique, maxv):
	checked, _ = _compare(technique, maxv, MIXED[maxv], seed=7000 + 100 * technique + maxv)
	assert checked > 0


def _error_batch(lib, symbol, technique, biased, maxv, vertices, rnd, error_factor):
	vertices = np.ascontiguousarray(vertices, dtype=np.float32); rnd = np.ascontiguousarray(rnd, dtype=np.float32)
	n = len(rnd); errors = np.zeros((n, 3), dtype=np.float32); colors = np.zeros((n, 3), dtype=np.float32)
	fn = getattr(lib, symbol); fn.restype = C.c_int
	on = fn(C.c_uint32(technique), C.c_int(biased), C.c_uint32(maxv), C.c_uint32(len(vertices)), vertices.ctypes.data_as(C.c_void_p), C.c_uint32(n), rnd.ctypes.data_as(C.c_void_p),
		C.c_float(error_factor), errors.ctypes.data_as(C.c_void_p), colors.ctypes.data_as(C.c_void_p))
	assert on >= 0
	return None if on == 0 else (errors, colors)


@pytest.mark.parametrize("technique,biased", [(11, 0), (11, 1), (10, 0)])
@pytest.mark.parametrize("maxv", [3, 4, 5, 6, 7])
def test_device_sampling_error_and_error_colours_match_oracle(technique, biased, maxv):
	"""Error display (ERROR_DISPLAY_*): the sampling error of projected solid angle sampling (ours: three measures, Arvo's: two) and the colour map."""
	lib = _lib(); oracle = O.load()
	rng = np.random.default_rng(31 * maxv + technique + biased)
	checked = 0; colours = set()
	for trial in range(60):
		count = maxv if trial % 3 else int(rng.integers(3, maxv + 1))
		angles = np.sort(rng.uniform(0.0, 2.0 * np.pi, count))
		centre = rng.normal(size=3) * np.array([1.5, 1.5, 0.8]) + np.array([0.0, 0.0, 0.6])
		u = rng.normal(size=3); u /= np.linalg.norm(u); w = np.cross(u, rng.normal(size=3)); w /= np.linalg.norm(w)
		vertices = centre + rng.uniform(0.3, 1.5) * (np.outer(np.cos(angles), u) + np.outer(np.sin(angles), w))
		rnd = rng.random((24, 2)).astype(np.float32)
		error_factor = float(10.0 ** rng.uniform(3.0, 8.0))
		ref = _error_batch(oracle, "vkr_oracle_error_display_batch", technique, biased, maxv, vertices, rnd, error_factor)
		dev = _error_batch(lib, "vkr_device_on_host_error_display_batch", technique, biased, maxv, vertices, rnd, error_factor)
		assert (ref is None) == (dev is None)
		if ref is None:
			continue
		assert np.array_equal(ref[0].view(np.uint32), dev[0].view(np.uint32)) and np.array_equal(ref[1].view(np.uint32), dev[1].view(np.uint32))
		checked += 1; colours |= {tuple(c) for c in ref[1]}
	assert checked > 10 and len(colours) > 3


@pytest.mark.parametrize("shape", [(64, 64), (32, 16), (5, 7), (1, 1)])
def test_device_texture_filter_matches_the_definition(shape):
	"""csrc/vkr_texture.cuh (textureGrad of the G-buffer producer) against oracle/texture_filter.h: magnification, minification over the whole
	chain, anisotropic footprints in every direction, repeat addressing, degenerate derivatives."""
	from vulkan_renderer_b200 import synth
	lib = _lib()
	h, w = shape
	rng = np.random.default_rng(w * 100 + h)
	levels = synth.mip_chain(rng.random((h, w, 4)).astype(np.float32))
	texels = np.concatenate([l.reshape(-1) for l in levels]).astype(np.float32)
	n = 4000
	uv = rng.uniform(-3.0, 4.0, (n, 2))
	scale = 10.0 ** rng.uniform(-4.0, 0.5, (n, 1))
	angle = rng.uniform(0.0, 2.0 * np.pi, (n, 1)); stretch = 10.0 ** rng.uniform(0.0, 1.6, (n, 1))
	ddx = scale * stretch * np.concatenate([np.cos(angle), np.sin(angle)], 1)
	ddy = scale * np.concatenate([-np.sin(angle), np.cos(angle)], 1) * rng.choice([1.0, 0.3, 3.0], (n, 1))
	inputs = np.concatenate([uv, ddx, ddy], 1).astype(np.float32)
	inputs[:8, 2:] = 0.0; inputs[8:12, 2:4] = 0.0; inputs[12, 0] = np.nan; inputs[13, 2] = np.inf; inputs[14, 4] = -np.inf; inputs[15, :2] = 1e30
	ref = O.texture_grad_batch(w, h, len(levels), texels, inputs)
	out = np.zeros((n, 4), dtype=np.float32)
	lib.vkr_device_on_host_texture_grad_batch(C.c_uint32(w), C.c_uint32(h), C.c_uint32(len(levels)), texels.ctypes.data_as(C.c_void_p), C.c_uint32(n),
		inputs.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
	assert np.isfinite(ref[16:]).all()


@pytest.mark.parametrize("name", ["mini_city", "mini_textured", "cornell"])
def test_gbuffer_kernel_body_matches_the_oracle(name):
	"""The whole per-pixel body of the G-buffer kernel (csrc/vkr_gbuffer.cuh: triangle decode, barycentrics, screen-space derivatives, three textureGrad over
	BC1 / RGBA16F / BC5 mip chains, normal mapping) run on the CPU for every pixel of a frame, against get_shading_data() of the oracle: bit-identical."""
	lib = _lib()
	width, height = 120, 68
	info = H.dataset(name); oi = H.OracleInputs(info)
	constants = host_constants(info, width, height, len(info["lights"]))
	vis = oi.visibility(width, height, constants)
	ref = oi.gbuffer(width, height, constants, vis)
	out = np.zeros((4, height, width, 4), dtype=np.float32)
	q = np.ascontiguousarray(oi.vks["positions"], dtype=np.uint32); nt = np.ascontiguousarray(oi.vks["normals_uv"], dtype=np.uint16)
	mi = np.ascontiguousarray(oi.vks["material_indices"], dtype=np.uint8); mp = np.ascontiguousarray(oi.material_params, dtype=np.float32)
	P = lambda a: a.ctypes.data_as(C.c_void_p)
	if oi.textures is not None:
		dims3, offsets, data = oi.textures
		dims = np.zeros((len(dims3), 4), dtype=np.uint32); dims[:, :3] = dims3
		offsets_texels = (offsets // 4).astype(np.uint64)
		tex = (P(dims), P(offsets_texels), P(data))
	else:
		tex = (None, None, None)
	cb = (C.c_uint8 * len(constants)).from_buffer_copy(constants)
	lib.vkr_device_on_host_gbuffer(C.c_uint32(width), C.c_uint32(height), cb, P(vis), P(q), P(nt), P(mi), P(mp), tex[0], tex[1], tex[2], P(out))
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
	assert (vis != 0xFFFFFFFF).mean() > 0.3


def _error_display_fixture_names():
	import os
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	return sorted({k.split("/")[0] for k in g.files if "_e" in k.split("/")[0]})


@pytest.mark.parametrize("name", _error_display_fixture_names())
def test_error_display_light_shader_reproduces_the_reference_shader_fixtures(name):
	"""csrc/vkr_error_display.cuh -- what error_display_kernel runs per (pixel, light): clipping in shading / cosine space, preparation, the one sample, its
	error, the colour map, noise consumption across lights -- executed on the CPU for whole frames, against the frames of the reference's own shader compiled
	with ERROR_DISPLAY_* (fixtures "_e<n>"). Bit-identical, pink pixels included."""
	import os
	from tests.test_ref_shader import _config_from_name
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	lib = _lib()
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
	constants = bytes(g[name + "/constants"])
	gb = np.ascontiguousarray(oi.gbuffer(WIDTH, HEIGHT, constants, g[name + "/visibility"]), dtype=np.float32)
	out = np.zeros((HEIGHT, WIDTH, 4), dtype=np.float32)
	technique = cfg["technique"] if cfg["technique"] != 11 else (12 if cfg["biased"] else 11)
	P = lambda a: a.ctypes.data_as(C.c_void_p)
	noise = np.ascontiguousarray(oi.noise, dtype=np.uint16); ltc0 = np.ascontiguousarray(oi.ltc0, dtype=np.uint16); ltc1 = np.ascontiguousarray(oi.ltc1, dtype=np.uint16)
	cb = (C.c_uint8 * len(constants)).from_buffer_copy(constants)
	rc = lib.vkr_device_on_host_error_display_frame(C.c_uint32(WIDTH), C.c_uint32(HEIGHT), C.c_uint32(cfg["max_vertices"]), C.c_uint32(cfg["lights"]), C.c_uint32(technique),
		C.c_uint32(cfg["error_display"]), C.c_int(cfg["show_lights"]), cb, P(gb), P(noise), C.c_uint32(noise.shape[2]), C.c_uint32(noise.shape[1]), C.c_uint32(noise.shape[0]),
		P(ltc0), P(ltc1), C.c_uint32(ltc0.shape[1]), C.c_uint32(ltc0.shape[0]), P(out))
	assert rc == 0
	assert_matches_fixture(g, name, out)


def _base_fixture_names():
	import os
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	return sorted({k.split("/")[0] for k in g.files if not any(t in k.split("/")[0] for t in ("_q", "_e", "_x", "_y"))})   # incl. "_o<srgb><frame bits>": the output stage


@pytest.mark.parametrize("name", _base_fixture_names())
def test_shade_light_without_rays_matches_oracle_and_fixtures(name):
	"""csrc/vkr_shade_light.cuh -- shade_light<STRATEGY, MAXP, BIASED, OPTIMAL, TRACE = false>, the per-(pixel, light) body of the benchmark kernel with the
	shadow test compiled out -- executed on the CPU for whole frames of every base fixture configuration (all strategies, heuristics, vertex bounds 3..7, mixed
	vertex counts, 1..32 lights, up to 256 spp). Against the oracle with rays off; the fixtures the reference shader rendered with rays off are compared
	directly as well. Bit-identical. With test_host_logic's traversal tests this leaves only the warp-level ray ring of the GPU path unexercised on the CPU."""
	import os
	from tests.test_ref_shader import _config_from_name, oracle_cfg
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	lib = _lib()
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
	constants = bytes(g[name + "/constants"])
	gb = np.ascontiguousarray(oi.gbuffer(WIDTH, HEIGHT, constants, g[name + "/visibility"]), dtype=np.float32)
	out = np.zeros((HEIGHT, WIDTH, 4), dtype=np.float32)
	P = lambda a: a.ctypes.data_as(C.c_void_p)
	noise = np.ascontiguousarray(oi.noise, dtype=np.uint16); ltc0 = np.ascontiguousarray(oi.ltc0, dtype=np.uint16); ltc1 = np.ascontiguousarray(oi.ltc1, dtype=np.uint16)
	cb = (C.c_uint8 * len(constants)).from_buffer_copy(constants)
	rc = lib.vkr_device_on_host_shade_frame(C.c_uint32(WIDTH), C.c_uint32(HEIGHT), C.c_uint32(cfg["max_vertices"]), C.c_uint32(cfg["lights"]), C.c_uint32(cfg["technique"]), C.c_uint32(cfg["strategy"]),
		C.c_uint32(cfg["heuristic"]), C.c_int(cfg["biased"]), C.c_uint32(cfg["samples"]), C.c_int(cfg["show_lights"]), cb, P(gb),
		P(noise), C.c_uint32(noise.shape[2]), C.c_uint32(noise.shape[1]), C.c_uint32(noise.shape[0]), P(ltc0), P(ltc1), C.c_uint32(ltc0.shape[1]), C.c_uint32(ltc0.shape[0]), C.c_int(cfg["srgb"]),
		C.c_uint32(0), None, None, None, P(out))
	assert rc == 0
	no_rays = dict(cfg, trace=0)
	ref, _ = oi.shade(oracle_cfg(no_rays), constants, gb)
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)
	if cfg["trace"] == 0:
		assert_matches_fixture(g, name, out)


def _related_work_fixture_names():
	import os
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	return sorted({k.split("/")[0] for k in g.files if "_q" in k.split("/")[0] and not any(t in k.split("/")[0] for t in ("_e", "_y"))})


@pytest.mark.parametrize("name", _related_work_fixture_names())
def test_related_work_light_shader_without_rays_matches_oracle_and_fixtures(name):
	"""csrc/vkr_related_work_light.cuh -- the per-(pixel, light) code of related_work_kernel: preparation, sample loop, the NaN rules, GGX MIS -- executed
	on the CPU for whole frames of every "_q<technique>" fixture configuration with the shadow test compiled out, against the oracle with rays off (and the
	fixture itself where the reference shader rendered it without rays). Bit-identical."""
	import os
	from tests.test_ref_shader import _config_from_name, oracle_cfg
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	lib = _lib()
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
	constants = bytes(g[name + "/constants"])
	gb = np.ascontiguousarray(oi.gbuffer(WIDTH, HEIGHT, constants, g[name + "/visibility"]), dtype=np.float32)
	out = np.zeros((HEIGHT, WIDTH, 4), dtype=np.float32)
	P = lambda a: a.ctypes.data_as(C.c_void_p)
	noise = np.ascontiguousarray(oi.noise, dtype=np.uint16); ltc0 = np.ascontiguousarray(oi.ltc0, dtype=np.uint16); ltc1 = np.ascontiguousarray(oi.ltc1, dtype=np.uint16)
	cb = (C.c_uint8 * len(constants)).from_buffer_copy(constants)
	rc = lib.vkr_device_on_host_shade_frame(C.c_uint32(WIDTH), C.c_uint32(HEIGHT), C.c_uint32(cfg["max_vertices"]), C.c_uint32(cfg["lights"]), C.c_uint32(cfg["technique"]), C.c_uint32(cfg["strategy"]),
		C.c_uint32(cfg["heuristic"]), C.c_int(0), C.c_uint32(cfg["samples"]), C.c_int(cfg["show_lights"]), cb, P(gb),
		P(noise), C.c_uint32(noise.shape[2]), C.c_uint32(noise.shape[1]), C.c_uint32(noise.shape[0]), P(ltc0), P(ltc1), C.c_uint32(ltc0.shape[1]), C.c_uint32(ltc0.shape[0]), C.c_int(0),
		C.c_uint32(0), None, None, None, P(out))
	assert rc == 0
	ref, _ = oi.shade(oracle_cfg(dict(cfg, trace=0)), constants, gb)
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)
	if cfg["trace"] == 0:
		assert_matches_fixture(g, name, out)


def _textured_light_fixture_names():
	import os
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	return sorted({k.split("/")[0] for k in g.files if "_y1" in k.split("/")[0]})   # incl. "_q4_y1": a related-work technique under textured lights


@pytest.mark.parametrize("name", _textured_light_fixture_names())
def test_textured_lights_without_rays_match_oracle_and_fixtures(name):
	"""The LIGHT_TEXTURES = true instantiation of shade_light() and of the light display (what csrc/vkr_textured_light_kernel.cu runs per pixel: area texture,
	portal onto a light probe, IES profile; get_polygon_radiance, shading_pass.frag.glsl:151-185) executed on the CPU for whole frames of the "_y1" fixture
	configurations, rays off: bit-identical to the oracle, and to the reference shader's own frame where the fixture was rendered without rays."""
	import os
	from tests.test_ref_shader import _config_from_name, oracle_cfg
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	lib = _lib()
	g = np.load(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"))
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
	assert oi.light_textures is not None
	constants = bytes(g[name + "/constants"])
	gb = np.ascontiguousarray(oi.gbuffer(WIDTH, HEIGHT, constants, g[name + "/visibility"]), dtype=np.float32)
	out = np.zeros((HEIGHT, WIDTH, 4), dtype=np.float32)
	P = lambda a: a.ctypes.data_as(C.c_void_p)
	noise = np.ascontiguousarray(oi.noise, dtype=np.uint16); ltc0 = np.ascontiguousarray(oi.ltc0, dtype=np.uint16); ltc1 = np.ascontiguousarray(oi.ltc1, dtype=np.uint16)
	dims3, offsets, data = oi.light_textures
	dims = np.zeros((len(dims3), 4), dtype=np.uint32); dims[:, :3] = dims3
	offsets_texels = np.ascontiguousarray(offsets // 4, dtype=np.uint64); data = np.ascontiguousarray(data, dtype=np.float32)
	cb = (C.c_uint8 * len(constants)).from_buffer_copy(constants)
	rc = lib.vkr_device_on_host_shade_frame(C.c_uint32(WIDTH), C.c_uint32(HEIGHT), C.c_uint32(cfg["max_vertices"]), C.c_uint32(cfg["lights"]), C.c_uint32(cfg["technique"]), C.c_uint32(cfg["strategy"]),
		C.c_uint32(cfg["heuristic"]), C.c_int(cfg["biased"]), C.c_uint32(cfg["samples"]), C.c_int(cfg["show_lights"]), cb, P(gb),
		P(noise), C.c_uint32(noise.shape[2]), C.c_uint32(noise.shape[1]), C.c_uint32(noise.shape[0]), P(ltc0), P(ltc1), C.c_uint32(ltc0.shape[1]), C.c_uint32(ltc0.shape[0]), C.c_int(0),
		C.c_uint32(len(dims)), P(dims), P(offsets_texels), P(data), P(out))
	assert rc == 0
	ref, _ = oi.shade(oracle_cfg(dict(cfg, trace=0)), constants, gb)
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)
	if cfg["trace"] == 0:
		assert_matches_fixture(g, name, out)
	# the textures matter: the same frame with white textures differs
	white, _ = H.oracle.shade(oracle_cfg(dict(cfg, trace=0)), constants, gb, oi.noise, oi.ltc0, oi.ltc1, np.zeros((0, 9), dtype=np.float32),
		light_textures=(np.array([[1, 1, 1]] * len(dims), dtype=np.uint32), np.arange(len(dims), dtype=np.uint64) * 4, np.ones(4 * len(dims), dtype=np.float32)))
	assert not np.array_equal(white, ref)


def test_samples_point_at_the_light_and_densities_integrate():
	"""Sanity of the oracle side itself (not only agreement): directions are unit vectors that hit the light's plane in front of the
	shading point, and 1/density averages to the solid angle for the solid-angle techniques (2, 3, 4 agree with each other)."""
	rng = np.random.default_rng(5)
	block = _light_blocks("mini_city", 4)[0]
	b = np.frombuffer(block, dtype=np.float32)
	plane = b[16:20]
	position, frame = _scenarios(block, rng, 1)[0]
	rnd = rng.random((4096, 2)).astype(np.float32)
	solid_angles = {}
	for technique in (2, 3, 4):
		dirs, dens, ggx = O.related_work_batch(technique, 4, block, position, frame, rnd)
		assert np.allclose(np.linalg.norm(dirs, axis=1), 1.0, atol=1e-4)
		tt = -(plane[:3] @ position + plane[3]) / (dirs @ plane[:3])
		assert (tt > 0).mean() > 0.999
		solid_angles[technique] = 1.0 / float(np.median(dens))
		assert abs(ggx * solid_angles[technique] - 1.0) < 1e-4
	assert abs(solid_angles[3] / solid_angles[4] - 1.0) < 1e-3
	assert abs(solid_angles[2] / solid_angles[4] - 1.0) < 1e-3   # the lights of mini_city are rectangles


@pytest.mark.parametrize("which_device,which_oracle,lo,hi", [(0, "atan", -50.0, 50.0), (1, "sin", -20.0, 20.0), (2, "cos", -20.0, 20.0), (3, "acos", -1.0, 1.0), (4, "atan2_pair", -4.0, 4.0), (5, "cbrt_pow", 0.0, 30.0), (6, "fast_positive_atan", -8.0, 8.0)])
def test_device_elementary_functions_match_oracle(which_device, which_oracle, lo, hi):
	lib = _lib()
	x = np.random.default_rng(which_device).uniform(lo, hi, 20000).astype(np.float32)
	y = np.zeros_like(x)
	lib.vkr_device_on_host_elementary_batch(C.c_int(which_device), C.c_uint32(len(x)), x.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p))
	ref = O.elementary(which_oracle, x)
	assert np.array_equal(y.view(np.uint32), ref.view(np.uint32))
