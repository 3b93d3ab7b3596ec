"""Pins the CPU oracle against the REFERENCE's own shader sources.

tests/golden/ref_shader.npz holds (SHA-256 digests of) frames shaded by src/shaders/shading_pass.frag.glsl (+ includes) compiled as C++
(oracle/build_ref.py, oracle/glsl_compat/). The oracle must reproduce them bit for bit, for every sampling strategy
and MIS heuristic of the projected-solid-angle technique and for the related-work techniques ("_q<technique>": Turk, Urena, Arvo, Hart; SURVEY 8 f4). Where oracle/_ref/libref_shader.so is present (build
container, or shipped prebuilt) the reference shader is also run live and checked against the fixtures.
"""
import hashlib
import json
import os
import re

import numpy as np
import pytest

from tests import harness as H
from tests.ref_frames import WIDTH, HEIGHT, assert_matches_fixture, dataset_for, frame_sha256, host_constants, oracle_cfg
from oracle import ref_binding as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shader.npz")
LIVE_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_live.npz")


def _golden():
	return np.load(GOLDEN)


def _config_from_name(name):
	m = re.match(r"s(\d+)_h(\d+)_b(\d+)_L(\d+)_V(\d+)(?:m(\d+))?_S(\d+)_t(\d+)_l(\d+)_M(\d+)(?:_q(\d+))?(?:_e(\d))?(?:_x(\d))?(?:_y(\d))?(?:_o(\d)(\d))?$", name)
	s, h, b, L, V, Vmin, S, t, l, M, q, e, x, y, srgb, frame_bits = (int(x) if x is not None else None for x in m.groups())
	return dict(name=name, entry="ref_shade_" + name.replace("_x1", "").replace("_y1", ""), strategy=s, heuristic=h, biased=b, lights=L, max_vertices=V, min_vertices=V if Vmin is None else Vmin,
		samples=S, trace=t, show_lights=l, materials=M, technique=11 if q is None else q, error_display=e or 0, textured=x or 0, light_textures=y or 0, srgb=srgb or 0, frame_bits=frame_bits or 0)


def _names():
	return sorted({k.split("/")[0] for k in _golden().files})


@pytest.mark.parametrize("name", _names())
def test_oracle_reproduces_reference_shader_bit_for_bit(name):
	g = _golden(); cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
	sha = hashlib.sha256(open(info["vks"], "rb").read()).digest()
	assert bytes(g[name + "/vks_sha256"]) == sha, "the synthetic scene generator drifted: regenerate with tools/make_ref_golden.py"
	constants = host_constants(info, WIDTH, HEIGHT, cfg["lights"], frame_bits=cfg["frame_bits"])
	assert constants == bytes(g[name + "/constants"]), "the constant block drifted"
	vis = oi.visibility(WIDTH, HEIGHT, constants)
	assert np.array_equal(vis, g[name + "/visibility"])
	gb = oi.gbuffer(WIDTH, HEIGHT, constants, vis)
	out, _ = oi.shade(oracle_cfg(cfg), constants, gb)
	assert_matches_fixture(g, name, out)
	assert float(out[..., :3].max()) > 0.0


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libref_shader.so not built (needs /root/reference)")
def test_live_reference_shader_matches_fixture():
	g = _golden()
	live = {c["name"]: c for c in R.configs()}
	checked = 0
	for name in _names():
		if name not in live:
			continue
		cfg = live[name]
		info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
		constants = bytes(g[name + "/constants"])
		ref = R.shade(cfg["entry"], WIDTH, HEIGHT, cfg, constants, g[name + "/visibility"], oi.vks, oi.material_params, oi.noise, oi.ltc0, oi.ltc1, oi.shadow_tris, textures=oi.textures, light_textures=oi.light_textures)
		assert frame_sha256(ref) == bytes(g[name + "/rgba_sha256"]), name
		checked += 1
	assert checked > 0


OTHER_RESOLUTIONS = [(40, 30), (97, 41)]
OTHER_RESOLUTION_PICKS = ["s0_h0_b0_L3_V4_S3_t1_l1_M8", "s1_h1_b0_L3_V4_S3_t1_l1_M8", "s2_h0_b0_L3_V4_S3_t1_l1_M8", "s3_h3_b0_L3_V4_S3_t1_l1_M8", "s4_h0_b0_L3_V4_S3_t1_l1_M8",
	"s3_h4_b0_L3_V4_S3_t1_l1_M8", "s3_h3_b1_L3_V4_S3_t1_l1_M8", "s3_h3_b0_L3_V7m5_S3_t1_l1_M8", "s3_h3_b0_L32_V4_S2_t1_l1_M8",
	"s0_h0_b0_L3_V4_S3_t1_l1_M8_q3", "s0_h0_b0_L3_V4_S3_t1_l1_M8_q9", "s1_h0_b0_L3_V4_S3_t1_l1_M8_q10", "s0_h0_b0_L3_V7m5_S3_t1_l1_M8_q7",
	"s3_h3_b0_L3_V4_S3_t1_l1_M8_e4", "s3_h3_b0_L3_V4_S3_t1_l1_M8_x1"]


@pytest.mark.parametrize("width,height", OTHER_RESOLUTIONS)
def test_oracle_follows_the_live_reference_shader_at_other_resolutions(width, height):
	"""The fixtures are 64x48; other resolutions move every pixel ray, sample and noise fetch. A spread of configurations (every strategy,
	related-work techniques, error display, textures) shaded by the reference shader (frozen as SHA-256 digests of its float32 frames in
	tests/golden/ref_live.npz by tools/make_ref_live_golden.py) and by the oracle: bit-identical again."""
	frozen = np.load(LIVE_GOLDEN)
	for name in OTHER_RESOLUTION_PICKS:
		cfg = _config_from_name(name)
		info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
		constants = host_constants(info, width, height, cfg["lights"])
		vis = oi.visibility(width, height, constants)
		gb = oi.gbuffer(width, height, constants, vis)
		out, _ = oi.shade(oracle_cfg(cfg, width, height), constants, gb)
		assert frame_sha256(out) == frozen["shader/%dx%d/%s" % (width, height, name)].tobytes(), name


def test_every_light_texturing_technique_shapes_the_textured_fixture():
	"""The "_y1" fixtures exercise all three branches of get_polygon_radiance() (shading_pass.frag.glsl:155-181): replacing the texture of any one
	light (area, portal, IES profile) by white changes the oracle's frame, and the frame with all three equals the reference shader's (test above)."""
	g = _golden(); name = "s3_h3_b0_L3_V4_S3_t1_l1_M8_y1"; cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg)); oi = H.OracleInputs(info)
	assert [l["texturing_technique"] for l in info["lights"][:3]] == [1, 2, 3]
	constants = bytes(g[name + "/constants"])
	gb = oi.gbuffer(WIDTH, HEIGHT, constants, g[name + "/visibility"])
	ref, _ = oi.shade(oracle_cfg(cfg), constants, gb)
	assert_matches_fixture(g, name, ref)
	dims, offsets, data = oi.light_textures
	for i in range(3):
		d = dims.copy(); o = offsets.copy(); white = np.concatenate([data, np.ones(4, dtype=np.float32)])
		d[i] = (1, 1, 1); o[i] = len(data)
		out, _ = H.oracle.shade(oracle_cfg(cfg), constants, gb, oi.noise, oi.ltc0, oi.ltc1, oi.shadow_tris, light_textures=(d, o, white))
		changed = (out.view(np.uint32) != ref.view(np.uint32)).any(axis=-1).mean()
		assert changed > 0.02, "light %d (technique %d) leaves the frame unchanged" % (i, i + 1)
