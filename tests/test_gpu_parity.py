"""Parity of the CUDA shading path (through the C-ABI) against the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star): per-pixel radiance within 1e-5 relative, shadow-ray hit/miss bit-exact.
Because oracle and kernel implement the same arithmetic contract (DESIGN.md) the expected result is
bit-identical float32 output; the tests assert the 1e-5 bar and report bit-exactness.
"""
import numpy as np
import pytest

from tests import harness as H
from tests.ref_frames import assert_matches_fixture
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu

REL_TOL = 1.0e-5  # relative per-pixel radiance tolerance stated by BASELINE.json


def _run_both(name, width, height, **settings):
	info = H.dataset(name)
	oi = H.OracleInputs(info)
	frame = H.open_frame(info)
	try:
		frame.configure(**settings)
		constants = frame.constants(width, height)
		vis_gpu, gb_gpu = frame.gbuffer_host(width, height)
		vis_cpu = oi.visibility(width, height, constants)
		gb_cpu = oi.gbuffer(width, height, constants, vis_cpu)
		out_gpu = frame.shade_host(width, height, gb_cpu)
		cfg = H.oracle_config(frame, width, height)
		out_cpu, rays = oi.shade(cfg, constants, gb_cpu)
	finally:
		frame.close()
	return dict(vis_gpu=vis_gpu, vis_cpu=vis_cpu, gb_gpu=gb_gpu, gb_cpu=gb_cpu, out_gpu=out_gpu, out_cpu=out_cpu, rays=rays)


def _assert_parity(r, label):
	cmp = H.compare_radiance(r["out_gpu"], r["out_cpu"], rel=REL_TOL)
	print(label, cmp, "oracle rays", r["rays"])
	assert cmp["nan_mismatch"] == 0
	assert cmp["bad_pixels"] == 0, cmp
	return cmp


@pytest.mark.parametrize("strategy", [api.STRATEGY_DIFFUSE_ONLY, api.STRATEGY_DIFFUSE_SPECULAR_MIS])
@pytest.mark.parametrize("trace", [0, 1])
def test_cornell_config1_like(strategy, trace):
	"""BASELINE config 1 (Cornell, 1 quad light, 1 spp) plus the MIS variant, rays off and on."""
	r = _run_both("cornell", 256, 256, sample_count=1, strategy=strategy, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=trace)
	cmp = _assert_parity(r, "cornell s=%d t=%d" % (strategy, trace))
	assert cmp["bit_exact"]


def test_visibility_and_gbuffer_producer_match_oracle():
	r = _run_both("mini_city", 160, 96, sample_count=1)
	assert np.array_equal(r["vis_gpu"], r["vis_cpu"])
	assert np.array_equal(r["gb_gpu"].view(np.uint32), r["gb_cpu"].view(np.uint32))


@pytest.mark.parametrize("strategy,heuristic", [
	(api.STRATEGY_DIFFUSE_ONLY, api.MIS_BALANCE),
	(api.STRATEGY_DIFFUSE_GGX_MIS, api.MIS_BALANCE), (api.STRATEGY_DIFFUSE_GGX_MIS, api.MIS_POWER),
	(api.STRATEGY_DIFFUSE_SPECULAR_SEPARATELY, api.MIS_BALANCE),
	(api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_BALANCE), (api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_POWER), (api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_WEIGHTED),
	(api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_OPTIMAL_CLAMPED), (api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_OPTIMAL),
	(api.STRATEGY_DIFFUSE_SPECULAR_RANDOM, api.MIS_BALANCE),
])
def test_all_strategies_and_heuristics(strategy, heuristic):
	r = _run_both("mini_city", 160, 96, sample_count=3, strategy=strategy, heuristic=heuristic, trace_shadow_rays=1)
	_assert_parity(r, "mini_city s=%d h=%d" % (strategy, heuristic))


def test_biased_variant():
	r = _run_both("mini_city", 160, 96, sample_count=2, technique=api.TECHNIQUE_PSA_BIASED, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, trace_shadow_rays=1)
	_assert_parity(r, "biased")


def test_config3_like_many_samples():
	"""8 lights would need the 'city' set; mini_city has 3 quads: 64 spp exercises the noise period (128 fetches/pixel wrap)."""
	r = _run_both("mini_city", 96, 64, sample_count=64, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)
	_assert_parity(r, "64spp")


def _fixture_names():
	import os
	g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shader.npz"))
	return sorted({k.split("/")[0] for k in g.files if not any(tag in k.split("/")[0] for tag in ("_q", "_e", "_x", "_y"))})   # "_q<technique>": tests/test_gpu_related_work.py, "_e<error display>": tests/test_gpu_zz_error_display.py, "_x1" (textured): tests/test_gpu_zzy_textured_gbuffer.py, "_y1" (textured lights): tests/test_gpu_zzx_textured_lights.py


@pytest.mark.parametrize("name", _fixture_names())
def test_cuda_path_reproduces_reference_shader_fixture(name):
	"""CUDA visibility + G-buffer producer + shading megakernel against frames shaded by the REFERENCE's own shader
	sources (tests/golden/ref_shader.npz, see tests/test_ref_shader.py): bit-identical float32 radiance."""
	import os
	from tests.test_ref_shader import _config_from_name
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shader.npz"))
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg))
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=cfg["samples"], strategy=cfg["strategy"], heuristic=cfg["heuristic"],
			technique=api.TECHNIQUE_PSA_BIASED if cfg["biased"] else api.TECHNIQUE_PSA, trace_shadow_rays=cfg["trace"], show_lights=cfg["show_lights"], light_count=cfg["lights"], output_srgb=cfg["srgb"], frame_bits=cfg["frame_bits"])
		constants = frame.constants(WIDTH, HEIGHT)
		assert constants == bytes(g[name + "/constants"])
		vis, gb = frame.gbuffer_host(WIDTH, HEIGHT)
		assert np.array_equal(vis, g[name + "/visibility"])
		out = frame.shade_host(WIDTH, HEIGHT, gb)
	finally:
		frame.close()
	assert_matches_fixture(g, name, out)
