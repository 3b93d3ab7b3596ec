"""The related-work polygon sampling techniques on the GPU (SURVEY 8 row f4: Turk, Urena, Arvo, Hart et al., solid angle sampling).

vkr_related_work_kernel.cu against (1) frames shaded by the REFERENCE's own shader sources with SAMPLE_POLYGON_<technique>
(tests/golden/ref_shader.npz, fixtures "_q<technique>", see tests/test_ref_shader.py) and (2) the CPU oracle on a larger
frame. Bar: BASELINE.json's 1e-5 relative per-pixel radiance; expected and asserted: bit-identical float32 frames.
The same device functions are held against the oracle on the CPU by tests/test_device_on_host.py.
"""
import os

import numpy as np
import pytest

from tests import harness as H
from tests.ref_frames import assert_matches_fixture
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu

REL_TOL = 1.0e-5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shader.npz")


def _fixture_names():
	g = np.load(GOLDEN)
	return sorted({k.split("/")[0] for k in g.files if "_q" in k.split("/")[0] and "_e" not in k.split("/")[0] and "_y" not in k.split("/")[0]})   # "_e<error display>": tests/test_gpu_zz_error_display.py, "_y1" (textured lights): tests/test_gpu_zzx_textured_lights.py


@pytest.mark.parametrize("name", _fixture_names())
def test_related_work_technique_reproduces_reference_shader_fixture(name):
	from tests.test_ref_shader import _config_from_name
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	g = np.load(GOLDEN)
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg))
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=cfg["samples"], strategy=cfg["strategy"], heuristic=cfg["heuristic"], technique=cfg["technique"],
			trace_shadow_rays=cfg["trace"], show_lights=cfg["show_lights"], light_count=cfg["lights"])
		constants = frame.constants(WIDTH, HEIGHT)
		assert constants == bytes(g[name + "/constants"])
		vis, gb = frame.gbuffer_host(WIDTH, HEIGHT)
		assert np.array_equal(vis, g[name + "/visibility"])
		out = frame.shade_host(WIDTH, HEIGHT, gb)
	finally:
		frame.close()
	assert_matches_fixture(g, name, out)


@pytest.mark.parametrize("technique", range(11))
def test_related_work_technique_matches_oracle_on_a_larger_frame(technique):
	"""160x90, 3 quad lights, 5 spp, shadow rays: more pixels, tiles that straddle the frame border, more ring traffic than the fixtures."""
	info = H.dataset("mini_city"); oi = H.OracleInputs(info)
	width, height = 160, 90
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=5, strategy=api.STRATEGY_DIFFUSE_ONLY, heuristic=api.MIS_BALANCE, technique=technique, trace_shadow_rays=1)
		constants = frame.constants(width, height)
		vis = oi.visibility(width, height, constants)
		gb = oi.gbuffer(width, height, constants, vis)
		out = frame.shade_host(width, height, gb)
		ref, _ = oi.shade(H.oracle_config(frame, width, height), constants, gb)
	finally:
		frame.close()
	cmp = H.compare_radiance(out, ref, rel=REL_TOL)
	assert cmp["bad_pixels"] == 0 and cmp["nan_mismatch"] == 0, cmp
	assert cmp["bit_exact"], cmp


def test_unsupported_combinations_are_rejected():
	"""The reference's interface offers the related-work techniques for diffuse-only sampling, and GGX MIS only where the density can be
	evaluated on its own (src/user_interface.cpp:124-175); create_shading_pass mirrors that with an error return."""
	info = H.dataset("mini_city")
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=1, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_BALANCE, technique=api.TECHNIQUE_SOLID_ANGLE)
		with pytest.raises(RuntimeError):
			frame.shade_host(32, 16, np.zeros((4, 16, 32, 4), dtype=np.float32))
		frame.configure(strategy=api.STRATEGY_DIFFUSE_GGX_MIS, technique=api.TECHNIQUE_AREA_TURK)
		with pytest.raises(RuntimeError):
			frame.shade_host(32, 16, np.zeros((4, 16, 32, 4), dtype=np.float32))
	finally:
		frame.close()
