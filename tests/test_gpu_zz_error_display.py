"""The error display modes of the shader on the GPU (ERROR_DISPLAY_DIFFUSE / ERROR_DISPLAY_SPECULAR, shading_pass.frag.glsl:462-493, 549-563):
error_display_kernel against frames of the REFERENCE's own shader sources compiled with those defines (fixtures "_e<error display>",
tests/test_ref_shader.py) -- bit-identical colour-coded errors. The device functions underneath are also held against the oracle on the
CPU (tests/test_device_on_host.py). (This file sorts last among the GPU tests: it is the newest code of the round.)"""
import os

import numpy as np
import pytest

from tests import harness as H
from tests.ref_frames import assert_matches_fixture
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shader.npz")


def _fixture_names():
	g = np.load(GOLDEN)
	return sorted({k.split("/")[0] for k in g.files if "_e" in k.split("/")[0]})


@pytest.mark.parametrize("name", _fixture_names())
def test_error_display_reproduces_reference_shader_fixture(name):
	from tests.test_ref_shader import _config_from_name
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	g = np.load(GOLDEN)
	cfg = _config_from_name(name)
	assert cfg["error_display"] != 0
	info = H.dataset(dataset_for(cfg))
	frame = H.open_frame(info)
	try:
		technique = cfg["technique"] if cfg["technique"] != api.TECHNIQUE_PSA else (api.TECHNIQUE_PSA_BIASED if cfg["biased"] else api.TECHNIQUE_PSA)
		frame.configure(sample_count=cfg["samples"], strategy=cfg["strategy"], heuristic=cfg["heuristic"], technique=technique,
			trace_shadow_rays=cfg["trace"], show_lights=cfg["show_lights"], light_count=cfg["lights"], error_display=cfg["error_display"])
		constants = frame.constants(WIDTH, HEIGHT)
		assert constants == bytes(g[name + "/constants"])
		vis, gb = frame.gbuffer_host(WIDTH, HEIGHT)
		out = frame.shade_host(WIDTH, HEIGHT, gb)
	finally:
		frame.close()
	assert_matches_fixture(g, name, out)
	assert len(np.unique(out.reshape(-1, 4), axis=0)) > 4       # several error magnitudes on screen


def test_error_display_follows_the_error_scale_and_matches_the_oracle():
	"""error_min_exponent moves the colour scale (g_error_factor = 10^-exponent, src/main.c:2127); a larger frame than the fixtures against the oracle."""
	info = H.dataset("mini_city"); oi = H.OracleInputs(info)
	width, height = 160, 90
	frames = []
	for exponent in (-7.0, -4.0):
		frame = H.open_frame(info)
		try:
			frame.settings.error_min_exponent = exponent
			frame.configure(sample_count=1, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, technique=api.TECHNIQUE_PSA, trace_shadow_rays=1,
				error_display=api.ERROR_DISPLAY_SPECULAR_BACKWARD)
			constants = frame.constants(width, height)
			vis = oi.visibility(width, height, constants); gb = oi.gbuffer(width, height, constants, vis)
			out = frame.shade_host(width, height, gb)
			ref, _ = oi.shade(H.oracle_config(frame, width, height), constants, gb)
		finally:
			frame.close()
		assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)
		frames.append(out)
	assert not np.array_equal(frames[0], frames[1])
