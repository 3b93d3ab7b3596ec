"""Material textures in the G-buffer producer on the GPU (SURVEY 8 row f1): gbuffer_kernel<true> -- screen-space derivatives, three textureGrad
per pixel over BC1 / RGBA16F / BC5 textures decoded at load time -- against (1) the frames of the REFERENCE's shader sources rendered with the same
textures (fixtures "_x1"; the filter definition is shared, oracle/texture_filter.h) and (2) the oracle's G-buffer on a larger frame. The filter
itself is held against its definition on the CPU (tests/test_device_on_host.py), the loader in tests/test_textures.py.
(Written after this round's GPU budget was spent: this file sorts last among the GPU tests.)"""
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
	return sorted({k.split("/")[0] for k in g.files if "_x1" in k.split("/")[0]})


@pytest.mark.parametrize("name", _fixture_names())
def test_textured_frame_reproduces_reference_shader_fixture(name):
	from tests.test_ref_shader import _config_from_name
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	g = np.load(GOLDEN)
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg))
	frame = H.open_frame(info)
	try:
		assert frame.scene.textured == 1 and frame.scene.texture_texel_count > 0
		frame.configure(sample_count=cfg["samples"], strategy=cfg["strategy"], heuristic=cfg["heuristic"], trace_shadow_rays=cfg["trace"], show_lights=cfg["show_lights"], light_count=cfg["lights"])
		constants = frame.constants(WIDTH, HEIGHT)
		assert constants == bytes(g[name + "/constants"])
		vis, gb = frame.gbuffer_host(WIDTH, HEIGHT)
		assert np.array_equal(vis, g[name + "/visibility"])
		out = frame.shade_host(WIDTH, HEIGHT, gb)
	finally:
		frame.close()
	assert_matches_fixture(g, name, out)


def test_textured_gbuffer_matches_the_oracle_and_differs_from_constant_materials():
	width, height = 200, 112
	info = H.dataset("mini_textured"); oi = H.OracleInputs(info)
	frame = H.open_frame(info)
	try:
		constants = frame.constants(width, height)
		vis, gb = frame.gbuffer_host(width, height)
	finally:
		frame.close()
	ref_vis = oi.visibility(width, height, constants)
	ref = oi.gbuffer(width, height, constants, ref_vis)
	assert np.array_equal(vis, ref_vis)
	assert np.array_equal(gb.view(np.uint32), ref.view(np.uint32))
	assert len(np.unique(ref[2].reshape(-1, 4), axis=0)) > 500           # albedo varies inside materials
	plain = H.open_frame(H.dataset("mini_city"))
	try:
		assert plain.scene.textured == 0 and not plain.scene.d_texture_data  # constant textures keep the one-texel path
	finally:
		plain.close()
