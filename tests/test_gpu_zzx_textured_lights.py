"""Textured polygonal lights on the GPU (get_polygon_radiance, shading_pass.frag.glsl:151-185: area texture, portal onto a light probe, IES profile):
textured_light_kernel (csrc/vkr_textured_light_kernel.cu) against frames of the REFERENCE's own shader sources fed with the same textures (fixtures
"_y1", tests/test_ref_shader.py) -- bit-identical -- and against the oracle on a larger frame. The per-pixel code underneath is also run on the CPU
(tests/test_device_on_host.py). Placed late in the order."""
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
	return sorted({k.split("/")[0] for k in g.files if "_y1" in k.split("/")[0]})   # incl. "_q4_y1": a related-work technique (vkr_textured_related_work_kernel.cu)


@pytest.mark.parametrize("name", _fixture_names())
def test_textured_lights_reproduce_reference_shader_fixture(name):
	from tests.test_ref_shader import _config_from_name
	from tests.ref_frames import WIDTH, HEIGHT, dataset_for
	g = np.load(GOLDEN)
	cfg = _config_from_name(name)
	info = H.dataset(dataset_for(cfg))
	frame = H.open_frame(info)
	try:
		assert frame.light_textures.texture_count == 3
		technique = cfg["technique"] if cfg["technique"] != api.TECHNIQUE_PSA else (api.TECHNIQUE_PSA_BIASED if cfg["biased"] else api.TECHNIQUE_PSA)
		frame.configure(sample_count=cfg["samples"], strategy=cfg["strategy"], heuristic=cfg["heuristic"], technique=technique,
			trace_shadow_rays=cfg["trace"], show_lights=cfg["show_lights"], light_count=cfg["lights"])
		constants = frame.constants(WIDTH, HEIGHT)
		assert constants == bytes(g[name + "/constants"])
		vis, gb = frame.gbuffer_host(WIDTH, HEIGHT)
		out = frame.shade_host(WIDTH, HEIGHT, gb)
	finally:
		frame.close()
	assert_matches_fixture(g, name, out)


@pytest.mark.parametrize("technique", [api.TECHNIQUE_PSA, api.TECHNIQUE_PSA_BIASED])
def test_textured_lights_match_the_oracle_on_a_larger_frame(technique):
	info = H.dataset("mini_lit"); oi = H.OracleInputs(info)
	width, height = 240, 136
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=4, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, technique=technique, trace_shadow_rays=1, show_lights=1)
		constants = frame.constants(width, height)
		vis = oi.visibility(width, height, constants); gb = oi.gbuffer(width, height, constants, vis)
		out = frame.shade_host(width, height, gb)
		ref, _ = oi.shade(H.oracle_config(frame, width, height), constants, gb)
	finally:
		frame.close()
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)


@pytest.mark.parametrize("technique,strategy", [(api.TECHNIQUE_AREA_TURK, api.STRATEGY_DIFFUSE_ONLY), (api.TECHNIQUE_RECTANGLE_SOLID_ANGLE_URENA, api.STRATEGY_DIFFUSE_GGX_MIS),
	(api.TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO, api.STRATEGY_DIFFUSE_GGX_MIS)])
def test_related_work_techniques_under_textured_lights_match_the_oracle(technique, strategy):
	info = H.dataset("mini_lit"); oi = H.OracleInputs(info)
	width, height = 160, 90
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=2, strategy=strategy, heuristic=api.MIS_BALANCE, technique=technique, trace_shadow_rays=1, show_lights=1)
		constants = frame.constants(width, height)
		vis = oi.visibility(width, height, constants); gb = oi.gbuffer(width, height, constants, vis)
		out = frame.shade_host(width, height, gb)
		ref, _ = oi.shade(H.oracle_config(frame, width, height), constants, gb)
	finally:
		frame.close()
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)


def test_the_error_display_refuses_textured_lights():
	"""The error display shows no radiance and has no textured variant: the pass says so instead of ignoring the textures silently."""
	info = H.dataset("mini_lit"); oi = H.OracleInputs(info)
	width, height = 64, 48
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=1, strategy=api.STRATEGY_DIFFUSE_ONLY, heuristic=api.MIS_BALANCE, technique=api.TECHNIQUE_PSA, trace_shadow_rays=0, error_display=api.ERROR_DISPLAY_DIFFUSE_BACKWARD)
		constants = frame.constants(width, height)
		vis = oi.visibility(width, height, constants); gb = oi.gbuffer(width, height, constants, vis)
		with pytest.raises(RuntimeError):
			frame.shade_host(width, height, gb)
	finally:
		frame.close()


def test_textured_light_figures_of_the_experiment_list_run(tmp_path):
	"""The IES-profile attic and the textured screen over the roughness planes (src/experiment_list.c:294-314, 341-362) through the experiment runner, small."""
	from vulkan_renderer_b200 import experiments as E
	todo = [dict(e) for e in E.experiment_list(all_timings=False) if e["name"] in ("ies_profile_attic_2spp", "roughness_planes_screen_2spp")]
	assert len(todo) == 2
	for e in todo:
		if e["scene"] == "room": e["scene_parameters"] = dict(e["scene_parameters"], detail=6, clutter=60, n_mat=8)   # the same room with few triangles
	records = E.run(todo, str(tmp_path / "data"), str(tmp_path / "out"), frames=3, warmup=1, width=160, height=128)
	for r in records:
		assert r["frame_time_ms"] > 0.0 and os.path.exists(r["screenshot"]) and os.path.getsize(r["screenshot"]) > 1000
