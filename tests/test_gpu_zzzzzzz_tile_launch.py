"""The dispatch of a frame to its tile kernel: one entry point per kernel family and light vertex bound (csrc/vkr_api.cu, vkr_tile_launch.cuh).
Small frames of the families and bounds no other test reaches -- textured lights with 3, 5, 6 and 7 vertices under projected solid angle sampling
and under a related-work technique, and the error display of hexagons -- against the oracle, bit for bit. A frame sent to the kernel of another
bound or family would differ. Placed last in the order."""
import numpy as np
import pytest

from tests import harness as H
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu

WIDTH, HEIGHT = 64, 32


def _shade_against_oracle(info, **settings):
	oi = H.OracleInputs(info)
	frame = H.open_frame(info)
	try:
		frame.configure(**settings)
		constants = frame.constants(WIDTH, HEIGHT)
		vis = oi.visibility(WIDTH, HEIGHT, constants); gb = oi.gbuffer(WIDTH, HEIGHT, constants, vis)
		out = frame.shade_host(WIDTH, HEIGHT, gb)
		ref, _ = oi.shade(H.oracle_config(frame, WIDTH, HEIGHT), constants, gb)
	finally:
		frame.close()
	assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), H.compare_radiance(out, ref)
	return out


@pytest.mark.parametrize("vertices", [3, 5, 6, 7])
def test_textured_polygons_under_projected_solid_angle_sampling(vertices):
	info = H.dataset("mini_lit", vertices=vertices)
	assert {len(l["vertices"]) for l in info["lights"]} == {vertices}
	out = _shade_against_oracle(info, sample_count=2, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, technique=api.TECHNIQUE_PSA,
		trace_shadow_rays=1, show_lights=1)
	assert (out[..., :3] > 0.0).any()


@pytest.mark.parametrize("vertices", [3, 5, 6, 7])
def test_textured_polygons_under_a_related_work_technique(vertices):
	info = H.dataset("mini_lit", vertices=vertices)
	out = _shade_against_oracle(info, sample_count=2, strategy=api.STRATEGY_DIFFUSE_GGX_MIS, heuristic=api.MIS_BALANCE, technique=api.TECHNIQUE_SOLID_ANGLE,
		trace_shadow_rays=1, show_lights=1)
	assert (out[..., :3] > 0.0).any()


def test_error_display_of_hexagons():
	out = _shade_against_oracle(H.dataset("mini_v6"), sample_count=1, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED,
		technique=api.TECHNIQUE_PSA, trace_shadow_rays=1, error_display=api.ERROR_DISPLAY_SPECULAR_BACKWARD)
	assert len(np.unique(out.reshape(-1, 4), axis=0)) > 4   # several error magnitudes on screen
