"""The GPU's shading pass against the float64 integral of the direct lighting: the cases, configurations, statistics and thresholds of
tests/test_estimator_float64.py (which justifies them), run through vkr_shading_pass_run on a synthetic G-buffer on the device, every light set with
every configuration, with shadow rays off and on (the trace warps' ray streams).
"""
import ctypes as C
import time

import numpy as np
import pytest

from tests import harness as H
from tests import test_estimator_float64 as E
from tests.test_float64_references import light_polygons
from vulkan_renderer_b200 import api
from vulkan_renderer_b200.noise_gen import LOADER_SEED

pytestmark = pytest.mark.gpu

BLOCK = 64
FRAMES = 384
SAMPLES = 4
RESOLUTION = 0.005
# 2048 x 2048 x 32 texels (1 GiB): 134 M texels against the 6.3 M a case reads (4096 pixels x 4 samples x 384 frames), so that the table's own
# quadrature error adds less than 5 % to the batch means' variance (test_estimator_float64's docstring)
NOISE = (2048, 2048, 32)
_table = []


def open_frame(info):
	"""A Frame whose noise table holds independent uniform texels (the same table for every light set), with animated noise and exposure 1."""
	if not _table:
		_table.append(np.ascontiguousarray(E.uniform_noise_table(NOISE)))
	frame = H.open_frame(info, noise=(64, 64, 1))
	frame.lib.vkr_destroy_noise_table(C.byref(frame.noise), C.byref(frame.device))
	assert frame.lib.vkr_noise_table_from_image(C.byref(frame.noise), C.byref(frame.device), NOISE[0], NOISE[1], NOISE[2], _table[0].ctypes.data, LOADER_SEED) == 0
	frame.settings.animate_noise = 1
	frame.settings.exposure_factor = 1.0
	return frame


def run_gpu(frame, config, shadows, case_list, frames=FRAMES, samples=SAMPLES, block=BLOCK, constants_list=None):
	"""Per-frame block means [frames, cases, 3] (float64, reduced on the device) and the last frame's constant block. constants_list: the frames'
	constant blocks, instead of the frame's next ones."""
	import torch
	strategy, heuristic, visibility = config
	frame.configure(sample_count=samples, strategy=strategy, heuristic=heuristic, technique=api.TECHNIQUE_PSA, trace_shadow_rays=int(shadows), show_lights=0)
	frame.settings.mis_visibility_estimate = visibility
	gb = E.synthetic_gbuffer(case_list, block)
	height, width = gb.shape[1:3]
	rows, columns = height // block, width // block
	dev = torch.device("cuda", frame.device.cuda_device)
	gbd = torch.from_numpy(gb).to(dev)
	out = torch.zeros((height, width, 4), dtype=torch.float32, device=dev)
	means = torch.zeros((frames, rows * columns, 3), dtype=torch.float64, device=dev)
	p = frame.create_pass(width, height)
	try:
		for f in range(frames):
			constants = frame.constants(width, height) if constants_list is None else constants_list[f]
			torch.cuda.synchronize()   # torch's stream is not the library's: the last reduction has read `out`
			assert frame.lib.vkr_shading_pass_run(C.byref(p), C.byref(frame.device), constants, len(constants), gbd.data_ptr(), out.data_ptr()) == 0
			assert frame.lib.vkr_shading_pass_wait(C.byref(p), C.byref(frame.device)) == 0
			means[f] = out[..., :3].to(torch.float64).reshape(rows, block, columns, block, 3).mean(dim=(1, 3)).reshape(-1, 3)
		torch.cuda.synchronize()
	finally:
		frame.destroy_pass(p)
	return means[:, :len(case_list)].cpu().numpy(), constants


def run_all(record=None):
	"""Every light set x configuration x shadows off / on; returns the failures. record: a list that receives (name, means, expected)."""
	import torch
	infos = E.dataset()
	oi = H.OracleInputs(infos["v4"])
	occluders = oi.shadow_tris.reshape(-1, 3, 3)
	start = time.time(); shading = 0.0
	failures = []; checked = 0
	truths = {}
	for light_set in E.LIGHT_SETS:
		frame = open_frame(infos[light_set])
		try:
			polygon = light_polygons(frame.constants(8, 8), frame.light_count)[0]
			case_list = E.cases(polygon)
			for config in E.CONFIGURATIONS:
				for shadows in (False, True):
					t0 = time.time()
					means, constants = run_gpu(frame, config, shadows, case_list)
					shading += time.time() - t0
					key = (light_set, shadows, config[0] == api.STRATEGY_DIFFUSE_SPECULAR_SEPARATELY)
					if key not in truths:
						truths[key] = E.truth(case_list, constants, frame.light_count, occluders if shadows else (), config[0], oi.ltc0, oi.ltc1)
					name = "%s %s shadows %d" % (E.config_name(config), light_set, shadows)
					if record is not None:
						record.append((name, means, truths[key]))
					try:
						E.check(name, case_list, means, truths[key], RESOLUTION)
					except AssertionError as e:
						failures.append(str(e))
					checked += 1
		finally:
			frame.close()
	print("GPU leg on %s: %d runs of %d frames, %.1f s (shading and reductions %.1f s)" % (torch.cuda.get_device_name(0), checked, FRAMES, time.time() - start, shading))
	return failures


def test_gpu_estimators_converge_to_the_float64_integral():
	failures = run_all()
	assert not failures, "\n".join(failures)


def test_gpu_clamped_optimal_at_visibility_one_is_the_weighted_heuristic():
	"""At visibility estimate 1 the clamped optimal weight fma(1, w_own / sum, fma(-1, balance, balance)) is w_own / sum: the weighted heuristic.
	On the same frames (same noise offsets), with shadow rays, the two configurations agree to rounding."""
	infos = E.dataset()
	frame = open_frame(infos["mixed"])
	try:
		case_list = E.cases(light_polygons(frame.constants(8, 8), frame.light_count)[0])
		frame.settings.mis_visibility_estimate = 1.0
		gb_shape = E.synthetic_gbuffer(case_list, BLOCK).shape
		constants_list = [frame.constants(gb_shape[2], gb_shape[1]) for _ in range(64)]
		weighted, _ = run_gpu(frame, (api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_WEIGHTED, 1.0), True, case_list, frames=64, constants_list=constants_list)
		clamped, _ = run_gpu(frame, (api.STRATEGY_DIFFUSE_SPECULAR_MIS, api.MIS_OPTIMAL_CLAMPED, 1.0), True, case_list, frames=64, constants_list=constants_list)
		difference = np.abs(weighted - clamped).max() / np.abs(weighted).max()
		print("clamped optimal at visibility 1 against weighted, same 64 frames: largest difference %.2e of the brightest block mean" % difference)
		assert np.isfinite(weighted).all() and difference <= 1e-5
	finally:
		frame.close()
