"""Averaging frames on the device and measuring their error (vkr_accumulator_t, vkr_compare_frames; vulkan_renderer_b200.convergence).

1. The kernels against the host build of vkr_accumulate.cuh (tests/accumulate_on_host.cpp) bit for bit: accumulate, resolve, mean variance, and every
   metric; the same call twice gives the same bits; a frame against itself gives zeros; copies of one frame resolve to it with variance 0.
2. Fixed noise (animate_noise = 0): frames of the Cornell box are identical, so their mean is the frame and their variance 0.
3. Animated noise: consecutive frames differ, and two fresh Frames that accumulate the same number of frames give the same mean bit for bit.
4. Convergence: the mean of n animated 1-spp frames approaches a reference of 256 frames at 16 spp like 1/n, and the error of one frame is the
   per-frame variance.
5. Projected solid angle sampling (technique 11) has less variance per frame than Turk's area sampling (technique 1) on the Cornell box.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import harness as H
from tests.test_accumulate_on_host import error_tuple, host_accumulate, host_compare
from vulkan_renderer_b200 import api, convergence

pytestmark = pytest.mark.gpu

WIDTH, HEIGHT = 128, 96


@pytest.fixture(scope="module")
def device():
	lib = api.load_library(); dev = api.Device()
	assert lib.vkr_create_device(C.byref(dev), 0, None) == 0
	yield lib, dev
	lib.vkr_destroy_device(C.byref(dev))


def _seeded_frames(seed, count, height, width):
	g = torch.Generator().manual_seed(seed)
	scale = torch.pow(10.0, torch.empty((height, width, 1), dtype=torch.float64).uniform_(-40.0, 30.0, generator=g))
	frames = (scale[None] * torch.rand((count, height, width, 4), dtype=torch.float64, generator=g) * 2.0).to(torch.float32)
	frames[:, torch.rand((height, width), generator=g) < 0.05] = 0.0
	frames[..., 3] = 1.0
	return frames


def _device_accumulate(lib, dev, frames):
	"""frames [F, H, W, 4] -> (mean, variance or None, mean variance or None) through the C-ABI"""
	count, height, width = frames.shape[:3]
	d_frames = frames.cuda(); mean = torch.empty((height, width, 4), dtype=torch.float32, device="cuda"); var = torch.empty_like(mean)
	torch.cuda.synchronize()
	acc = api.Accumulator()
	assert lib.vkr_create_accumulator(C.byref(acc), C.byref(dev), width, height) == 0
	try:
		for f in range(count):
			assert lib.vkr_accumulate_frame(C.byref(acc), C.byref(dev), d_frames[f].data_ptr()) == 0
		assert acc.frame_count == count
		mv = None
		if count >= 2:
			assert lib.vkr_accumulator_resolve(C.byref(acc), C.byref(dev), mean.data_ptr(), var.data_ptr()) == 0
			mv = np.zeros(3, dtype=np.float64)
			assert lib.vkr_accumulator_mean_variance(C.byref(acc), C.byref(dev), mv.ctypes.data_as(C.POINTER(C.c_double))) == 0
		else:
			assert lib.vkr_accumulator_resolve(C.byref(acc), C.byref(dev), mean.data_ptr(), None) == 0
		assert lib.vkr_device_wait_idle(C.byref(dev)) == 0
	finally:
		lib.vkr_destroy_accumulator(C.byref(acc), C.byref(dev))
	return mean.cpu().numpy(), (var.cpu().numpy() if count >= 2 else None), mv


def _device_compare(lib, dev, frame, reference):
	height, width = frame.shape[:2]
	a = torch.as_tensor(frame).cuda(); b = torch.as_tensor(reference).cuda()
	torch.cuda.synchronize()
	out = api.FrameError()
	assert lib.vkr_compare_frames(C.byref(dev), width, height, a.data_ptr(), b.data_ptr(), C.byref(out)) == 0
	return out


def _bits(a):
	return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("count,height,width", [(2, 96, 128), (7, 61, 83), (3, 1080, 1920)])
def test_accumulator_and_metrics_match_the_host_build_bit_for_bit(device, count, height, width):
	lib, dev = device
	frames = _seeded_frames(count * 1000 + width, count, height, width)
	mean, var, mv = _device_accumulate(lib, dev, frames)
	_, h_mean, h_var, h_mv = host_accumulate(frames.numpy())
	assert np.array_equal(_bits(mean), _bits(h_mean)) and np.array_equal(_bits(var), _bits(h_var))
	assert mv.view(np.uint64).tolist() == h_mv.view(np.uint64).tolist()
	for x, r in ((frames[0].numpy(), mean), (mean, frames[-1].numpy())):
		first = _device_compare(lib, dev, x, r)
		assert error_tuple(first) == error_tuple(_device_compare(lib, dev, x, r)) == error_tuple(host_compare(x, r))
		assert first.pixel_count == height * width and first.mse[0] > 0.0
	x = frames[0].numpy().copy(); x[0, 0, 1] = np.nan; x[1, 2, 0] = -np.inf
	assert error_tuple(_device_compare(lib, dev, x, mean)) == error_tuple(host_compare(x, mean))
	assert _device_compare(lib, dev, x, mean).nonfinite_pixels == 2
	assert error_tuple(_device_compare(lib, dev, frames[1].numpy(), frames[1].numpy())) == (0.0,) * 10 + (height * width, 0)


def test_copies_of_one_frame_resolve_to_it_with_zero_variance(device):
	lib, dev = device
	frame = _seeded_frames(11, 1, HEIGHT, WIDTH)
	mean, var, mv = _device_accumulate(lib, dev, frame.repeat(5, 1, 1, 1))
	assert np.array_equal(_bits(mean[..., :3]), _bits(frame[0, ..., :3].numpy())) and (mean[..., 3] == 1.0).all()
	assert (var == 0.0).all() and mv.tolist() == [0.0, 0.0, 0.0]


def test_reset_and_refusals(device, capfd):
	lib, dev = device
	frames = _seeded_frames(12, 3, 8, 16).cuda(); out = torch.empty((8, 16, 4), dtype=torch.float32, device="cuda")
	torch.cuda.synchronize()
	acc = api.Accumulator()
	assert lib.vkr_create_accumulator(C.byref(acc), C.byref(dev), 0, 8) == 1 and acc.d_state is None
	assert lib.vkr_create_accumulator(C.byref(acc), C.byref(dev), 16, 8) == 0
	try:
		assert lib.vkr_accumulator_resolve(C.byref(acc), C.byref(dev), out.data_ptr(), None) == 1          # no frame yet
		assert lib.vkr_accumulate_frame(C.byref(acc), C.byref(dev), None) == 1
		assert lib.vkr_accumulate_frame(C.byref(acc), C.byref(dev), frames[0].data_ptr()) == 0
		assert lib.vkr_accumulator_resolve(C.byref(acc), C.byref(dev), None, out.data_ptr()) == 1          # a variance needs 2 frames
		mv = (C.c_double * 3)()
		assert lib.vkr_accumulator_mean_variance(C.byref(acc), C.byref(dev), mv) == 1
		assert lib.vkr_accumulate_frame(C.byref(acc), C.byref(dev), frames[1].data_ptr()) == 0
		assert lib.vkr_accumulator_reset(C.byref(acc), C.byref(dev)) == 0 and acc.frame_count == 0
		assert lib.vkr_accumulate_frame(C.byref(acc), C.byref(dev), frames[2].data_ptr()) == 0
		assert lib.vkr_accumulator_resolve(C.byref(acc), C.byref(dev), out.data_ptr(), None) == 0
		assert lib.vkr_device_wait_idle(C.byref(dev)) == 0
		assert np.array_equal(_bits(out[..., :3].cpu().numpy()), _bits(frames[2, ..., :3].cpu().numpy()))   # the reset forgot frames 0 and 1
	finally:
		lib.vkr_destroy_accumulator(C.byref(acc), C.byref(dev))
	lib.vkr_destroy_accumulator(C.byref(acc), C.byref(dev))   # a zeroed struct
	e = api.FrameError()
	assert lib.vkr_compare_frames(C.byref(dev), 0, 8, out.data_ptr(), out.data_ptr(), C.byref(e)) == 1
	assert lib.vkr_compare_frames(C.byref(dev), 16, 8, None, out.data_ptr(), C.byref(e)) == 1
	assert "Failed" in capfd.readouterr().out


def _cornell(**settings):
	frame = H.open_frame(H.dataset("cornell"))
	frame.configure(**settings)
	return frame


MIS = dict(sample_count=1, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)


def test_fixed_noise_frames_average_to_the_frame():
	frame = _cornell(**MIS)
	try:
		assert frame.settings.animate_noise == 0
		acc = convergence.accumulate(frame, WIDTH, HEIGHT, 3, animate=False)
		_, gb = frame.gbuffer_host(WIDTH, HEIGHT)
		single = frame.shade_host(WIDTH, HEIGHT, gb)
	finally:
		frame.close()
	assert np.array_equal(_bits(acc.mean[..., :3]), _bits(single[..., :3])) and (acc.mean[..., :3] > 0).any()
	assert (acc.variance == 0.0).all() and acc.mean_variance.tolist() == [0.0, 0.0, 0.0]
	assert acc.accumulate_ms_per_frame > 0.0


def test_animated_noise_differs_per_frame_and_is_deterministic():
	means = []
	for _ in range(2):
		frame = _cornell(**MIS)
		try:
			acc = convergence.accumulate(frame, WIDTH, HEIGHT, 8, animate=True)
			assert frame.settings.animate_noise == 0       # restored
		finally:
			frame.close()
		assert (acc.variance[..., :3] > 0).mean() > 0.1 and (acc.mean_variance > 0).all()
		means.append(acc.mean)
	assert np.array_equal(_bits(means[0]), _bits(means[1]))
	frame = _cornell(**MIS)
	try:
		with pytest.raises(ValueError):
			convergence.accumulate(frame.configure(output_srgb=1), WIDTH, HEIGHT, 2)
	finally:
		frame.close()


def test_the_mean_of_animated_frames_converges_to_the_reference():
	frame = _cornell(**dict(MIS, sample_count=16))
	try:
		frame.noise.random_seed += 1000003    # random numbers of its own, not those of the frames under test
		reference = convergence.accumulate(frame, WIDTH, HEIGHT, 256, animate=True).mean
	finally:
		frame.close()
	frame = _cornell(**MIS)
	try:
		mse = {}
		for n in (1, 4, 16):
			mse[n] = float(np.mean(convergence.frame_error(frame, convergence.accumulate(frame, WIDTH, HEIGHT, n, animate=True).mean, reference)["mse"]))
		noise = float(np.mean(convergence.accumulate(frame, WIDTH, HEIGHT, 16, animate=True).mean_variance))
	finally:
		frame.close()
	print("MSE of the mean of n frames against 256 x 16 spp: %s; mean variance per frame %.4e" % (mse, noise))
	assert mse[1] > mse[4] > mse[16] > 0.0
	assert 1.0 / 32.0 <= mse[16] / mse[1] <= 1.0 / 8.0
	assert 0.5 <= mse[1] / noise <= 2.0


def test_projected_solid_angle_sampling_has_less_variance_than_area_sampling():
	variance = {}
	for technique in (api.TECHNIQUE_AREA_TURK, api.TECHNIQUE_PSA):
		frame = _cornell(sample_count=1, strategy=api.STRATEGY_DIFFUSE_ONLY, technique=technique, trace_shadow_rays=1)
		try:
			variance[technique] = float(np.mean(convergence.accumulate(frame, WIDTH, HEIGHT, 32, animate=True).mean_variance))
		finally:
			frame.close()
	print("mean variance per frame: area (Turk) %.4e, projected solid angle %.4e" % (variance[api.TECHNIQUE_AREA_TURK], variance[api.TECHNIQUE_PSA]))
	assert variance[api.TECHNIQUE_PSA] < 0.8 * variance[api.TECHNIQUE_AREA_TURK]
