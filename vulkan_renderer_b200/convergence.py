"""Averaging frames on the device and measuring a frame's error against a converged reference (include/vkr_b200.h, vkr_accumulator_t, vkr_compare_frames).

The noise accessor of a pixel repeats after 128 texel fetches, so more samples per pixel in one frame soon stop adding independent random numbers.
Frames with animate_noise = 1 draw new random numbers each (vkr_set_noise_constants); their mean is how a converged image is made. Everything that
computes goes through libvkr_b200.so (float64 on the device, sums in a fixed order); there is no CPU fallback.
"""
import collections
import ctypes as C

import numpy as np

from . import api

Accumulation = collections.namedtuple("Accumulation", "mean variance mean_variance accumulate_ms_per_frame")
Accumulation.__doc__ = """mean: [H, W, 4] float32 (alpha 1); variance: per-frame sample variance [H, W, 4] float32 (alpha 0), None for one frame;
mean_variance: [3] float64 (the mean of the variance over the pixels), None for one frame; accumulate_ms_per_frame: the accumulate kernel's mean
device time (CUDA events)."""


def _check(code, what):
	if code != 0:
		raise RuntimeError("%s failed with code %d" % (what, code))


def accumulate(frame, width, height, frames, animate=True):
	"""Renders `frames` frames of a vulkan_renderer_b200.Frame with its current settings through one shading pass on device buffers and averages
	them on the device. animate = True sets animate_noise = 1 while it runs, so every constant block draws new random numbers (the seed sequence
	of the noise table goes on from where it is); animate = False renders the same frame every time. Returns an Accumulation of numpy arrays.
	Refuses what is not linear radiance: sRGB output, half-bit screenshot frames and the error display."""
	import torch
	if getattr(frame, "output_srgb", 0) or getattr(frame, "frame_bits", 0) or getattr(frame, "error_display", 0):
		raise ValueError("only linear radiance can be accumulated: output_srgb, frame_bits and error_display must be 0")
	if frames < 1:
		raise ValueError("at least one frame is needed")
	lib = frame.lib; device = C.byref(frame.device)
	targets = api.RenderTargets(); acc = api.Accumulator(); p = None
	saved = frame.settings.animate_noise
	frame.settings.animate_noise = int(animate)
	try:
		constants = frame.constants(width, height)
		_check(lib.vkr_create_render_targets(C.byref(targets), device, width, height), "vkr_create_render_targets")
		_check(lib.vkr_run_visibility_pass(device, C.byref(frame.scene), constants, width, height, targets.d_visibility), "vkr_run_visibility_pass")
		_check(lib.vkr_run_gbuffer_pass(device, C.byref(frame.scene), constants, width, height, targets.d_visibility, targets.d_gbuffer), "vkr_run_gbuffer_pass")
		p = frame.create_pass(width, height)
		_check(lib.vkr_create_accumulator(C.byref(acc), device, width, height), "vkr_create_accumulator")
		stream = torch.cuda.ExternalStream(frame.device.stream, device=torch.device("cuda", frame.device.cuda_device))
		events = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(frames)]
		for i in range(frames):
			if i:
				constants = frame.constants(width, height)
			_check(lib.vkr_shading_pass_run(C.byref(p), device, constants, len(constants), targets.d_gbuffer, targets.d_frame), "vkr_shading_pass_run")
			events[i][0].record(stream)
			_check(lib.vkr_accumulate_frame(C.byref(acc), device, targets.d_frame), "vkr_accumulate_frame")
			events[i][1].record(stream)
		# the frame target is free once the last frame is accumulated (stream order): the resolved images go through it to the host
		mean = np.zeros((height, width, 4), dtype=np.float32)
		_check(lib.vkr_accumulator_resolve(C.byref(acc), device, targets.d_frame, None), "vkr_accumulator_resolve")
		_check(lib.vkr_download_frame(C.byref(targets), device, mean.ctypes.data), "vkr_download_frame")
		variance = mean_variance = None
		if frames >= 2:
			variance = np.zeros((height, width, 4), dtype=np.float32)
			_check(lib.vkr_accumulator_resolve(C.byref(acc), device, None, targets.d_frame), "vkr_accumulator_resolve")
			_check(lib.vkr_download_frame(C.byref(targets), device, variance.ctypes.data), "vkr_download_frame")
			mean_variance = np.zeros(3, dtype=np.float64)
			_check(lib.vkr_accumulator_mean_variance(C.byref(acc), device, mean_variance.ctypes.data_as(C.POINTER(C.c_double))), "vkr_accumulator_mean_variance")
		_check(lib.vkr_device_wait_idle(device), "vkr_device_wait_idle")
		ms = sum(begin.elapsed_time(end) for begin, end in events) / frames
		return Accumulation(mean, variance, mean_variance, ms)
	finally:
		frame.settings.animate_noise = saved
		lib.vkr_destroy_accumulator(C.byref(acc), device)
		if p is not None:
			frame.destroy_pass(p)
		lib.vkr_destroy_render_targets(C.byref(targets), device)


def frame_error(frame, test, reference):
	"""vkr_compare_frames on the device of a vulkan_renderer_b200.Frame: test and reference are [H, W, 4] float32 arrays (numpy, or torch tensors on
	that device). Returns a dict of mse, rel_mse, mae (per channel), max_abs_error, pixel_count and nonfinite_pixels."""
	import torch
	dev = torch.device("cuda", frame.device.cuda_device)
	def on_device(x):
		if not torch.is_tensor(x):
			x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
		return x.to(dev, torch.float32).contiguous()
	t, r = on_device(test), on_device(reference)
	if t.shape != r.shape or t.dim() != 3 or t.shape[2] != 4:
		raise ValueError("frames must be [H, W, 4] of one shape, got %s and %s" % (tuple(t.shape), tuple(r.shape)))
	torch.cuda.synchronize(dev)   # the library works on its own stream
	out = api.FrameError()
	_check(frame.lib.vkr_compare_frames(C.byref(frame.device), t.shape[1], t.shape[0], t.data_ptr(), r.data_ptr(), C.byref(out)), "vkr_compare_frames")
	return error_dict(out)


def error_dict(e):
	return dict(mse=list(e.mse), rel_mse=list(e.rel_mse), mae=list(e.mae), max_abs_error=e.max_abs_error, pixel_count=int(e.pixel_count), nonfinite_pixels=int(e.nonfinite_pixels))
