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


AdaptiveAccumulation = collections.namedtuple("AdaptiveAccumulation",
	"mean variance tile_frames estimated_rel_mse frames tile_frames_shaded tile_frames_full shade_ms accumulate_ms")
AdaptiveAccumulation.__doc__ = """mean, variance: as Accumulation, each pixel over its own tile's frames; tile_frames: [tiles_y, tiles_x] uint32, the frames
each 16x8 tile took; estimated_rel_mse: [3] float64, the mean over the pixels of the estimated variance of the mean over (mean^2 + 0.01); frames: frames
shaded before no tile was left (at most max_frames); tile_frames_shaded: tile launches, against tile_frames_full = tiles * max_frames for the plain
path; shade_ms, accumulate_ms: device time of the shading and accumulate launches over the whole run (CUDA events)."""


def accumulate_adaptive(frame, width, height, max_frames, target_rel_mse, min_frames=16, batch=8):
	"""Like accumulate(frame, width, height, max_frames) with animated noise, but a 16x8 tile stops being shaded and accumulated once its mean has
	converged (vkr_adaptive_accumulator_t): every `batch` frames the tile test stops the tiles with at least min_frames frames whose every pixel and
	channel has an estimated variance of the mean of at most target_rel_mse * (mean^2 + 0.01), and the tiles that reached max_frames. The remaining
	tiles are shaded in the pass's launch order (vkr_shading_pass_run_tiles). A tile's mean and variance are therefore those of the plain path after
	that tile's frame count. frame.constants() is called once per frame up to max_frames, also after the last tile stopped, so the seed sequence is
	the one accumulate() draws. Refuses what accumulate() refuses. Returns an AdaptiveAccumulation of numpy arrays."""
	import torch
	if getattr(frame, "output_srgb", 0) or getattr(frame, "frame_bits", 0) or getattr(frame, "error_display", 0):
		raise ValueError("only linear radiance can be accumulated: output_srgb, frame_bits and error_display must be 0")
	if not (2 <= min_frames <= max_frames) or batch < 1:
		raise ValueError("need 2 <= min_frames <= max_frames and batch >= 1, got %d, %d, %d" % (min_frames, max_frames, batch))
	if not (np.isfinite(target_rel_mse) and target_rel_mse >= 0.0):
		raise ValueError("the target relMSE must be finite and not negative, got %r" % target_rel_mse)
	lib = frame.lib; device = C.byref(frame.device)
	targets = api.RenderTargets(); acc = api.AdaptiveAccumulator(); p = None
	saved = frame.settings.animate_noise
	frame.settings.animate_noise = 1
	try:
		constants = frame.constants(width, height)
		_check(lib.vkr_create_render_targets(C.byref(targets), device, width, height), "vkr_create_render_targets")
		_check(lib.vkr_run_visibility_pass(device, C.byref(frame.scene), constants, width, height, targets.d_visibility), "vkr_run_visibility_pass")
		_check(lib.vkr_run_gbuffer_pass(device, C.byref(frame.scene), constants, width, height, targets.d_visibility, targets.d_gbuffer), "vkr_run_gbuffer_pass")
		p = frame.create_pass(width, height)
		_check(lib.vkr_create_adaptive_accumulator(C.byref(acc), device, width, height), "vkr_create_adaptive_accumulator")
		tiles_y, tiles_x = acc.tiles_y, acc.tiles_x
		order = np.ctypeslib.as_array((C.c_uint32 * p.tile_count).from_address(p.h_tile_list)).copy()   # the pass's launch order
		active = np.ones(tiles_y * tiles_x, dtype=np.uint8)
		todo = order
		stream = torch.cuda.ExternalStream(frame.device.stream, device=torch.device("cuda", frame.device.cuda_device))
		events = []
		shaded = frames = 0
		for i in range(max_frames):
			if i:
				constants = frame.constants(width, height)
			if not todo.size:
				continue
			e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
			e[0].record(stream)
			_check(lib.vkr_shading_pass_run_tiles(C.byref(p), device, constants, len(constants), targets.d_gbuffer, targets.d_frame, todo.ctypes.data, todo.size), "vkr_shading_pass_run_tiles")
			e[1].record(stream)
			_check(lib.vkr_adaptive_accumulate_frame(C.byref(acc), device, targets.d_frame), "vkr_adaptive_accumulate_frame")
			e[2].record(stream)
			events.append(e)
			shaded += int(todo.size); frames += 1
			if (i + 1) % batch == 0:
				_check(lib.vkr_adaptive_update_tiles(C.byref(acc), device, float(target_rel_mse), min_frames, max_frames, active.ctypes.data, None), "vkr_adaptive_update_tiles")
				todo = order[active[order] != 0]
		mean = np.zeros((height, width, 4), dtype=np.float32); variance = np.zeros_like(mean)
		_check(lib.vkr_adaptive_resolve(C.byref(acc), device, targets.d_frame, None), "vkr_adaptive_resolve")
		_check(lib.vkr_download_frame(C.byref(targets), device, mean.ctypes.data), "vkr_download_frame")
		_check(lib.vkr_adaptive_resolve(C.byref(acc), device, None, targets.d_frame), "vkr_adaptive_resolve")
		_check(lib.vkr_download_frame(C.byref(targets), device, variance.ctypes.data), "vkr_download_frame")
		estimate = np.zeros(3, dtype=np.float64)
		_check(lib.vkr_adaptive_estimated_rel_mse(C.byref(acc), device, estimate.ctypes.data_as(C.POINTER(C.c_double))), "vkr_adaptive_estimated_rel_mse")
		tile_frames = np.zeros((tiles_y, tiles_x), dtype=np.uint32)
		_check(lib.vkr_adaptive_tile_frames(C.byref(acc), device, tile_frames.ctypes.data), "vkr_adaptive_tile_frames")
		_check(lib.vkr_device_wait_idle(device), "vkr_device_wait_idle")
		shade_ms = sum(e[0].elapsed_time(e[1]) for e in events); accumulate_ms = sum(e[1].elapsed_time(e[2]) for e in events)
		return AdaptiveAccumulation(mean, variance, tile_frames, estimate, frames, shaded, tiles_y * tiles_x * max_frames, shade_ms, accumulate_ms)
	finally:
		frame.settings.animate_noise = saved
		lib.vkr_destroy_adaptive_accumulator(C.byref(acc), device)
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
