"""The accumulator's arithmetic and the frame metrics (vulkan_renderer_b200/csrc/vkr_accumulate.cuh) compiled for the CPU (tests/accumulate_on_host.cpp,
the kernels' loops as plain loops in the same order), against numpy float64: Welford's running mean and variance against the two-pass mean and the
ddof = 1 variance, and every metric of vkr_frame_error_t against its definition, on seeded frames with magnitudes from float subnormals to 1e30,
zeros, and NaN / +-inf injected. The -m gpu tests then hold the kernels against this build bit for bit (tests/test_gpu_zzzzzz_convergence.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from vulkan_renderer_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libaccumulate_on_host.so")
REL = 1.0e-12


def host_lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	lib = C.CDLL(LIB_PATH)
	lib.vkr_host_accumulate.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]; lib.vkr_host_accumulate.restype = None
	lib.vkr_host_resolve.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]; lib.vkr_host_resolve.restype = None
	lib.vkr_host_mean_variance.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]; lib.vkr_host_mean_variance.restype = None
	lib.vkr_host_compare.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(api.FrameError)]; lib.vkr_host_compare.restype = None
	return lib


def host_accumulate(frames):
	"""frames [F, H, W, 4] float32 -> (state [6, H*W] float64, mean [H, W, 4] float32, variance [H, W, 4] float32 or None, mean variance [3] or None)"""
	lib = host_lib()
	frames = np.ascontiguousarray(frames, dtype=np.float32)
	count, pixels = frames.shape[0], frames.shape[1] * frames.shape[2]
	state = np.zeros((6, pixels), dtype=np.float64)
	lib.vkr_host_accumulate(pixels, count, frames.ctypes.data, state.ctypes.data)
	mean = np.zeros(frames.shape[1:], dtype=np.float32)
	variance = np.zeros(frames.shape[1:], dtype=np.float32) if count >= 2 else None
	lib.vkr_host_resolve(pixels, count, state.ctypes.data, mean.ctypes.data, variance.ctypes.data if variance is not None else None)
	mean_variance = None
	if count >= 2:
		mean_variance = np.zeros(3, dtype=np.float64)
		lib.vkr_host_mean_variance(pixels, count, state.ctypes.data, mean_variance.ctypes.data)
	return state, mean, variance, mean_variance


def host_compare(frame, reference):
	lib = host_lib()
	frame = np.ascontiguousarray(frame, dtype=np.float32); reference = np.ascontiguousarray(reference, dtype=np.float32)
	assert frame.shape == reference.shape
	out = api.FrameError()
	lib.vkr_host_compare(frame.shape[0] * frame.shape[1], frame.ctypes.data, reference.ctypes.data, C.byref(out))
	return out


def error_tuple(e):
	"""vkr_frame_error_t as a tuple of Python numbers (for bit-exact comparisons)"""
	return tuple(e.mse) + tuple(e.rel_mse) + tuple(e.mae) + (e.max_abs_error, e.pixel_count, e.nonfinite_pixels)


def numpy_error(frame, reference):
	x = np.asarray(frame, dtype=np.float64)[..., :3].reshape(-1, 3); r = np.asarray(reference, dtype=np.float64)[..., :3].reshape(-1, 3)
	ok = np.isfinite(x).all(1) & np.isfinite(r).all(1)
	d = x[ok] - r[ok]; n = int(ok.sum())
	return dict(mse=(d * d).sum(0) / n, rel_mse=(d * d / (r[ok] * r[ok] + 0.01)).sum(0) / n, mae=np.abs(d).sum(0) / n,
		max_abs_error=float(np.abs(d).max()) if n else 0.0, pixel_count=n, nonfinite_pixels=int((~ok).sum()))


def seeded_frames(seed, count, height, width, nonfinite=True):
	"""Non-negative radiance-like frames: per pixel a scale 10^U(-44, 30) (float subnormals up to 1e30), per frame a factor U(0, 2); some pixels zero
	in every frame, some zero in single frames; optionally NaN / +inf / -inf injected into single channels."""
	rng = np.random.default_rng(seed)
	scale = 10.0 ** rng.uniform(-44.0, 30.0, (height, width, 1))
	frames = scale[None] * rng.uniform(0.0, 2.0, (count, height, width, 4))
	frames[:, rng.random((height, width)) < 0.05] = 0.0
	frames[rng.random((count, height, width)) < 0.02] = 0.0
	frames = frames.astype(np.float32)
	frames[..., 3] = 1.0
	if nonfinite:
		for value in (np.nan, np.inf, -np.inf):
			hit = rng.random((count, height, width)) < 0.003
			frames[hit, rng.integers(0, 3)] = value
	return frames


def _close(a, b, rel=REL):
	a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
	return np.abs(a - b) <= rel * np.abs(b)


@pytest.mark.parametrize("seed,count", [(1, 2), (2, 5), (3, 16)])
def test_welford_state_matches_two_pass_float64(seed, count):
	frames = seeded_frames(seed, count, 37, 53)
	state, mean, variance, mean_variance = host_accumulate(frames)
	x = frames[..., :3].astype(np.float64).reshape(count, -1, 3)
	finite = np.isfinite(x).all(axis=0)                    # [pixels, 3]: the channel's whole sequence is finite
	ref_mean = x.mean(axis=0); ref_var = x.var(axis=0, ddof=1)
	got_mean = state[:3].T; got_var = state[3:].T / (count - 1)
	assert finite.mean() > 0.8 and (~finite).any()
	assert _close(got_mean[finite], ref_mean[finite]).all()
	assert _close(got_var[finite], ref_var[finite]).all()
	assert (ref_var[finite] > 0).mean() > 0.9 and (got_var[finite] < 1e-300).sum() == (ref_var[finite] == 0).sum()
	# a non-finite sample leaves the channel non-finite (NaN or inf), never a finite number
	assert not (np.isfinite(got_mean[~finite]) & np.isfinite(got_var[~finite])).any()
	# resolve = the state rounded to float; alpha 1 / 0
	assert np.array_equal(mean[..., :3].reshape(-1, 3), got_mean.astype(np.float32), equal_nan=True) and (mean[..., 3] == 1.0).all()
	assert np.array_equal(variance[..., :3].reshape(-1, 3), got_var.astype(np.float32), equal_nan=True) and (variance[..., 3] == 0.0).all()
	# the mean variance: the mean over all pixels of m2 / (n - 1); with non-finite pixels it is not finite, on the finite pixels it is numpy's
	assert not np.isfinite(mean_variance).all()
	_, _, _, mv_finite = host_accumulate(np.where(np.isfinite(frames), frames, np.float32(0.5)))
	x0 = np.where(np.isfinite(x), x, 0.5)
	assert _close(mv_finite, x0.var(axis=0, ddof=1).mean(axis=0)).all()


@pytest.mark.parametrize("seed", [4, 5, 6])
def test_frame_metrics_match_their_float64_definitions(seed):
	frames = seeded_frames(seed, 2, 61, 47)
	frame, reference = frames[0], frames[1]
	got = host_compare(frame, reference)
	ref = numpy_error(frame, reference)
	assert got.nonfinite_pixels == ref["nonfinite_pixels"] > 0 and got.pixel_count == ref["pixel_count"] == 61 * 47 - ref["nonfinite_pixels"]
	for key in ("mse", "rel_mse", "mae"):
		assert _close(list(getattr(got, key)), ref[key]).all(), key
	assert got.max_abs_error == ref["max_abs_error"]
	assert error_tuple(host_compare(frame, reference)) == error_tuple(got)
	# a reference close to the frame: small differences, still every metric to 1e-12
	near = (reference * np.float32(1.0 + 1e-3)).astype(np.float32)
	got = host_compare(reference, near); ref = numpy_error(reference, near)
	for key in ("mse", "rel_mse", "mae"):
		assert _close(list(getattr(got, key)), ref[key]).all(), key


def test_metrics_on_a_larger_frame_span_every_partition():
	"""More pixels than 1024 blocks x 256 threads: every thread of every block sums several pixels."""
	rng = np.random.default_rng(7)
	frame = rng.uniform(0.0, 4.0, (720, 400, 4)).astype(np.float32); reference = rng.uniform(0.0, 4.0, (720, 400, 4)).astype(np.float32)
	frame[3, 5, 1] = np.inf
	got = host_compare(frame, reference); ref = numpy_error(frame, reference)
	assert (got.pixel_count, got.nonfinite_pixels) == (720 * 400 - 1, 1)
	for key in ("mse", "rel_mse", "mae"):
		assert _close(list(getattr(got, key)), ref[key]).all(), key
	assert got.max_abs_error == ref["max_abs_error"]


def test_identical_frames_give_their_value_and_zero_variance():
	frames = seeded_frames(8, 1, 29, 31, nonfinite=False)
	frames[0, 0, 0, :3] = -0.0
	five = np.repeat(frames, 5, axis=0)
	state, mean, variance, mean_variance = host_accumulate(five)
	assert np.array_equal(mean[..., :3].view(np.uint32), frames[0, ..., :3].view(np.uint32))
	assert (state[3:] == 0.0).all() and (variance == 0.0).all() and (mean_variance == 0.0).all()
	same = host_compare(frames[0], frames[0])
	assert error_tuple(same) == (0.0,) * 10 + (29 * 31, 0)


def test_no_finite_pixel_gives_nan_means():
	frame = np.full((2, 3, 4), np.nan, dtype=np.float32)
	got = host_compare(frame, frame)
	assert (got.pixel_count, got.nonfinite_pixels) == (0, 6) and np.isnan(got.mse[0]) and got.max_abs_error == 0.0
