"""The adaptive accumulator's arithmetic (vulkan_renderer_b200/csrc/vkr_accumulate.cuh) compiled for the CPU (tests/adaptive_on_host.cpp, the kernels'
loops as plain loops in the same order), against numpy float64 on seeded frame sequences and seeded patterns of active tiles, on frames that are not a
multiple of the 16x8 tile: the masked Welford state and every tile decision are exactly numpy's, the estimated relMSE agrees to 1e-12, and with every
tile active the state is the plain accumulator's (tests/accumulate_on_host.cpp) bit for bit. The -m gpu tests then hold the kernels against this build
bit for bit (tests/test_gpu_zzzzzzzzzzz_adaptive_convergence.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.test_accumulate_on_host import host_accumulate, seeded_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libadaptive_on_host.so")
TILE_W, TILE_H = 16, 8
EPS = 0.01   # the relMSE epsilon of vkr_compare_frames


def host_lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	lib = C.CDLL(LIB_PATH)
	P = C.c_void_p
	lib.vkr_host_adaptive_accumulate.argtypes = [C.c_uint32, C.c_uint32, P, P, P, P]; lib.vkr_host_adaptive_accumulate.restype = None
	lib.vkr_host_adaptive_update.argtypes = [C.c_uint32, C.c_uint32, P, P, P, C.c_double, C.c_uint32, C.c_uint32]; lib.vkr_host_adaptive_update.restype = None
	lib.vkr_host_adaptive_resolve.argtypes = [C.c_uint32, C.c_uint32, P, P, P, P]; lib.vkr_host_adaptive_resolve.restype = None
	lib.vkr_host_adaptive_estimate.argtypes = [C.c_uint32, C.c_uint32, P, P, P]; lib.vkr_host_adaptive_estimate.restype = None
	return lib


def tile_grid(width, height):
	return (height + TILE_H - 1) // TILE_H, (width + TILE_W - 1) // TILE_W


def pixel_tiles(width, height):
	"""[H * W] tile index of every pixel"""
	ys, xs = np.mgrid[0:height, 0:width]
	return ((ys // TILE_H) * tile_grid(width, height)[1] + xs // TILE_W).reshape(-1)


class HostAdaptive:
	"""The host build's state: state [6, H*W] float64, tile_frames [tiles] uint32, active [tiles] uint8."""

	def __init__(self, width, height):
		self.lib = host_lib(); self.width, self.height = width, height
		tiles = int(np.prod(tile_grid(width, height)))
		self.state = np.zeros((6, width * height), dtype=np.float64)
		self.tile_frames = np.zeros(tiles, dtype=np.uint32); self.active = np.ones(tiles, dtype=np.uint8)

	def accumulate(self, frame):
		frame = np.ascontiguousarray(frame, dtype=np.float32)
		self.lib.vkr_host_adaptive_accumulate(self.width, self.height, frame.ctypes.data, self.state.ctypes.data, self.tile_frames.ctypes.data, self.active.ctypes.data)

	def update(self, target, min_frames, max_frames):
		self.lib.vkr_host_adaptive_update(self.width, self.height, self.state.ctypes.data, self.tile_frames.ctypes.data, self.active.ctypes.data, target, min_frames, max_frames)

	def resolve(self, variance=True):
		mean = np.zeros((self.height, self.width, 4), dtype=np.float32); var = np.zeros_like(mean) if variance else None
		self.lib.vkr_host_adaptive_resolve(self.width, self.height, self.state.ctypes.data, self.tile_frames.ctypes.data, mean.ctypes.data, var.ctypes.data if variance else None)
		return mean, var

	def estimate(self):
		out = np.zeros(3, dtype=np.float64)
		self.lib.vkr_host_adaptive_estimate(self.width, self.height, self.state.ctypes.data, self.tile_frames.ctypes.data, out.ctypes.data)
		return out


class NumpyAdaptive:
	"""The same definitions in numpy float64, whole arrays at a time."""

	def __init__(self, width, height):
		self.width, self.height = width, height
		self.tile_of = pixel_tiles(width, height)
		tiles = int(np.prod(tile_grid(width, height)))
		self.mean = np.zeros((3, width * height)); self.m2 = np.zeros((3, width * height))
		self.tile_frames = np.zeros(tiles, dtype=np.uint32); self.active = np.ones(tiles, dtype=np.uint8)

	def accumulate(self, frame):
		x = np.asarray(frame, dtype=np.float32)[..., :3].reshape(-1, 3).T.astype(np.float64)
		live = self.active[self.tile_of] != 0
		n = (self.tile_frames[self.tile_of] + 1).astype(np.float64)[None].repeat(3, 0)
		first = live & (n == 1.0)
		with np.errstate(invalid="ignore", over="ignore"):
			d = x - self.mean
			step = live & (n != 1.0) & (d != 0.0)       # d == 0 (or a NaN difference that compares unequal) as the C rule
			mean = np.where(step, self.mean + d / n, self.mean)
			m2 = np.where(step, self.m2 + d * (x - mean), self.m2)
		self.mean = np.where(first, x, mean); self.m2 = np.where(first, 0.0, m2)
		self.tile_frames = np.where(self.active != 0, self.tile_frames + 1, self.tile_frames).astype(np.uint32)

	def variance_of_mean(self):
		n = self.tile_frames[self.tile_of].astype(np.float64)
		with np.errstate(invalid="ignore", divide="ignore"):
			return self.m2 / (n * (n - 1.0))

	def update(self, target, min_frames, max_frames):
		with np.errstate(invalid="ignore", over="ignore"):
			ok = (np.isfinite(self.mean) & np.isfinite(self.m2) & (self.variance_of_mean() <= target * (self.mean * self.mean + EPS))).all(0)
		converged = np.ones_like(self.active, dtype=bool)
		np.logical_and.at(converged, self.tile_of, ok)
		n = self.tile_frames
		stop = (n >= max_frames) | ((n >= min_frames) & converged)
		self.active = np.where((self.active != 0) & ~stop, 1, 0).astype(np.uint8)

	def estimate(self):
		with np.errstate(invalid="ignore", over="ignore"):
			return (self.variance_of_mean() / (self.mean * self.mean + EPS)).mean(1)

	def state(self):
		return np.concatenate([self.mean, self.m2])


def graded_frames(seed, count, height, width, nonfinite_tiles=2):
	"""Frames whose noise level is a property of the tile: per tile a relative amplitude from {0, 1e-3, 1e-2, 0.1, 1}, so that tiles converge after
	different numbers of frames; per pixel a base value 10^U(-3, 1); a few tiles carry a NaN or an infinity in one of the first two frames (which every
	tile takes)."""
	rng = np.random.default_rng(seed)
	tiles_y, tiles_x = tile_grid(width, height)
	amplitude = rng.choice([0.0, 1e-3, 1e-2, 0.1, 1.0], tiles_y * tiles_x)[pixel_tiles(width, height)].reshape(height, width, 1)
	base = 10.0 ** rng.uniform(-3.0, 1.0, (height, width, 1))
	frames = (base[None] * np.abs(1.0 + amplitude[None] * rng.standard_normal((count, height, width, 4)))).astype(np.float32)
	frames[..., 3] = 1.0
	for k in range(nonfinite_tiles):
		y, x = rng.integers(0, height), rng.integers(0, width)
		frames[rng.integers(0, 2), y, x, rng.integers(0, 3)] = (np.nan, np.inf)[k % 2]
	return frames


def _same_bits(a, b):
	"""bit for bit, except that any NaN equals any NaN (numpy and C do not propagate the same NaN payloads)"""
	a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
	if a.shape != b.shape or a.dtype != b.dtype:
		return False
	bits = np.uint64 if a.dtype == np.float64 else np.uint32
	return bool(((a.view(bits) == b.view(bits)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("seed,width,height", [(1, 83, 61), (2, 128, 96), (3, 47, 25)])
def test_masked_accumulate_under_seeded_activity_matches_numpy(seed, width, height):
	frames = seeded_frames(seed, 12, height, width)
	rng = np.random.default_rng(100 + seed)
	host, ref = HostAdaptive(width, height), NumpyAdaptive(width, height)
	for f, frame in enumerate(frames):
		if f >= 2:   # a seeded pattern of active tiles; a tile that stopped stays stopped
			keep = (rng.random(host.active.size) < 0.9).astype(np.uint8)
			host.active &= keep; ref.active &= keep
		host.accumulate(frame); ref.accumulate(frame)
		assert np.array_equal(host.tile_frames, ref.tile_frames)
		assert _same_bits(host.state, ref.state())
	assert 0 < host.active.sum() < host.active.size and len(set(host.tile_frames.tolist())) > 3
	mean, var = host.resolve()
	n = host.tile_frames[pixel_tiles(width, height)].astype(np.float64)
	with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
		assert _same_bits(mean[..., :3].reshape(-1, 3), ref.mean.T.astype(np.float32)) and (mean[..., 3] == 1.0).all()
		assert _same_bits(var[..., :3].reshape(-1, 3), (ref.m2 / (n - 1.0)).T.astype(np.float32)) and (var[..., 3] == 0.0).all()


@pytest.mark.parametrize("seed,width,height,target", [(4, 83, 61, 1e-4), (5, 83, 61, 1e-2), (6, 200, 45, 1e-3), (7, 33, 100, 0.0)])
def test_tile_decisions_and_estimate_match_numpy(seed, width, height, target):
	min_frames, max_frames, batch = 4, 20, 2
	frames = graded_frames(seed, max_frames, height, width)
	host, ref = HostAdaptive(width, height), NumpyAdaptive(width, height)
	history = []
	for f, frame in enumerate(frames):
		host.accumulate(frame); ref.accumulate(frame)
		if (f + 1) % batch == 0:
			host.update(target, min_frames, max_frames); ref.update(target, min_frames, max_frames)
			assert np.array_equal(host.active, ref.active)
			history.append(int(host.active.sum()))
		assert _same_bits(host.state, ref.state()) and np.array_equal(host.tile_frames, ref.tile_frames)
	# the decisions went several ways: some tiles stopped early, the last ones at max_frames
	assert history[-1] == 0 and (target == 0.0 or len(set(history)) > 2)
	counts = set(host.tile_frames.tolist())
	assert max(counts) == max_frames and (target == 0.0 or min(counts) < max_frames)
	got, want = host.estimate(), ref.estimate()
	finite = np.isfinite(want)
	assert np.array_equal(finite, np.isfinite(got)) and np.all(np.abs(got[finite] - want[finite]) <= 1e-12 * np.abs(want[finite]))


def test_a_nonfinite_value_keeps_its_tile_active_until_max_frames():
	width, height = 40, 16
	frames = np.ones((10, height, width, 4), dtype=np.float32)   # constant: v = 0, every tile passes at min_frames
	frames[3, 2, 3, 1] = np.inf; frames[5, 12, 37, 0] = np.nan
	host = HostAdaptive(width, height)
	for frame in frames[:6]:
		host.accumulate(frame)
	host.update(1e-3, 2, 8)
	assert host.active.reshape(2, 3).tolist() == [[1, 0, 0], [0, 0, 1]]
	for frame in frames[6:]:
		host.accumulate(frame)
	host.update(1e-3, 2, 8)
	assert host.active.sum() == 0 and host.tile_frames.reshape(2, 3).tolist() == [[10, 6, 6], [6, 6, 10]]


@pytest.mark.parametrize("seed,count,width,height", [(8, 2, 83, 61), (9, 9, 37, 53)])
def test_every_tile_active_is_the_plain_accumulator(seed, count, width, height):
	frames = seeded_frames(seed, count, height, width)
	host = HostAdaptive(width, height)
	for frame in frames:
		host.accumulate(frame)
	state, mean, variance, _ = host_accumulate(frames)
	assert _same_bits(host.state, state) and (host.tile_frames == count).all()
	got_mean, got_var = host.resolve()
	assert _same_bits(got_mean, mean) and _same_bits(got_var, variance)
