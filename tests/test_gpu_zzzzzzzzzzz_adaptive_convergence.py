"""Adaptive convergence: the adaptive accumulator (vkr_adaptive_accumulator_t), the tile-subset launch (vkr_shading_pass_run_tiles) and
convergence.accumulate_adaptive.

1. The kernels against the host build of vkr_accumulate.cuh (tests/adaptive_on_host.cpp) bit for bit on seeded frame sequences, through the tile tests
   that stop tiles along the way: flags, counts, resolved mean and variance, estimated relMSE; a second run gives the same bits.
2. vkr_shading_pass_run_tiles on the Cornell box (diffuse, projected solid angle, shadow rays; and diffuse + specular MIS): the listed tiles equal a
   full frame bit for bit, every other pixel keeps the sentinel written before, a full frame afterwards equals the one before, and it refuses what it
   must.
3. The prefix property: every tile of an adaptive run equals the plain accumulator after that tile's frame count, bit for bit; two adaptive runs are
   identical; min_frames = max_frames is the plain run.
4. What it saves on the Cornell box at a fixed target, and how far its mean is from the full reference.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import harness as H
from tests.test_adaptive_on_host import HostAdaptive, _same_bits, graded_frames, pixel_tiles
from vulkan_renderer_b200 import api, convergence

pytestmark = pytest.mark.gpu

WIDTH, HEIGHT = 136, 100     # 9 x 13 tiles, the last column and row clipped
DIFFUSE = dict(sample_count=1, strategy=api.STRATEGY_DIFFUSE_ONLY, technique=api.TECHNIQUE_PSA, trace_shadow_rays=1)
MIS = dict(sample_count=1, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)


@pytest.fixture(scope="module")
def device():
	lib = api.load_library(); dev = api.Device()
	assert lib.vkr_create_device(C.byref(dev), 0, None) == 0
	yield lib, dev
	lib.vkr_destroy_device(C.byref(dev))


def _device_sequence(lib, dev, frames, target, min_frames, max_frames, batch):
	"""frames [F, H, W, 4] through the adaptive accumulator with a tile test every `batch` frames -> (flags after each test, counts, mean, variance, estimate)"""
	count, height, width = frames.shape[:3]
	d_frames = torch.as_tensor(frames).cuda(); mean = torch.empty((height, width, 4), dtype=torch.float32, device="cuda"); var = torch.empty_like(mean)
	torch.cuda.synchronize()
	acc = api.AdaptiveAccumulator()
	assert lib.vkr_create_adaptive_accumulator(C.byref(acc), C.byref(dev), width, height) == 0
	try:
		tiles = acc.tiles_x * acc.tiles_y
		assert acc.active_tile_count == tiles and acc.frame_count == 0
		flags = []
		for f in range(count):
			assert lib.vkr_adaptive_accumulate_frame(C.byref(acc), C.byref(dev), d_frames[f].data_ptr()) == 0
			if (f + 1) % batch == 0:
				active = np.zeros(tiles, dtype=np.uint8); n = C.c_uint32()
				assert lib.vkr_adaptive_update_tiles(C.byref(acc), C.byref(dev), target, min_frames, max_frames, active.ctypes.data, C.byref(n)) == 0
				assert n.value == acc.active_tile_count == active.sum()
				flags.append(active)
		counts = np.zeros(tiles, dtype=np.uint32)
		assert lib.vkr_adaptive_tile_frames(C.byref(acc), C.byref(dev), counts.ctypes.data) == 0
		assert lib.vkr_adaptive_resolve(C.byref(acc), C.byref(dev), mean.data_ptr(), var.data_ptr()) == 0
		estimate = np.zeros(3, dtype=np.float64)
		assert lib.vkr_adaptive_estimated_rel_mse(C.byref(acc), C.byref(dev), estimate.ctypes.data_as(C.POINTER(C.c_double))) == 0
		assert lib.vkr_device_wait_idle(C.byref(dev)) == 0
	finally:
		lib.vkr_destroy_adaptive_accumulator(C.byref(acc), C.byref(dev))
	return flags, counts, mean.cpu().numpy(), var.cpu().numpy(), estimate


@pytest.mark.parametrize("seed,width,height,target,nonfinite", [(1, 83, 61, 1e-4, 2), (2, 200, 45, 1e-3, 0), (3, 1920, 1080, 1e-4, 0)])
def test_kernels_match_the_host_build_bit_for_bit(device, seed, width, height, target, nonfinite):
	lib, dev = device
	min_frames, max_frames, batch = 4, 12, 2
	frames = graded_frames(seed, max_frames, height, width, nonfinite_tiles=nonfinite)
	host = HostAdaptive(width, height)
	host_flags = []
	for f, frame in enumerate(frames):
		host.accumulate(frame)
		if (f + 1) % batch == 0:
			host.update(target, min_frames, max_frames); host_flags.append(host.active.copy())
	h_mean, h_var = host.resolve()
	first = _device_sequence(lib, dev, frames, target, min_frames, max_frames, batch)
	flags, counts, mean, var, estimate = first
	assert [f.tolist() for f in flags] == [f.tolist() for f in host_flags]
	assert np.array_equal(counts, host.tile_frames) and len(set(counts.tolist())) > 1
	assert _same_bits(mean, h_mean) and _same_bits(var, h_var)
	h_estimate = host.estimate()
	assert _same_bits(estimate, h_estimate) and np.isfinite(estimate).all() == (nonfinite == 0)
	again = _device_sequence(lib, dev, frames, target, min_frames, max_frames, batch)
	assert [f.tolist() for f in again[0]] == [f.tolist() for f in flags] and np.array_equal(again[1], counts)
	assert np.array_equal(again[2].view(np.uint32), mean.view(np.uint32)) and np.array_equal(again[3].view(np.uint32), var.view(np.uint32))
	assert again[4].view(np.uint64).tolist() == estimate.view(np.uint64).tolist()


def test_adaptive_refusals(device, capfd):
	lib, dev = device
	frame = torch.ones((8, 16, 4), dtype=torch.float32, device="cuda"); out = torch.empty_like(frame)
	torch.cuda.synchronize()
	acc = api.AdaptiveAccumulator()
	assert lib.vkr_create_adaptive_accumulator(C.byref(acc), C.byref(dev), 16, 0) == 1 and acc.d_state is None
	assert lib.vkr_create_adaptive_accumulator(C.byref(acc), C.byref(dev), 16, 8) == 0
	try:
		est = (C.c_double * 3)()
		assert lib.vkr_adaptive_resolve(C.byref(acc), C.byref(dev), out.data_ptr(), None) == 1          # no frame yet
		assert lib.vkr_adaptive_accumulate_frame(C.byref(acc), C.byref(dev), None) == 1
		assert lib.vkr_adaptive_accumulate_frame(C.byref(acc), C.byref(dev), frame.data_ptr()) == 0
		assert lib.vkr_adaptive_resolve(C.byref(acc), C.byref(dev), None, out.data_ptr()) == 1          # a variance needs 2 frames
		assert lib.vkr_adaptive_estimated_rel_mse(C.byref(acc), C.byref(dev), est) == 1
		for target, lo, hi in ((-1e-3, 2, 8), (float("nan"), 2, 8), (float("inf"), 2, 8), (1e-3, 1, 8), (1e-3, 8, 7)):
			assert lib.vkr_adaptive_update_tiles(C.byref(acc), C.byref(dev), target, lo, hi, None, None) == 1
		assert lib.vkr_adaptive_accumulate_frame(C.byref(acc), C.byref(dev), frame.data_ptr()) == 0
		assert lib.vkr_adaptive_update_tiles(C.byref(acc), C.byref(dev), 0.0, 2, 8, None, None) == 0 and acc.active_tile_count == 0   # constant frames: v = 0
		assert lib.vkr_adaptive_accumulator_reset(C.byref(acc), C.byref(dev)) == 0 and acc.frame_count == 0 and acc.active_tile_count == 1
		counts = np.ones(1, dtype=np.uint32)
		assert lib.vkr_adaptive_tile_frames(C.byref(acc), C.byref(dev), counts.ctypes.data) == 0 and counts[0] == 0
	finally:
		lib.vkr_destroy_adaptive_accumulator(C.byref(acc), C.byref(dev))
	lib.vkr_destroy_adaptive_accumulator(C.byref(acc), C.byref(dev))   # a zeroed struct
	assert "Failed" in capfd.readouterr().out


def _cornell(**settings):
	frame = H.open_frame(H.dataset("cornell"))
	frame.configure(**settings)
	return frame


SENTINEL = np.float32(-7.25)


@pytest.mark.parametrize("settings", [DIFFUSE, MIS], ids=["diffuse_psa_rays", "mis_rays"])
def test_run_tiles_shades_the_listed_tiles_only(device, settings, capfd):
	frame = _cornell(**settings)
	lib, dev = frame.lib, C.byref(frame.device)
	targets = api.RenderTargets()
	try:
		constants = frame.constants(WIDTH, HEIGHT)
		assert lib.vkr_create_render_targets(C.byref(targets), dev, WIDTH, HEIGHT) == 0
		assert lib.vkr_run_visibility_pass(dev, C.byref(frame.scene), constants, WIDTH, HEIGHT, targets.d_visibility) == 0
		assert lib.vkr_run_gbuffer_pass(dev, C.byref(frame.scene), constants, WIDTH, HEIGHT, targets.d_visibility, targets.d_gbuffer) == 0
		p = frame.create_pass(WIDTH, HEIGHT, timing=True)
		tiles_x, tiles_y = (WIDTH + 15) // 16, (HEIGHT + 7) // 8
		assert p.tile_count == tiles_x * tiles_y
		out = torch.empty((HEIGHT, WIDTH, 4), dtype=torch.float32, device="cuda")

		def full():
			torch.cuda.synchronize()
			assert lib.vkr_shading_pass_run(C.byref(p), dev, constants, len(constants), targets.d_gbuffer, out.data_ptr()) == 0
			assert lib.vkr_shading_pass_wait(C.byref(p), dev) == 0
			return out.cpu().numpy()

		def subset(tiles):
			out.fill_(float(SENTINEL)); torch.cuda.synchronize()
			tiles = np.ascontiguousarray(tiles, dtype=np.uint32)
			rc = lib.vkr_shading_pass_run_tiles(C.byref(p), dev, constants, len(constants), targets.d_gbuffer, out.data_ptr(), tiles.ctypes.data, tiles.size)
			assert lib.vkr_shading_pass_wait(C.byref(p), dev) == 0
			return rc, out.cpu().numpy()

		before = full(); full()    # the second frame runs in the cost order the first one measured
		order = np.ctypeslib.as_array((C.c_uint32 * p.tile_count).from_address(p.h_tile_list)).copy()
		launches, pending, reorder = p.kernel_launches, p.costs_pending, p.reorder_tiles
		rng = np.random.default_rng(5)
		listed = rng.permutation(p.tile_count)[:40]
		p.last_kernel_ms = 0.0
		rc, got = subset(listed)
		assert rc == 0 and p.last_kernel_ms > 0.0 and p.kernel_launches == launches + 1
		tile_of = pixel_tiles(WIDTH, HEIGHT).reshape(HEIGHT, WIDTH)
		inside = np.isin(tile_of, listed)
		assert np.array_equal(got[inside].view(np.uint32), before[inside].view(np.uint32)) and (got[inside][:, :3] > 0).any()
		assert (got[~inside] == SENTINEL).all()
		# the pass's own state is as it was
		assert np.array_equal(np.ctypeslib.as_array((C.c_uint32 * p.tile_count).from_address(p.h_tile_list)), order)
		assert (p.costs_pending, p.reorder_tiles) == (pending, reorder)
		assert np.array_equal(full().view(np.uint32), before.view(np.uint32))
		# an empty list launches nothing; refusals write nothing
		launches = p.kernel_launches
		assert subset([])[0] == 0 and p.kernel_launches == launches
		for bad in ([tiles_x * tiles_y], [3, 7, 3], list(range(p.tile_count)) + [0]):
			rc, got = subset(bad)
			assert rc == 1 and (got == SENTINEL).all() and p.kernel_launches == launches
		# a tile of the other instance of a two-way split
		half = frame.create_pass(WIDTH, HEIGHT, stripe_index=0, stripe_count=2)
		share = set(np.ctypeslib.as_array((C.c_uint32 * half.tile_count).from_address(half.h_tile_list)).tolist())
		other = np.array([t for t in range(tiles_x * tiles_y) if t not in share][:1], dtype=np.uint32)
		mine = np.array(sorted(share)[:3], dtype=np.uint32)
		assert lib.vkr_shading_pass_run_tiles(C.byref(half), dev, constants, len(constants), targets.d_gbuffer, out.data_ptr(), other.ctypes.data, 1) == 1
		assert lib.vkr_shading_pass_run_tiles(C.byref(half), dev, constants, len(constants), targets.d_gbuffer, out.data_ptr(), mine.ctypes.data, 3) == 0
		assert lib.vkr_shading_pass_wait(C.byref(half), dev) == 0
	finally:
		lib.vkr_destroy_render_targets(C.byref(targets), dev)
		frame.close()
	assert "Failed to shade a tile list" in capfd.readouterr().out


def _plain_snapshots(frame, width, height, frames, every):
	"""The plain path as accumulate_adaptive draws its frames (animated noise, one constant block per frame, the first also for the G-buffer),
	resolved after every `every` frames -> {n: (mean, variance)}"""
	lib, dev = frame.lib, C.byref(frame.device)
	targets = api.RenderTargets(); acc = api.Accumulator()
	saved = frame.settings.animate_noise
	frame.settings.animate_noise = 1
	snapshots = {}
	try:
		constants = frame.constants(width, height)
		assert lib.vkr_create_render_targets(C.byref(targets), dev, width, height) == 0
		assert lib.vkr_run_visibility_pass(dev, C.byref(frame.scene), constants, width, height, targets.d_visibility) == 0
		assert lib.vkr_run_gbuffer_pass(dev, C.byref(frame.scene), constants, width, height, targets.d_visibility, targets.d_gbuffer) == 0
		p = frame.create_pass(width, height)
		assert lib.vkr_create_accumulator(C.byref(acc), dev, width, height) == 0
		mean = torch.empty((height, width, 4), dtype=torch.float32, device="cuda"); var = torch.empty_like(mean)
		torch.cuda.synchronize()
		for i in range(frames):
			if i:
				constants = frame.constants(width, height)
			assert lib.vkr_shading_pass_run(C.byref(p), dev, constants, len(constants), targets.d_gbuffer, targets.d_frame) == 0
			assert lib.vkr_accumulate_frame(C.byref(acc), dev, targets.d_frame) == 0
			if (i + 1) % every == 0:
				assert lib.vkr_accumulator_resolve(C.byref(acc), dev, mean.data_ptr(), var.data_ptr()) == 0
				assert lib.vkr_device_wait_idle(dev) == 0
				snapshots[i + 1] = (mean.cpu().numpy(), var.cpu().numpy())
	finally:
		frame.settings.animate_noise = saved
		lib.vkr_destroy_accumulator(C.byref(acc), dev)
		lib.vkr_destroy_render_targets(C.byref(targets), dev)
	return snapshots


def test_every_tile_is_the_plain_accumulator_after_its_frame_count():
	min_frames, max_frames, batch = 8, 32, 4
	frame = _cornell(**DIFFUSE)
	try:
		seed = frame.noise.random_seed
		plain = _plain_snapshots(frame, WIDTH, HEIGHT, max_frames, batch)
		seed_after = frame.noise.random_seed
		# a target that stops about half the tiles at min_frames: the median over the tiles of their largest v / (mean^2 + 0.01) after min_frames
		mean, var = plain[min_frames]
		ratio = (var[..., :3].astype(np.float64) / min_frames / (mean[..., :3].astype(np.float64) ** 2 + 0.01)).max(-1).reshape(-1)
		worst = np.zeros(((HEIGHT + 7) // 8) * ((WIDTH + 15) // 16)); np.maximum.at(worst, pixel_tiles(WIDTH, HEIGHT), ratio)
		target = float(np.median(worst))
		runs = []
		for _ in range(2):
			frame.noise.random_seed = seed
			runs.append(convergence.accumulate_adaptive(frame, WIDTH, HEIGHT, max_frames, target, min_frames=min_frames, batch=batch))
			assert frame.noise.random_seed == seed_after and frame.settings.animate_noise == 0
		frame.noise.random_seed = seed
		whole = convergence.accumulate_adaptive(frame, WIDTH, HEIGHT, max_frames, target, min_frames=max_frames, batch=batch)
	finally:
		frame.close()
	a, b = runs
	counts = a.tile_frames.reshape(-1)
	print("adaptive Cornell %dx%d, target %.3e: tile frame counts %s, %d of %d tile-frames" % (WIDTH, HEIGHT, target, np.bincount(counts).nonzero()[0].tolist(),
		a.tile_frames_shaded, a.tile_frames_full))
	assert set(counts.tolist()) <= set(range(min_frames, max_frames + 1, batch)) and len(set(counts.tolist())) > 1
	assert a.tile_frames_shaded == int(counts.sum()) and a.tile_frames_full == counts.size * max_frames and a.frames == counts.max()
	tile_of = pixel_tiles(WIDTH, HEIGHT).reshape(HEIGHT, WIDTH)
	for n in set(counts.tolist()):
		sel = np.isin(tile_of, np.nonzero(counts == n)[0])
		assert np.array_equal(a.mean[sel].view(np.uint32), plain[n][0][sel].view(np.uint32)), n
		assert np.array_equal(a.variance[sel].view(np.uint32), plain[n][1][sel].view(np.uint32)), n
	assert np.array_equal(a.tile_frames, b.tile_frames) and np.array_equal(a.mean.view(np.uint32), b.mean.view(np.uint32))
	assert np.array_equal(a.variance.view(np.uint32), b.variance.view(np.uint32)) and a.estimated_rel_mse.tolist() == b.estimated_rel_mse.tolist()
	assert (whole.tile_frames == max_frames).all() and whole.tile_frames_shaded == whole.tile_frames_full
	assert np.array_equal(whole.mean.view(np.uint32), plain[max_frames][0].view(np.uint32))
	assert np.array_equal(whole.variance.view(np.uint32), plain[max_frames][1].view(np.uint32))


# Cornell box, diffuse, projected solid angle sampling, shadow rays, 256x256: adaptive to the target with 8 .. 64 frames, tested every 8, against the
# plain 64-frame mean of the same frames. Measured on an H100 80GB HBM3 (700 W power limit): 0.2126 of the tile-frames shaded, relMSE against the
# full mean 4.40e-6 = 0.0044 x target (DESIGN §5). The results are bit-identical from device to device; the bounds leave room for changes of the scene.
SAVINGS = dict(width=256, height=256, max_frames=64, min_frames=8, batch=8, target=1e-3)
MAX_SHADED_FRACTION = 0.3
MAX_REL_MSE_OVER_TARGET = 0.05


def test_adaptive_reference_shades_less_at_a_bounded_error():
	s = SAVINGS
	frame = _cornell(**DIFFUSE)
	try:
		seed = frame.noise.random_seed
		adaptive = convergence.accumulate_adaptive(frame, s["width"], s["height"], s["max_frames"], s["target"], min_frames=s["min_frames"], batch=s["batch"])
		frame.noise.random_seed = seed
		full = convergence.accumulate(frame, s["width"], s["height"], s["max_frames"], animate=True)
		error = convergence.frame_error(frame, adaptive.mean, full.mean)
	finally:
		frame.close()
	fraction = adaptive.tile_frames_shaded / adaptive.tile_frames_full
	rel_mse = float(np.mean(error["rel_mse"]))
	print("adaptive Cornell reference %s: %d of %d tile-frames (%.4f), estimated relMSE %s, relMSE against the full mean %.4e (%.3f x target), "
		"frame counts %s, shading %.2f ms, accumulate %.2f ms" % (s, adaptive.tile_frames_shaded, adaptive.tile_frames_full, fraction,
		adaptive.estimated_rel_mse.tolist(), rel_mse, rel_mse / s["target"], np.bincount(adaptive.tile_frames.reshape(-1)).nonzero()[0].tolist(),
		adaptive.shade_ms, adaptive.accumulate_ms))
	assert fraction < MAX_SHADED_FRACTION
	assert rel_mse <= MAX_REL_MSE_OVER_TARGET * s["target"]
