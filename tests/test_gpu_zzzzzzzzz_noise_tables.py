"""Generating the noise tables on the device (vkr_generate_noise_table; vulkan_renderer_b200.noise_gen) and shading with them.

1. Both default tables (blue 64 x 64 x 64, Ahmed-Wonka 256 x 256 x 64) equal the host build of vkr_noise_gen.cuh (tests/noise_gen_on_host.cpp) bit
   for bit, and a second run gives the same bits.
2. Shading reads them exactly: a Cornell frame with diffuse + specular MIS and shadow rays, shaded with each table, equals the oracle fed the same
   texels bit for bit (the first GPU test with a noise table other than 256 x 256 x 64).
3. The tables do not move the converged image: the means of K animated frames with white noise and with the Ahmed-Wonka table agree within what
   their per-frame variances allow.
4. They move the error to high frequencies: single frames against a converged reference have the per-pixel MSE of white noise, and a lower
   MSE of 8 x 8 block means. The MSE is averaged over SINGLE_FRAMES frames, each with the offsets and layer of one animated constant block: in
   this scene most pixels are lit without occlusion and shade exactly, so a frame's error sits in few pixels (penumbrae), and the error of the
   one unanimated screenshot frame is too uneven to compare (DESIGN.md §5; it is printed).
"""
import numpy as np
import pytest

from tests import harness as H
from tests.test_noise_gen_on_host import host_ahmed, host_blue
from vulkan_renderer_b200 import api, convergence, experiments, noise_gen

pytestmark = pytest.mark.gpu

EXPERIMENT = "cornell_box_projected_solid_angle_ours_1spp"
SIZE, MEAN_FRAMES, REFERENCE_FRAMES, REFERENCE_SPP, SINGLE_FRAMES = 256, 64, 1024, 4, 16
BLOCKS = (1, 2, 4, 8)
# DESIGN.md §5, measured on an H100 80GB HBM3 (700 W power limit), mean over the 16 frames: block-mean MSE over white noise's at block sizes
# 1, 2, 4, 8 -- Ahmed-Wonka 1.067, 1.010, 0.829, 0.669; blue noise 0.914, 0.826, 0.686, 0.650. The frames are deterministic; the 8 x 8 bound
# leaves a margin of 1.3x over both measured ratios and still requires a drop below white noise.
BLOCK8_BOUND = 0.87


@pytest.fixture(scope="module")
def tables():
	out = {}
	for name, noise_type in noise_gen.NAMES.items():
		texels, stats = noise_gen.generate_noise_table(noise_type)
		print("%s %s on %s: %.3f ms (kernel, CUDA events), relaxation limit hits %d" % (name, texels.shape, stats["device"], stats["kernel_ms"], stats["relaxation_limit_hits"]))
		out[name] = texels
	return out


@pytest.fixture(scope="module")
def noise_root(tables, tmp_path_factory):
	root = str(tmp_path_factory.mktemp("noise_root"))
	for name, texels in tables.items():
		noise_gen.write_noise_table(root, noise_gen.NAMES[name], texels)
	return root


def test_the_default_tables_equal_the_host_build_and_repeat(tables):
	assert np.array_equal(tables["ahmed"], host_ahmed())
	blue, hits = host_blue()
	assert np.array_equal(tables["blue"], blue)
	for name, noise_type in noise_gen.NAMES.items():
		again, stats = noise_gen.generate_noise_table(noise_type)
		assert np.array_equal(again, tables[name]), name
	assert stats["relaxation_limit_hits"] == int(hits.sum())


@pytest.mark.parametrize("name", ["blue", "ahmed"])
def test_shading_with_the_table_equals_the_oracle(noise_root, tables, name):
	width, height = 128, 96
	texels = tables[name]
	layers, h, w, _ = texels.shape
	info = H.dataset("cornell")
	oi = H.OracleInputs(info)
	oi.noise = texels
	frame = H.open_frame(info, noise=(w, h, layers), noise_type=noise_gen.NAMES[name], noise_root=noise_root)
	try:
		assert (frame.noise.width, frame.noise.height, frame.noise.layers, frame.noise.random_seed) == (w, h, layers, noise_gen.LOADER_SEED)
		frame.configure(sample_count=2, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)
		constants = frame.constants(width, height)
		vis = oi.visibility(width, height, constants)
		gb = oi.gbuffer(width, height, constants, vis)
		out = frame.shade_host(width, height, gb)
		ref, rays = oi.shade(H.oracle_config(frame, width, height), constants, gb)
	finally:
		frame.close()
	cmp = H.compare_radiance(out, ref, rel=1.0e-5)
	print(name, cmp, "oracle rays", rays)
	assert cmp["bit_exact"] and rays > 0


def _frame(root, noise_type, reseed=False):
	experiment = [e for e in experiments.experiment_list(all_timings=False) if e["name"] == EXPERIMENT][0]
	info = experiments.prepare_data(experiment, root + "/data_sets")
	from vulkan_renderer_b200.frame import Frame
	noise = (64, 64, 64) if noise_type == api.NOISE_BLUE else (256, 256, 64)
	frame = Frame(info["vks"], info["textures"], info["save"], info["ltc"], noise=noise, noise_type=noise_type,
		noise_root=None if noise_type == api.NOISE_WHITE else root)
	experiments._configure(frame, experiment)
	if reseed:
		frame.noise.random_seed += 1000003    # random numbers of its own, not those of the frames under test
	return frame


def _accumulate(root, noise_type, frames, animate, **settings):
	frame = _frame(root, noise_type, reseed=animate)
	try:
		frame.configure(**settings)
		return convergence.accumulate(frame, SIZE, SIZE, frames, animate=animate)
	finally:
		frame.close()


def test_the_ahmed_table_does_not_move_the_converged_image(noise_root):
	a = _accumulate(noise_root, api.NOISE_WHITE, MEAN_FRAMES, True)
	b = _accumulate(noise_root, api.NOISE_AHMED, MEAN_FRAMES, True)
	difference = (a.mean[..., :3].astype(np.float64) - b.mean[..., :3]) ** 2
	allowed = (a.variance[..., :3].astype(np.float64) + b.variance[..., :3]) / MEAN_FRAMES
	ratio = difference.sum() / allowed.sum()
	print("%s %dx%d, %d animated frames: sum of squared mean differences / sum of their expected variances = %.4f" % (EXPERIMENT, SIZE, SIZE, MEAN_FRAMES, ratio))
	assert allowed.sum() > 0.0 and ratio < 1.5


def block_means(error, block):
	h, w, c = error.shape
	return error.reshape(h // block, block, w // block, block, c).mean(axis=(1, 3))


def test_the_tables_move_the_error_to_high_frequencies(noise_root):
	"""one unanimated frame (the screenshot) and SINGLE_FRAMES single frames with the animated offsets and layers of vkr_set_noise_constants"""
	reference = _accumulate(noise_root, api.NOISE_WHITE, REFERENCE_FRAMES, True, sample_count=REFERENCE_SPP).mean[..., :3].astype(np.float64)
	mse, screenshot = {}, {}
	for name, noise_type in (("white", api.NOISE_WHITE), ("ahmed", api.NOISE_AHMED), ("blue", api.NOISE_BLUE)):
		frame = _frame(noise_root, noise_type)
		try:
			errors = [convergence.accumulate(frame, SIZE, SIZE, 1, animate=False).mean[..., :3].astype(np.float64) - reference]
			errors += [convergence.accumulate(frame, SIZE, SIZE, 1, animate=True).mean[..., :3].astype(np.float64) - reference for _ in range(SINGLE_FRAMES)]
		finally:
			frame.close()
		screenshot[name] = [float(np.mean(block_means(errors[0], b) ** 2)) for b in BLOCKS]
		mse[name] = [float(np.mean([np.mean(block_means(e, b) ** 2) for e in errors[1:]])) for b in BLOCKS]
	for label, table in (("screenshot frame MSE", screenshot), ("mean MSE of %d frames" % SINGLE_FRAMES, mse)):
		print("%s %dx%d against %d x %d spp, block sizes %s, %s: white %s; over white: ahmed %s, blue %s" % (EXPERIMENT, SIZE, SIZE, REFERENCE_FRAMES, REFERENCE_SPP,
			BLOCKS, label, ["%.4e" % m for m in table["white"]], ["%.3f" % (m / w) for m, w in zip(table["ahmed"], table["white"])],
			["%.3f" % (m / w) for m, w in zip(table["blue"], table["white"])]))
	for name in ("ahmed", "blue"):
		assert 0.8 <= mse[name][0] / mse["white"][0] <= 1.25, name
		assert mse[name][-1] / mse["white"][-1] < BLOCK8_BOUND, name
