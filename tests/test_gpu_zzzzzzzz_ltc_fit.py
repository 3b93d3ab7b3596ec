"""Fitting the LTC table on the device (vkr_fit_ltc_table; vulkan_renderer_b200.ltc_fit).

1. The kernel against the host build of vkr_ltc_fit.cuh (tests/ltc_fit_on_host.cpp) bit for bit: a reduced table (N = 8, F = 3) whole, and four
   chains of the full 64 x 64 x 51 table.
2. The full table fits, every entry is representable by the loader, and a second run gives the same bits.
3. The LTC only steers sampling and MIS weights: on the roughness planes (diffuse + specular MIS, clamped optimal heuristic) the means of K animated
   frames with the synthetic and with the fitted table agree within what their per-frame variances allow.
4. The fitted table gives less variance per frame than the synthetic one there.
"""
import numpy as np
import pytest

from tests.test_ltc_fit_on_host import host_fit_chains
from vulkan_renderer_b200 import api, convergence, experiments, ltc_fit

pytestmark = pytest.mark.gpu

WIDTH, HEIGHT, FRAMES = 288, 128, 48


@pytest.fixture(scope="module")
def full_table():
	fits, stats = ltc_fit.fit_ltc_table()
	print("full table on %s: %.1f ms, %d objective evaluations, %d iteration limit hits, L3 max %.4g median %.4g" % (stats["device"], stats["fit_ms"],
		stats["objective_evaluations"], stats["iteration_limit_hits"], stats["max_error"], stats["median_error"]))
	return fits, stats


def test_reduced_table_matches_the_host_build_bit_for_bit():
	fits, stats = ltc_fit.fit_ltc_table(resolution=8, fresnel_count=3)
	h_fits, h_errors, h_evaluations, _ = host_fit_chains(8, 3, range(24))
	assert np.array_equal(fits.view(np.uint32), h_fits.reshape(3, 8, 8, 5).view(np.uint32))
	assert np.array_equal(stats["cell_errors"].view(np.uint64), h_errors.reshape(3, 8, 8).view(np.uint64))
	assert stats["objective_evaluations"] == int(h_evaluations.sum()) and stats["cell_count"] == 192


def test_full_table_matches_the_host_build_on_four_chains(full_table):
	fits, stats = full_table
	chains = [0, 63, 25 * 64 + 31, 50 * 64 + 1]
	h_fits, h_errors, _, _ = host_fit_chains(64, 51, chains)
	for k, chain in enumerate(chains):
		layer, row = divmod(chain, 64)
		assert np.array_equal(fits[layer, row].view(np.uint32), h_fits[k].view(np.uint32)), chain
		assert np.array_equal(stats["cell_errors"][layer, row].view(np.uint64), h_errors[k].view(np.uint64)), chain


def test_full_table_is_representable_and_deterministic(full_table):
	fits, stats = full_table
	assert fits.shape == (51, 64, 64, 5) and np.isfinite(fits).all() and stats["cell_count"] == 51 * 64 * 64
	entries, determinant = ltc_fit.unclamped_entries(fits)
	assert (entries >= 0.0).all() and (entries <= 1.0).all() and (determinant > 0.0).all()
	again, stats_again = ltc_fit.fit_ltc_table()
	assert np.array_equal(fits.view(np.uint32), again.view(np.uint32))
	assert np.array_equal(stats["cell_errors"].view(np.uint64), stats_again["cell_errors"].view(np.uint64))
	assert stats["objective_evaluations"] == stats_again["objective_evaluations"]


@pytest.fixture(scope="module")
def planes(full_table, tmp_path_factory):
	"""mean and variance of FRAMES animated frames of the roughness planes with each table"""
	root = tmp_path_factory.mktemp("ltc_planes")
	fitted_dir = str(root / "fitted")
	ltc_fit.write_ltc_fits(fitted_dir, full_table[0])
	experiment = [e for e in experiments.experiment_list(all_timings=False) if e["name"] == "roughness_planes_lambertian_2spp"][0]
	out = {}
	for label, ltc_dir in (("synthetic", None), ("fitted", fitted_dir)):
		info = experiments.prepare_data(experiment, str(root / "data"), ltc_dir)
		from vulkan_renderer_b200.frame import Frame
		frame = Frame(info["vks"], info["textures"], info["save"], info["ltc"])
		try:
			experiments._configure(frame, experiment)
			frame.configure(heuristic=api.MIS_OPTIMAL_CLAMPED, sample_count=1)
			out[label] = convergence.accumulate(frame, WIDTH, HEIGHT, FRAMES, animate=True)
		finally:
			frame.close()
	return out


def test_the_fitted_table_does_not_move_the_converged_image(planes):
	a, b = planes["synthetic"], planes["fitted"]
	difference = (a.mean[..., :3].astype(np.float64) - b.mean[..., :3]) ** 2
	allowed = (a.variance[..., :3].astype(np.float64) + b.variance[..., :3]) / FRAMES
	ratio = difference.sum() / allowed.sum()
	print("roughness planes, %d frames: sum of squared mean differences / sum of their expected variances = %.4f" % (FRAMES, ratio))
	assert allowed.sum() > 0.0 and ratio < 1.5


def test_the_fitted_table_has_less_variance_than_the_synthetic_one(planes):
	synthetic = float(np.mean(planes["synthetic"].mean_variance)); fitted = float(np.mean(planes["fitted"].mean_variance))
	print("roughness planes %dx%d, 1 spp, diffuse + specular MIS, clamped optimal: mean variance per frame synthetic %.5e, fitted %.5e" % (WIDTH, HEIGHT, synthetic, fitted))
	assert fitted < synthetic
