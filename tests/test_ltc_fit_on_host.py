"""The LTC fit (vulkan_renderer_b200/csrc/vkr_ltc_fit.cuh) compiled for the CPU (tests/ltc_fit_on_host.cpp: the kernel's loops as plain loops in the
same order), held against float64 numpy and scipy, and the fit<i>.dat round trip through the library's writer and loader. Single chains of reduced
tables at the full quadrature; the -m gpu tests hold the kernel against this build bit for bit (tests/test_gpu_zzzzzzzz_ltc_fit.py).

1. The BRDF term against a numpy restatement of brdfs.glsl:60-90.   2. The albedo against scipy quadrature, and the mirror limit.
3. The fit, measured as the shader evaluates it from the quantised table, against the synthetic table and an absolute bound.
4. Rotational symmetry on the row theta = 0.   5. No entry is clamped by the loader.   6. The file round trip.   7. Determinism.
"""
import ctypes as C
import os

import numpy as np
import pytest
from scipy import integrate

from vulkan_renderer_b200 import api, ltc_fit, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libltc_fit_on_host.so")
REF_HOST = os.path.join(ROOT, "oracle", "_ref", "libref_host.so")
N, F = 8, 3                     # the reduced table of these tests
QUADRATURE, ITERATION_LIMIT = 32, 400   # the defaults of vkr_ltc_fit_default_desc
L1_BOUND = 1.1                  # DESIGN.md §5: the largest L1 distance measured on the cells below is 0.93 (alpha = 0.02 at grazing incidence)
# F0 = 0 near normal incidence: Fresnel-Schlick vanishes towards the mirror direction, the narrow lobe is a ring that no LTC represents, and its
# albedo is below 1e-6 (DESIGN.md §5); neither table comes close there
DEGENERATE_CELLS = [(0, 1, 1)]


def host_lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	lib = C.CDLL(LIB_PATH)
	lib.vkr_host_ltc_specular_brdf.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]; lib.vkr_host_ltc_specular_brdf.restype = None
	lib.vkr_host_ltc_albedo.argtypes = [C.c_uint32, C.c_double, C.c_double, C.c_double, C.c_double]; lib.vkr_host_ltc_albedo.restype = C.c_double
	lib.vkr_host_ltc_fit_chains.argtypes = [C.c_uint32] * 5 + [C.c_void_p] * 5; lib.vkr_host_ltc_fit_chains.restype = None
	return lib


def host_fit_chains(resolution, fresnel_count, chains, quadrature=QUADRATURE, iteration_limit=ITERATION_LIMIT):
	"""the chains (layer * resolution + row) as the kernel fits them -> (fits [chains, N, 5], errors [chains, N], evaluations [chains, N], limit hits)"""
	chains = np.ascontiguousarray(list(chains), dtype=np.uint32)
	k = len(chains)
	fits = np.zeros((k, resolution, 5), dtype=np.float32); errors = np.zeros((k, resolution)); evaluations = np.zeros((k, resolution), dtype=np.uint32)
	hits = np.zeros(k, dtype=np.uint32)
	host_lib().vkr_host_ltc_fit_chains(resolution, fresnel_count, quadrature, iteration_limit, k, chains.ctypes.data, fits.ctypes.data, errors.ctypes.data,
		evaluations.ctypes.data, hits.ctypes.data)
	return fits, errors, evaluations, hits


@pytest.fixture(scope="module")
def table():
	fits, errors, evaluations, hits = host_fit_chains(N, F, range(N * F))
	return fits.reshape(F, N, N, 5), errors.reshape(F, N, N), evaluations, hits


def _unit(v):
	return v / np.linalg.norm(v, axis=-1, keepdims=True)


def test_brdf_term_matches_numpy():
	rng = np.random.default_rng(3)
	count = 4000
	wo = _unit(rng.normal(size=(count, 3))); wo[:, 2] = np.abs(wo[:, 2])
	wi = _unit(rng.normal(size=(count, 3))); wi[:, 2] = np.abs(wi[:, 2])
	wo[:200, 2] = 1.0e-3 * rng.random(200); wi[200:400, 2] = 1.0e-3 * rng.random(200)   # grazing
	wo = _unit(wo); wi = _unit(wi)
	alpha = rng.uniform(0.05, 1.0, count); f0 = rng.random(count)
	out = np.zeros(count); directions = np.ascontiguousarray(np.concatenate([wo, wi], axis=1))
	host_lib().vkr_host_ltc_specular_brdf(count, directions.ctypes.data, alpha.ctypes.data, f0.ctypes.data, out.ctypes.data)
	expected = np.array([ltc_fit.specular_brdf(wo[i], wi[i], alpha[i], f0[i]) for i in range(count)])
	assert np.isfinite(out).all() and (out > 0).all()
	assert np.max(np.abs(out - expected) / np.abs(expected)) < 1.0e-12


def _albedo_scipy(theta, alpha, f0):
	wo = np.array([np.sin(theta), 0.0, np.cos(theta)])
	def f(t, p):
		wi = np.array([np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)])
		return float(ltc_fit.specular_brdf(wo, wi, alpha, f0)) * wi[2] * np.sin(t)
	value, _ = integrate.dblquad(f, 0.0, np.pi, 0.0, 0.5 * np.pi, epsabs=1.0e-7, epsrel=1.0e-6)   # y >= 0, twice (the lobe is symmetric in y)
	return 2.0 * value


@pytest.mark.parametrize("alpha,theta_degrees,f0", [(0.05, 0, 0.0), (0.05, 45, 0.5), (0.05, 80, 1.0), (0.2, 0, 0.5), (0.2, 45, 1.0), (0.2, 80, 0.0),
	(0.5, 0, 1.0), (0.5, 45, 0.0), (0.5, 80, 0.5), (1.0, 0, 0.0), (1.0, 45, 0.5), (1.0, 80, 1.0)])
def test_albedo_matches_scipy(alpha, theta_degrees, f0):
	theta = np.deg2rad(theta_degrees)
	albedo = host_lib().vkr_host_ltc_albedo(QUADRATURE, np.cos(theta), np.sin(theta), alpha, f0)
	assert abs(albedo - _albedo_scipy(theta, alpha, f0)) < 1.0e-3


@pytest.mark.parametrize("theta_degrees", [0, 20, 45, 60, 80])
@pytest.mark.parametrize("f0", [0.0, 0.5, 1.0])
def test_albedo_at_the_smallest_roughness_is_the_mirror_fresnel(theta_degrees, f0):
	theta = np.deg2rad(theta_degrees)
	albedo = host_lib().vkr_host_ltc_albedo(QUADRATURE, np.cos(theta), np.sin(theta), ltc_fit.ALPHA_MIN, f0)
	assert abs(albedo - (f0 + (1.0 - f0) * (1.0 - np.cos(theta)) ** 5)) < 2.0e-3


def test_fit_beats_the_synthetic_table_where_the_shader_evaluates_it(table, tmp_path):
	fits = table[0]
	synth.write_ltc_fits(str(tmp_path), N, F)
	synthetic = ltc_fit.read_ltc_fits(str(tmp_path), F)
	grid = ltc_fit.hemisphere_grid(512, 1024)
	cells = [(f, row, column) for f in range(F) for row in (1, 3, 5, 7) for column in (1, 3, 5, 7) if (f, row, column) not in DEGENERATE_CELLS]
	fitted_l1 = [ltc_fit.l1_distance(fits, N, F, *c, grid=grid) for c in cells]
	synthetic_l1 = [ltc_fit.l1_distance(synthetic, N, F, *c, grid=grid) for c in cells]
	print("L1 distance, fitted: median %.4f max %.4f; synthetic: median %.4f max %.4f" % (np.median(fitted_l1), max(fitted_l1), np.median(synthetic_l1), max(synthetic_l1)))
	for c, a, b in zip(cells, fitted_l1, synthetic_l1):
		assert a < b and a < L1_BOUND, (c, a, b)


def test_row_theta_zero_is_rotationally_symmetric(table):
	m = table[0][:, 0].astype(np.float64)
	assert (np.abs(m[..., 1]) < 1.0e-2 * m[..., 0]).all() and (np.abs(m[..., 3]) < 1.0e-2 * m[..., 0]).all()
	assert (np.abs(m[..., 0] - m[..., 2]) < 1.0e-2 * m[..., 0]).all()


def test_no_entry_is_clamped_by_the_loader(table):
	fits, errors, _, hits = table
	entries, determinant = ltc_fit.unclamped_entries(fits)
	assert np.isfinite(fits).all() and np.isfinite(errors).all() and hits.sum() == 0
	assert (entries >= 0.0).all() and (entries <= 1.0).all() and (determinant > 0.0).all()


def test_files_round_trip_through_the_loader(table, tmp_path):
	fits = table[0]
	lib = api.load_library()
	ltc_fit.write_ltc_fits(str(tmp_path), fits)
	assert np.array_equal(ltc_fit.read_ltc_fits(str(tmp_path), F).view(np.uint32), fits.view(np.uint32))
	loaded = api.LtcTable()
	assert lib.vkr_load_ltc_table(C.byref(loaded), None, str(tmp_path).encode(), F) == 0
	try:
		assert loaded.roughness_count == N and loaded.fresnel_count == F
		table0 = np.ctypeslib.as_array(loaded.h_table0, (F, N, N, 4)).copy(); table1 = np.ctypeslib.as_array(loaded.h_table1, (F, N, N, 2)).copy()
	finally:
		lib.vkr_destroy_ltc_table(C.byref(loaded), None)
	q0, q1 = ltc_fit.quantise(fits)
	assert np.array_equal(table0, q0) and np.array_equal(table1, q1)
	if os.path.exists(REF_HOST):   # the reference's own load_ltc_table
		ref = C.CDLL(REF_HOST)
		res = C.c_uint32(); t0 = C.c_void_p(); t1 = C.c_void_p(); constants = (C.c_float * 8)()
		assert ref.ref_probe_load_ltc(str(tmp_path).encode(), F, C.byref(res), C.byref(t0), C.byref(t1), constants) == 0 and res.value == N
		assert np.array_equal(np.ctypeslib.as_array(C.cast(t0, C.POINTER(C.c_uint16)), (F, N, N, 4)), table0)
		assert np.array_equal(np.ctypeslib.as_array(C.cast(t1, C.POINTER(C.c_uint16)), (F, N, N, 2)), table1)


def test_refusals(tmp_path, capfd):
	lib = api.load_library()
	device = api.Device()
	out = np.zeros(5 * 64 * 64 * 51, dtype=np.float32)
	for bad in ((1, 51, 32, 400), (64, 1, 32, 400), (64, 51, 1, 400), (64, 51, 32, 0), (5000, 51, 32, 400), (64, 51, 300, 400)):
		assert lib.vkr_fit_ltc_table(C.byref(device), C.byref(api.LtcFitDesc(*bad)), out.ctypes.data, None) == 1
	assert lib.vkr_fit_ltc_table(C.byref(device), None, out.ctypes.data, None) == 1
	fits = np.zeros((1, 2, 2, 5), dtype=np.float32)
	assert lib.vkr_write_ltc_fits(str(tmp_path / "missing" / "dir").encode(), 2, 1, fits.ctypes.data) == 1
	assert lib.vkr_write_ltc_fits(str(tmp_path).encode(), 0, 1, fits.ctypes.data) == 1
	assert lib.vkr_write_ltc_fits(str(tmp_path).encode(), 2, 1, None) == 1
	assert "Failed" in capfd.readouterr().out
	desc = ltc_fit.default_desc()
	assert (desc.resolution, desc.fresnel_count, desc.quadrature_size, desc.iteration_limit) == (64, 51, QUADRATURE, ITERATION_LIMIT)


def test_fits_are_deterministic_and_chains_independent(table):
	fits, errors = table[0], table[1]
	again, again_errors, _, _ = host_fit_chains(N, F, range(N * F))
	assert np.array_equal(again.reshape(F, N, N, 5).view(np.uint32), fits.view(np.uint32)) and np.array_equal(again_errors.reshape(F, N, N), errors)
	for chain in (N * F - 1, 0, N + 3):
		single, single_errors, _, _ = host_fit_chains(N, F, [chain])
		layer, row = divmod(chain, N)
		assert np.array_equal(single[0].view(np.uint32), fits[layer, row].view(np.uint32)) and np.array_equal(single_errors[0], errors[layer, row])
