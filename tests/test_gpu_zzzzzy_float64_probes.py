"""The GPU's polygon sampler and shadow-ray query through their probes (vkr_sample_polygon_batch, vkr_trace_shadow_rays), with the polygons, random
numbers and ray families of tests/test_float64_references.py: bit for bit against the oracle, and independently against the float64 references
(tests/float64_ref.py) -- a pair that agrees bit for bit can still be wrong together. The undecided fractions and tolerances are those of the CPU half
and are justified there.

The shadow probe walks node pairs per thread with the same ray_box / ray_triangle as the trace warps of the shading kernel; their interleaved loop is
covered by the frame comparisons and, on the CPU, by test_interleaved_node_pairs_visit_and_answer_like_the_float_pairs. (The trace warps set up the
slab test without the guard against direction components below 2^-64, vkr_trace.cuh: make_slabs; the unusual-direction family needs that guard.)
"""
import ctypes as C
import time

import numpy as np
import pytest

from oracle import binding as oracle
from tests import float64_ref as R
from tests import harness as H
from tests import test_float64_references as F
from tests.test_host_logic import _probe_bvh, BUILDERS
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu


def _device():
	lib = api.load_library(); dev = api.Device()
	assert lib.vkr_create_device(C.byref(dev), 0, None) == 0
	return lib, dev


def _gpu_sample(lib, dev, pts, biased, u):
	pts = np.ascontiguousarray(pts, dtype=np.float32); u = np.ascontiguousarray(u, dtype=np.float32)
	dirs = np.zeros((len(u), 3), dtype=np.float32); info = np.zeros(11, dtype=np.float32)
	assert lib.vkr_sample_polygon_batch(C.byref(dev), len(pts), pts.ctypes.data, int(biased), len(u), u.ctypes.data, dirs.ctypes.data, info.ctypes.data) == 0
	return dirs, info


def _same_bits(a, b):
	a = np.asarray(a, dtype=np.float32); b = np.asarray(b, dtype=np.float32)
	return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


@pytest.mark.parametrize("biased", [False, True])
def test_gpu_sampler_equals_the_oracle_and_meets_the_float64_references(biased):
	lib, dev = _device()
	try:
		stats = {}; samples = 0
		for index, (family, n, pts) in enumerate(F.POLYGONS):
			u, kind, dirs_o, info_o = F.sampling_case(family, n, pts, biased, index)
			dirs, raw = _gpu_sample(lib, dev, pts, biased, u)
			assert _same_bits(dirs, dirs_o).all(), (family, n, biased, index, u[~_same_bits(dirs, dirs_o).all(1)][:4])
			ref_info = np.concatenate([[info_o["psa"], float(info_o["central"]), float(info_o["vc"])], info_o["sectors"]]).astype(np.float32)
			assert _same_bits(raw, ref_info).all(), (family, n, biased, index, raw, ref_info)
			info = dict(psa=float(raw[0]), central=bool(raw[1]), vc=int(raw[2]), sectors=raw[3:].copy())
			F.check_sampling_against_float64(family, n, pts, biased, u, kind, dirs, info, stats)
			samples += len(u)
		print("GPU sampler, biased=%d: %d polygons, %d samples, largest relative PSA error %.2e, worst backward error %.2e, %d NaN samples"
			% (biased, len(F.POLYGONS), samples, stats.get("psa_rel", 0), stats.get("backward", 0), stats.get("nan", 0)))
		# 2 or 8 vertices: refused before anything is allocated or launched, the outputs stay as they were
		for count in (2, 8):
			pts = np.tile(np.float32([[0.1, 0.2, 1.0]]), (count, 1)); u = np.full((4, 2), 0.5, dtype=np.float32)
			dirs = np.full((4, 3), 7.0, dtype=np.float32); info = np.full(11, 7.0, dtype=np.float32)
			assert lib.vkr_sample_polygon_batch(C.byref(dev), count, pts.ctypes.data, int(biased), 4, u.ctypes.data, dirs.ctypes.data, info.ctypes.data) == 1
			assert (dirs == 7.0).all() and (info == 7.0).all()
	finally:
		lib.vkr_destroy_device(C.byref(dev))


def _gpu_trace(frame, rays):
	rays = np.ascontiguousarray(rays, dtype=np.float32); out = np.zeros(len(rays), dtype=np.uint8)
	assert frame.lib.vkr_trace_shadow_rays(C.byref(frame.device), C.byref(frame.scene), len(rays), rays.ctypes.data, out.ctypes.data) == 0
	return out


def _frame_inputs(frame, width=96, height=64):
	"""G-buffer surface points of lit pixels (from the device's G-buffer pass) and the lights' world-space polygons (from the constant block)."""
	_, gb = frame.gbuffer_host(width, height)
	gb = np.asarray(gb).reshape(4, height, width, 4)
	valid = np.argwhere(gb[1, :, :, 3] != 0)
	return np.ascontiguousarray(gb[0, valid[:, 0], valid[:, 1], :3], dtype=np.float32), F.light_polygons(frame.constants(width, height), frame.light_count)


@pytest.mark.parametrize("name", F.SHADOW_SCENES)
def test_gpu_shadow_rays_equal_the_oracle_and_meet_the_float64_truth(name, monkeypatch):
	"""Every scene under each BVH builder: the probe's answers equal the oracle's brute force on every ray and shadow_truth on every decided ray."""
	info = H.dataset(name); tris = H.OracleInputs(info).shadow_tris
	lib = api.load_library()
	answers = {}
	for builder in ("sah", "lbvh", "lbvh_gpu"):
		monkeypatch.setenv("VKR_BVH_BUILDER", builder)
		frame = H.open_frame(info)
		try:
			surface, lights = _frame_inputs(frame)
			nodes = _probe_bvh(lib, tris, BUILDERS["sah" if builder == "sah" else "lbvh"])[0]
			for family, rays in F.shadow_ray_families(tris, 7, nodes=nodes, surface=surface, lights=lights).items():
				key = rays.tobytes()
				if key not in answers:
					answers[key] = (oracle.trace_any(tris, rays)[1],) + R.shadow_truth(tris, rays)
				brute, truth, decided = answers[key]
				undecided = F.check_shadow_answers(name, family, rays, _gpu_trace(frame, rays), brute, truth, decided, "GPU probe, " + builder)
				print("%s %-8s %-9s %5d rays, %5.1f %% occluded, undecided %.2f %%" % (name, builder, family, len(rays), 100.0 * brute.mean(), 100.0 * undecided))
		finally:
			frame.close()


def test_gpu_shadow_rays_on_the_city_equal_the_oracle():
	"""The 2.8 M-triangle city of the benchmark, 100 k rays of the families shadow rays to the lights, unusual directions and long rays, against the
	oracle's own BVH (brute force is too slow at this size). No float64 check here: the float64 truth tests every ray against every triangle, 2.8e11
	pairs; the small scenes carry that check."""
	info = H.dataset("city"); tris = H.OracleInputs(info).shadow_tris
	frame = H.open_frame(info)
	try:
		surface, lights = _frame_inputs(frame)
		families = F.shadow_ray_families(tris, 11, n=34000, surface=surface, lights=lights, families=["light", "unusual", "long"])
		for family, rays in families.items():
			t0 = time.time(); got = _gpu_trace(frame, rays); t_gpu = time.time() - t0
			t0 = time.time(); ref = oracle.trace_any(tris, rays, brute=False)[0]; t_cpu = time.time() - t0
			bad = np.nonzero(got != ref)[0]
			print("city %-8s %6d rays, %5.1f %% occluded; GPU %.2f s, oracle %.1f s" % (family, len(rays), 100.0 * ref.mean(), t_gpu, t_cpu))
			assert len(bad) == 0, (family, len(bad), rays[bad[:5]].tolist())
	finally:
		frame.close()
