"""The GPU's related-work samplers through their probe (vkr_sample_related_work_batch: the prepare() and sample() of the related-work tile kernel, one
thread per sample), with the cases and random numbers of tests/test_related_work_float64.py: directions, densities, GGX density factor and culling
bit for bit against the oracle, and independently through the same float64 checks (tolerances and recorded exceptions are justified there)."""
import ctypes as C

import numpy as np
import pytest

from tests import test_related_work_float64 as F
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu


def _device():
	lib = api.load_library(); dev = api.Device()
	assert lib.vkr_create_device(C.byref(dev), 0, None) == 0
	return lib, dev


def _probe(lib, dev, technique, maxv, block, position, frame, u):
	"""(return code, lit, dirs, densities, GGX density factor); the directions and densities of a culled light stay 0."""
	u = np.ascontiguousarray(u, dtype=np.float32); n = len(u)
	position = np.ascontiguousarray(position, dtype=np.float32); frame = np.ascontiguousarray(frame, dtype=np.float32)
	dirs = np.zeros((n, 3), dtype=np.float32); dens = np.zeros(n, dtype=np.float32)
	ggx = C.c_float(0.0); lit = C.c_int32(-1)
	blk = (C.c_uint8 * len(block)).from_buffer_copy(block)
	rc = lib.vkr_sample_related_work_batch(C.byref(dev), technique, maxv, blk, len(block), position.ctypes.data, frame.ctypes.data,
		n, u.ctypes.data, dirs.ctypes.data, dens.ctypes.data, C.byref(ggx), C.byref(lit))
	return rc, lit.value, dirs, dens, ggx.value


def _same_bits(a, b):
	a = np.asarray(a, dtype=np.float32); b = np.asarray(b, dtype=np.float32)
	return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


@pytest.mark.parametrize("technique", sorted(F.TECHNIQUES))
def test_gpu_related_work_samplers_equal_the_oracle_and_meet_the_float64_references(technique):
	lib, dev = _device()
	try:
		stats = {}; checked = culled = 0
		for dataset, maxv in F.DATA_SETS:
			for case in F.cases(dataset, maxv):
				u, kind = F.random_numbers(case, technique)
				ref = F.run(technique, case, u)
				rc, lit, dirs, dens, ggx = _probe(lib, dev, technique, maxv, case["block"], case["position"], case["frame"], u)
				label = (technique, dataset, case["light"], case["family"])
				assert rc == 0 and lit == (ref is not None), (label, rc, lit)
				if ref is None:
					culled += 1
					assert ggx == 0.0 and not dirs.any() and not dens.any()
				else:
					assert _same_bits(dirs, ref[0]).all(), (label, u[~_same_bits(dirs, ref[0]).all(1)][:4])
					assert _same_bits(dens, ref[1]).all(), (label, u[~_same_bits(dens, ref[1])][:4])
					assert _same_bits(ggx, ref[2]), (label, ggx, ref[2])
					checked += 1
				F.check_case(technique, case, u, kind, None if ref is None else (dirs, dens, ggx), stats)
		F.report("GPU probe, technique %d (%s): %d cases lit, %d culled" % (technique, F.TECHNIQUES[technique], checked, culled), stats)
		F.check_totals(technique, stats)
		assert checked > 0
	finally:
		lib.vkr_destroy_device(C.byref(dev))


def test_gpu_related_work_probe_refuses_what_it_cannot_sample():
	"""A technique above 10, a vertex bound outside 3..7, a block of the wrong size, a null device, block or frame: refused, the outputs stay as they were."""
	lib, dev = _device()
	try:
		case = F.cases("mini_city", 4)[0]
		u = np.full((4, 2), 0.5, dtype=np.float32)
		frame = np.ascontiguousarray(case["frame"], dtype=np.float32); position = np.ascontiguousarray(case["position"], dtype=np.float32)
		def untouched(**kw):
			dirs = np.full((4, 3), 7.0, dtype=np.float32); dens = np.full(4, 7.0, dtype=np.float32)
			ggx = C.c_float(7.0); lit = C.c_int32(7)
			args = dict(device=C.byref(dev), technique=4, maxv=4, block=(C.c_uint8 * len(case["block"])).from_buffer_copy(case["block"]), bytes=len(case["block"]), frame=frame.ctypes.data)
			args.update(kw)
			rc = lib.vkr_sample_related_work_batch(args["device"], args["technique"], args["maxv"], args["block"], args["bytes"], position.ctypes.data, args["frame"],
				4, u.ctypes.data, dirs.ctypes.data, dens.ctypes.data, C.byref(ggx), C.byref(lit))
			assert rc == 1 and (dirs == 7.0).all() and (dens == 7.0).all() and ggx.value == 7.0 and lit.value == 7, kw
		untouched(technique=11)
		untouched(technique=12)
		untouched(maxv=2)
		untouched(maxv=8)
		untouched(maxv=5)            # the block of bound 4 is not one of bound 5
		untouched(bytes=len(case["block"]) - 16)
		untouched(device=None)
		untouched(block=None)
		untouched(frame=None)
		# the same call with valid arguments samples
		rc, lit, dirs, dens, ggx = _probe(lib, dev, 4, 4, case["block"], case["position"], case["frame"], u)
		assert rc == 0 and lit == 1 and np.isfinite(dirs).all() and (dens > 0).all()
	finally:
		lib.vkr_destroy_device(C.byref(dev))
