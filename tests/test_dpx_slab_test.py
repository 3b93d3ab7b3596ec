"""The slab test of the shading kernel's trace warps with signed-integer min / max (vkr_trace.cuh: make_clamped_slabs() + ray_box_pair<true>, one
VIMNMX3 + one VIMNMX per child and side on sm_90a) against the fmaxf form it replaced, on the CPU (tests/dpx_slab_on_host.cpp compiles the header
for the host, where the DPX intrinsics are plain C++ with the same integer semantics).

- Pair test, random shading-domain rays (normalised directions, tmin = 1e-3 < tmax; some with exactly zero components of either sign; boxes ahead
  of and behind the origin): the integer min / max gives the fmaxf answers bit for bit on the same set-up; against the unclamped set-up the trace
  warps ran before, decisions and entry distances differ only on rays with a zero component, and there only by culling boxes whose slab of that
  axis does not hold the origin; no box the exact float64 slab test accepts with a margin above the rounding is culled.
- Per-thread traversal over interleaved pairs (occluded_interleaved<true>, the reference form of the trace warps' loop) on the ray families of
  tests/test_float64_references.py: the brute force's answer on every ray, and the same pairs visited as the fmaxf form on every ray the trace warps
  can get (tmin > 0) without a direction component below 2^-64 in magnitude.
"""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import binding as oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libdpx_slab_on_host.so")
TWO_M64 = 2.0 ** -64


def _lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	return C.CDLL(LIB_PATH)


def _ptr(a):
	return a.ctypes.data_as(C.c_void_p)


def _pair_inputs(seed, n=200000):
	"""rays [n, 8] and one interleaved pair [n, 16] per ray, float32; zero_axis [n, 3]: the components that are exactly +-0."""
	rng = np.random.default_rng(seed)
	o = rng.uniform(-20.0, 20.0, (n, 3))
	d = rng.normal(size=(n, 3))
	kind = rng.integers(0, 4, n)                        # 0: generic; 1: one zero component; 2: two; 3: an axis, either sign
	for k in (1, 2):
		rows = np.nonzero(kind == k)[0]
		for a in range(k):
			d[rows, (rng.integers(0, 3, len(rows)) + a) % 3] = 0.0
	axis_rows = np.nonzero(kind == 3)[0]
	d[axis_rows] = np.eye(3)[rng.integers(0, 3, len(axis_rows))] * rng.choice([-1.0, 1.0], (len(axis_rows), 1))
	d /= np.linalg.norm(d, axis=1, keepdims=True)
	d = d.astype(np.float32)
	zeros = d == 0.0
	d[zeros] = np.where(rng.uniform(size=zeros.sum()) < 0.5, np.float32(0.0), np.float32(-0.0))   # +0 and -0
	tmax = rng.uniform(0.01, 40.0, n)
	rays = np.concatenate([o, d.astype(np.float64), np.full((n, 1), 1e-3), tmax[:, None]], axis=1).astype(np.float32)
	boxes = []
	for _ in range(2):
		s = rng.uniform(-25.0, 45.0, (n, 1))           # along the ray, behind the origin for s < 0
		c = o + d.astype(np.float64) * s + rng.normal(scale=3.0, size=(n, 3))
		near_origin = rng.uniform(size=n) < 0.25       # boxes whose zero-component slabs hold the origin or just miss it
		c[near_origin] = o[near_origin] + rng.normal(scale=1.0, size=(near_origin.sum(), 3))
		if boxes:                                      # siblings that overlap, as in a BVH: both children hit, the order decides
			sibling = rng.uniform(size=n) < 0.5
			c[sibling] = boxes[0][0][sibling] + rng.normal(scale=1.0, size=(sibling.sum(), 3))
		h = np.exp(rng.uniform(np.log(0.01), np.log(6.0), (n, 3)))
		boxes.append((c.astype(np.float32), h.astype(np.float32)))
	(c0, h0), (c1, h1) = boxes
	pairs = np.zeros((n, 16), dtype=np.float32)
	pairs[:, 0:6:2] = c0; pairs[:, 1:6:2] = c1; pairs[:, 6:12:2] = h0; pairs[:, 7:12:2] = h1
	return rays, pairs, zeros, boxes


def _exact_accepts(rays, c, h):
	"""float64 slab test of the segment (tmin, tmax) against each box, only where it is decided with a margin above fp32 rounding: True = the ray
	crosses the box with room to spare (those must never be culled)."""
	o = rays[:, 0:3].astype(np.float64); d = rays[:, 3:6].astype(np.float64); c = c.astype(np.float64); h = h.astype(np.float64)
	tmin = rays[:, 6].astype(np.float64); tmax = rays[:, 7].astype(np.float64)
	scale = np.abs(c) + np.abs(o) + h
	eps = 2.0 ** -20 * scale                                    # a few ulp of the coordinates: the rounding of the fp32 slab distances
	nonzero = d != 0.0
	safe_d = np.where(nonzero, d, 1.0)
	lo = np.where(nonzero, np.minimum((c - h - o) / safe_d, (c + h - o) / safe_d), -np.inf)
	hi = np.where(nonzero, np.maximum((c - h - o) / safe_d, (c + h - o) / safe_d), np.inf)
	err = np.where(nonzero, eps / np.abs(safe_d), 0.0).max(axis=1)
	inside = np.where(nonzero, True, np.abs(o - c) < h - eps).all(axis=1)   # a zero component: the origin must lie in the slab
	t_in = np.maximum(lo.max(axis=1), tmin); t_out = np.minimum(hi.min(axis=1), tmax)
	return inside & (t_out - t_in > 4.0 * err + 1e-6)


def test_integer_pair_test_gives_the_fmaxf_decisions():
	lib = _lib()
	rays, pairs, zeros, boxes = _pair_inputs(11)
	n = len(rays)
	hits = np.zeros((n, 6), dtype=np.uint8); tn = np.zeros((n, 6), dtype=np.float32)
	lib.vkr_dpx_pair_tests(C.c_uint32(n), _ptr(rays), _ptr(pairs), _ptr(hits), _ptr(tn))
	old, new, fmax_clamped = hits[:, 0:2].astype(bool), hits[:, 2:4].astype(bool), hits[:, 4:6].astype(bool)
	t_old, t_new, t_fmax_clamped = tn[:, 0:2], tn[:, 2:4], tn[:, 4:6]
	# (1) integer min / max == fmaxf / fminf on the clamped set-up: decisions and entry distances, bit for bit
	assert np.array_equal(new, fmax_clamped)
	assert np.array_equal(t_new.view(np.uint32), t_fmax_clamped.view(np.uint32))
	assert np.isfinite(t_new).all() and (t_new >= np.float32(1e-3)).all()
	# (2) against the unclamped set-up: identical on rays without a zero component
	plain = ~zeros.any(axis=1)
	assert plain.sum() > n // 5 and (~plain).sum() > n // 2
	assert np.array_equal(new[plain], old[plain])
	assert np.array_equal(t_new[plain].view(np.uint32), t_old[plain].view(np.uint32))
	# (3) rays with a zero component: the clamp only culls (the unclamped test drops that axis), and only boxes whose slab misses the origin
	assert not (new & ~old).any()
	culled = old & ~new
	assert culled[~plain].sum() > 1000 and not culled[plain].any()
	for k, (c, h) in enumerate(boxes):
		rows = np.nonzero(culled[:, k])[0]
		o = rays[rows, 0:3].astype(np.float64)
		outside = (zeros[rows] & (np.abs(o - c[rows]) > h[rows].astype(np.float64) * (1.0 - 1e-6))).any(axis=1)
		assert outside.all(), rays[rows[~outside][:5]].tolist()
	# the nearer child first: the same order wherever both ways hit both children
	both = old.all(axis=1) & new.all(axis=1)
	assert both.sum() > 300
	assert np.array_equal((t_new[both, 1] < t_new[both, 0]), (t_old[both, 1] < t_old[both, 0]))
	# (4) conservative: no box the exact float64 test accepts with a margin is culled
	for k, (c, h) in enumerate(boxes):
		accepts = _exact_accepts(rays, c, h)
		assert accepts.sum() > n // 50 and accepts[~plain].sum() > n // 200
		missed = np.nonzero(accepts & ~new[:, k])[0]
		assert len(missed) == 0, rays[missed[:5]].tolist()


def test_integer_pair_test_on_special_values():
	"""Boxes at the edges of the integer ordering and of the clamp: zero components against boxes that do or do not hold the origin, or hold it
	exactly on a face (a grazing ray: which side is kept depends on the sign of the zero, the padding of the boxes covers it), far distances of
	exactly zero and negative ones, and tmax = +infinity."""
	lib = _lib()
	f = np.float32
	rays, pairs = [], []
	def add(o, d, tmax, c0, h0, c1, h1):
		rays.append(list(o) + list(d) + [1e-3, tmax])
		p = np.zeros(16, dtype=np.float32)
		p[0:6:2] = c0; p[1:6:2] = c1; p[6:12:2] = h0; p[7:12:2] = h1
		pairs.append(p)
	add((0, 0, 0), (0, 0, 1), 10, (0, 0, 5), (1, 1, 1), (3, 0, 5), (1, 1, 1))              # child 1: its x slab [2, 4] misses the origin
	add((0, 0, 0), (0, 0, 1), 10, (1, 0, 5), (1, 1, 1), (-1, 0, 5), (1, 1, 1))             # the origin on face x = 0 of both; d.x = +0 keeps child 0
	add((0, 0, 0), (-0.0, 0, 1), 10, (1, 0, 5), (1, 1, 1), (-1, 0, 5), (1, 1, 1))          # ... and d.x = -0 child 1
	# tmax = inf, boxes far away: the zero components bound the far distance by h * 2^64 (vkr_trace.cuh: make_clamped_slabs)
	add((0, 0, 0), (0, -0.0, 1), np.inf, (0, 0, 1e15), (1, 1, 1), (0, 0, 1e30), (1, 1, 1))
	add((0, 0, 0), (1, 0, 0), 10, (-1, 0, 0), (1, 1, 1), (-3, 0, 0), (1, 1, 1))            # far distance exactly 0, and negative (behind)
	add((0, 0, 0), (-1, 0, 0), 10, (-0.0, 0, 0), (0.0, 1, 1), (2, 0, 0), (2, 1, 1))         # a flat box through the origin; a box with its far face there
	rays = np.array(rays, dtype=np.float32); pairs = np.array(pairs, dtype=np.float32)
	n = len(rays)
	hits = np.zeros((n, 6), dtype=np.uint8); tn = np.zeros((n, 6), dtype=np.float32)
	lib.vkr_dpx_pair_tests(C.c_uint32(n), _ptr(rays), _ptr(pairs), _ptr(hits), _ptr(tn))
	assert np.array_equal(hits[:, 2:4], hits[:, 4:6]) and np.array_equal(tn[:, 2:4].view(np.uint32), tn[:, 4:6].view(np.uint32))
	new = hits[:, 2:4].astype(bool)
	assert new.tolist() == [[True, False], [True, False], [False, True], [True, False], [False, False], [False, False]]
	assert tn[0, 2] == f(4.0) and tn[1, 2] == f(4.0) and tn[2, 3] == f(4.0) and tn[3, 2] == f(1e15)


def _traversal_cases():
	from tests.test_float64_references import SHADOW_SCENES
	return SHADOW_SCENES


@pytest.mark.parametrize("name", _traversal_cases())
def test_integer_traversal_answers_and_visits_like_the_fmaxf_one(name):
	from tests.test_float64_references import scene_inputs, shadow_ray_families
	from tests.test_host_logic import _probe_bvh, BUILDERS
	from vulkan_renderer_b200 import api
	dev = _lib(); lib = api.load_library()
	tris, surface, lights = scene_inputs(name)
	nodes, slots, ids, depth = _probe_bvh(lib, tris, BUILDERS["sah"])
	nodes = np.ascontiguousarray(nodes, dtype=np.float32); slots = np.ascontiguousarray(slots, dtype=np.float32)
	families = shadow_ray_families(tris, 7, nodes=nodes, surface=surface, lights=lights)
	compared = 0
	for family, rays in families.items():
		m = len(rays)
		brute = oracle.trace_any(tris, rays)[1].astype(bool)
		out_f = np.zeros(m, dtype=np.uint8); out_i = np.zeros(m, dtype=np.uint8)
		v_f = np.zeros(m, dtype=np.uint32); v_i = np.zeros(m, dtype=np.uint32)
		dev.vkr_dpx_trace_interleaved(_ptr(nodes), C.c_uint64(len(nodes)), _ptr(slots), C.c_uint32(m), _ptr(rays), _ptr(out_f), _ptr(out_i), _ptr(v_f), _ptr(v_i))
		bad = np.nonzero(out_i.astype(bool) != brute)[0]
		assert len(bad) == 0, (name, family, len(bad), rays[bad[:5]].tolist())
		assert np.array_equal(out_f.astype(bool), brute), (name, family)
		d = np.abs(rays[:, 3:6].astype(np.float64))
		domain = (rays[:, 6] > 0) & (rays[:, 7] > rays[:, 6]) & (d >= TWO_M64).all(axis=1)
		diff = np.nonzero(domain & (v_f != v_i))[0]
		assert len(diff) == 0, (name, family, len(diff), rays[diff[:5]].tolist())
		compared += int(domain.sum())
		print("%s %-9s %5d rays, %5d compared visit for visit; %d / %d pairs visited (fmaxf / integer)" % (
			name, family, m, domain.sum(), v_f.sum(), v_i.sum()))
	assert compared > 1500
