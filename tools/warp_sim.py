#!/usr/bin/env python3
"""Developer tool: lock-step emulation of the trace warps' loop on the CPU (tools/warp_sim.cpp) to judge scheduling policies of that loop without a GPU.

  python tools/warp_sim.py

Builds the benchmark scene (C3), takes 48 random 8x4 pixel patches of its G-buffer and generates the shadow rays of 12 sample pairs per light in the order the
shading warps submit them; 32 emulated lanes then run the per-lane state machine of vkr_ray_stream.cuh (tickets, occluder cache, slab set-up, node loop with
the postponed leaf, leaf tests, anchored starts) with phases costed in warp instructions taken from the kernel's SASS. The baseline reproduces what ncu
measured on the GPU in an earlier round (24.2 vs 23.7 lanes per node step, 13.2 vs 13.4 lanes per triangle test, 4444 vs ~4270 warp instructions per 32 rays), which
is what makes its verdicts on variants (refill thresholds, one leaf per round, anchored rays) worth having before GPU time is spent on them."""
import ctypes as C, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
from tests import harness as H
from tests.ref_frames import host_constants
from vulkan_renderer_b200 import api, synth
P = C.POINTER
lights = 8; width, height = 1920, 1080
info = synth.build_dataset('/tmp/vkr_b200_data/city', 'city')
constants = host_constants(info, width, height, lights)
oi = H.OracleInputs(info)
gb = oi.gbuffer(width, height, constants, oi.visibility(width, height, constants))
lib = api.load_library()
tris = np.ascontiguousarray(oi.shadow_tris, dtype=np.float32)
nodes = P(C.c_float)(); tri = P(C.c_float)(); ids = P(C.c_uint32)(); nc = C.c_uint64(); md = C.c_uint32()
assert lib.vkr_bvh_build_probe(tris.ctypes.data, len(tris), C.byref(nodes), C.byref(nc), C.byref(tri), C.byref(ids), C.byref(md)) == 0
cb = np.frombuffer(constants, dtype=np.uint8)
lv = np.zeros((lights, 4, 4), dtype=np.float32)
for l in range(lights):
	base = 256 + 320 * l + 160 + 64
	lv[l] = np.frombuffer(cb[base:base + 64].tobytes(), dtype=np.float32).reshape(4, 4)
rng = np.random.default_rng(9)
origins = []; rays = []
SPP = 12
for patch in range(48):
	px = int(rng.integers(0, width // 8)) * 8; py = int(rng.integers(0, height // 4)) * 4
	pix = [(py + (lane >> 3), px + (lane & 7)) for lane in range(32)]
	base = len(origins)
	for (y, x) in pix: origins.append(gb[0, y, x, :3])
	valid = [gb[1, y, x, 3] != 0 for (y, x) in pix]
	for l in range(lights):
		for s in range(SPP):
			for j in range(2):
				for lane in range(32):
					if not valid[lane]: continue
					y, x = pix[lane]
					uv = rng.random(2)
					pt = lv[l, 0, :3] + uv[0] * (lv[l, 1, :3] - lv[l, 0, :3]) + uv[1] * (lv[l, 3, :3] - lv[l, 0, :3])
					e = pt - gb[0, y, x, :3]; dist = float(np.linalg.norm(e)); d = e / dist
					if float(d @ gb[1, y, x, :3]) <= 0: continue
					rays.append((base + lane, d[0], d[1], d[2], dist, float(l)))
origins = np.ascontiguousarray(np.array(origins, dtype=np.float32)); rays = np.ascontiguousarray(np.array(rays, dtype=np.float32))
print('pixels', len(origins), 'rays', len(rays))
so = os.path.join(ROOT, "tools", "build", "libwarp_sim.so")
os.makedirs(os.path.dirname(so), exist_ok=True)
subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-mfma", "-mavx2", "-I", os.path.join(ROOT, "vulkan_renderer_b200", "csrc"), os.path.join(ROOT, "tools", "warp_sim.cpp"), "-o", so])
sim = C.CDLL(so)
paths = np.zeros((len(origins), 22), dtype=np.uint32)
sim.prepare(nodes, origins.ctypes.data_as(C.c_void_p), C.c_uint32(len(origins)), lv.ctypes.data_as(C.c_void_p), C.c_uint32(len(rays)), rays.ctypes.data_as(C.c_void_p), paths.ctypes.data_as(C.c_void_p))
for name, prm in (("baseline (node loop left below 16 lanes, refill at once, all leaves per round, plain)", (16, 1, 0, 0, 0)), ("node loop left below 8 lanes", (8, 1, 0, 0, 0)), ("node loop left below 24 lanes", (24, 1, 0, 0, 0)),
	("refill once 8 lanes are free", (16, 8, 0, 0, 0)), ("one leaf per round", (16, 1, 1, 0, 0)), ("pooled triangle tests", (16, 1, 0, 0, 1)), ("pooled triangle tests, one leaf per round", (16, 1, 1, 0, 1)),
	("anchored", (16, 1, 0, 1, 0)), ("anchored, one leaf per round", (16, 1, 1, 1, 0)), ("anchored, refill 8, one leaf per round", (16, 8, 1, 1, 0)), ("anchored, pooled triangle tests, one leaf per round", (16, 1, 1, 1, 1)),
	("anchored, one leaf per round, loop left below 20", (20, 1, 1, 1, 0)), ("anchored, one leaf per round, loop left below 24", (24, 1, 1, 1, 0)), ("one leaf per round, loop left below 20", (20, 1, 1, 0, 0)),
	("anchored, pooled triangle tests, one leaf per round, loop left below 12", (12, 1, 1, 1, 1)), ("anchored, pooled triangle tests, one leaf per round, loop left below 20", (20, 1, 1, 1, 1))):
	out = (C.c_double * 16)(); p = (C.c_int * 5)(*prm)
	sim.simulate(nodes, tri, origins.ctypes.data_as(C.c_void_p), C.c_uint32(len(origins)), paths.ctypes.data_as(C.c_void_p), C.c_uint32(len(rays)), rays.ctypes.data_as(C.c_void_p), p, out)
	o = list(out)
	print('%-78s warp-instr per 32 rays %7.0f | lanes/node step %.1f lanes/tri test %.1f lanes/setup %.1f | visits/ray %.1f tri tests/ray %.1f occluded %.2f | lane-instr/ray %.0f rounds/32 rays %.1f' % (name, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7], o[8]))
