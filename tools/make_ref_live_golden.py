#!/usr/bin/env python3
"""Freezes what the REFERENCE's own code computes for the tests that compare with it, so that they run without the reference sources.

  python tools/make_ref_live_golden.py     (needs oracle/_ref, built by oracle/build_ref.py from the reference sources)

Output: tests/golden/ref_live.npz (committed), read by
  tests/test_ref_host.py       the reference's loaders and host maths over shim/ (oracle/_ref/libref_host.so): small outputs as they are,
                               large buffers as SHA-256 digests;
  tests/test_ref_shader.py     SHA-256 digests of frames of the reference shader (oracle/_ref/libref_shader.so) at resolutions other than the fixtures' 64x48;
  tests/test_fuzz_parity.py    SHA-256 digests of the reference shader's frames of one seeded run of tools/fuzz_parity.py.
Every comparison stays bit for bit.
"""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tests import harness as H  # noqa: E402
from tests import test_ref_host as T  # noqa: E402
from tests import test_ref_shader as S  # noqa: E402
from tests import test_fuzz_parity as F  # noqa: E402
from tests.ref_frames import host_constants  # noqa: E402
from oracle import ref_binding as R  # noqa: E402
import fuzz_parity  # noqa: E402


def sha256(data):
	return np.frombuffer(hashlib.sha256(bytes(data)).digest(), dtype=np.uint8)


def host_goldens(out):
	ref = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_host.so"))
	ref.ref_probe_material_name.restype = C.c_char_p
	ref.ref_probe_material_name.argtypes = [C.c_uint64]
	ref.ref_probe_sizes.restype = C.c_uint32
	out["struct_sizes"] = np.array([ref.ref_probe_sizes(i) for i in range(5)], dtype=np.uint32)
	for name in T.LOAD_SCENE_DATASETS:
		info = H.dataset(name)
		tri = C.c_uint64(); mat = C.c_uint64(); fs = (C.c_float * 6)(); pos = C.c_void_p(); nuv = C.c_void_p(); mi = C.c_void_p(); soup = C.POINTER(C.c_float)(); ntri = C.c_uint64()
		assert ref.ref_probe_load_scene(info["vks"].encode(), info["textures"].encode(), C.byref(tri), C.byref(mat), fs, C.byref(pos), C.byref(nuv), C.byref(mi), C.byref(soup), C.byref(ntri)) == 0
		n = tri.value
		assert ntri.value == n
		key = "load_scene/%s/" % name
		out[key + "counts"] = np.array([n, mat.value], dtype=np.uint64)
		out[key + "factor_summand"] = np.array(list(fs), dtype=np.float32)
		out[key + "positions_sha256"] = sha256(np.ctypeslib.as_array(C.cast(pos, C.POINTER(C.c_uint32)), (3 * n, 2)))
		out[key + "normals_uv_sha256"] = sha256(np.ctypeslib.as_array(C.cast(nuv, C.POINTER(C.c_uint16)), (3 * n, 4)))
		out[key + "material_indices_sha256"] = sha256(np.ctypeslib.as_array(C.cast(mi, C.POINTER(C.c_uint8)), (n,)))
		out[key + "soup_sha256"] = sha256(np.ctypeslib.as_array(soup, (n, 9)))
		out[key + "material_names"] = np.frombuffer(b"\0".join(ref.ref_probe_material_name(m) for m in range(mat.value)), dtype=np.uint8)
		texels = np.zeros((mat.value, 3, 8), dtype=np.uint16)
		for m in range(mat.value):
			for t in range(3):
				texel = (C.c_uint16 * 8)()
				assert ref.ref_probe_material_texel(C.c_uint64(m), t, texel) == 97
				texels[m, t] = np.frombuffer(bytes(texel), dtype=np.uint16)
		out[key + "material_texels"] = texels
		ref.ref_probe_destroy_scene()
	info = H.dataset("cornell")
	res = C.c_uint32(); t0 = C.c_void_p(); t1 = C.c_void_p(); consts = (C.c_float * 8)()
	assert ref.ref_probe_load_ltc(info["ltc"].encode(), 51, C.byref(res), C.byref(t0), C.byref(t1), consts) == 0
	r = res.value
	out["ltc/resolution"] = np.array([r], dtype=np.uint32)
	out["ltc/table0_sha256"] = sha256(np.ctypeslib.as_array(C.cast(t0, C.POINTER(C.c_uint16)), (51, r, r, 4)))
	out["ltc/table1_sha256"] = sha256(np.ctypeslib.as_array(C.cast(t1, C.POINTER(C.c_uint16)), (51, r, r, 2)))
	out["ltc/constants"] = np.frombuffer(bytes(consts), dtype=np.uint8)
	ref.ref_probe_destroy_ltc()
	digests = set()
	for animate in (0, 1):
		data = C.c_void_p(); mr = (C.c_uint32 * 7)()
		assert ref.ref_probe_load_noise(256, 256, 64, 0, C.byref(data), mr, animate) == 0
		digests.add(sha256(np.ctypeslib.as_array(C.cast(data, C.POINTER(C.c_uint16)), (64 * 256 * 256 * 4,))).tobytes())
		out["noise/constants_animate%d" % animate] = np.array(list(mr), dtype=np.uint32)
		ref.ref_probe_destroy_noise()
	assert len(digests) == 1
	out["noise/texels_sha256"] = np.frombuffer(digests.pop(), dtype=np.uint8)
	lights = 0; matrices = []
	for a, b, vp in T.light_trials():
		if vp is not None:
			light, n = a, b
			ref_bytes = (C.c_uint8 * 160).from_buffer_copy(bytes(light)[:160])
			vw_ref = np.zeros((n, 4), dtype=np.float32); fa_ref = np.zeros((n - 2, 4), dtype=np.float32)
			ref.ref_probe_update_light(ref_bytes, n, vp.ctypes.data, vw_ref.ctypes.data, fa_ref.ctypes.data)
			key = "host_maths/light%03d/" % lights
			out[key + "parameters"] = np.frombuffer(bytes(ref_bytes), dtype=np.uint8)
			out[key + "vertices_world_space"] = vw_ref
			out[key + "fan_areas"] = fa_ref
			lights += 1
		else:
			m = (C.c_float * 16)()
			ref.ref_probe_world_to_projection(C.byref(a), C.c_float(b), m)
			matrices.append(np.frombuffer(bytes(m), dtype=np.float32))
	out["host_maths/world_to_projection"] = np.stack(matrices)
	_, w2p = T.world_to_projection_for_the_inverse()
	inv = (C.c_float * 16)()
	ref.ref_probe_matrix_inverse(w2p.ctypes.data, inv)
	out["matrix_inverse/input"] = w2p
	out["matrix_inverse/output"] = np.frombuffer(bytes(inv), dtype=np.float32)
	for name, lights, width, height in T.CONSTANT_BLOCK_FRAMES:
		out["constants/%s_%d_%dx%d" % (name, lights, width, height)] = np.frombuffer(H.reference_constants(H.dataset(name), width, height, lights, sample_count=4), dtype=np.uint8)


def shader_goldens(out):
	live = {c["name"]: c for c in R.configs()}
	for width, height in S.OTHER_RESOLUTIONS:
		for name in S.OTHER_RESOLUTION_PICKS:
			cfg = live[name]
			info = H.dataset(S.dataset_for(cfg)); oi = H.OracleInputs(info)
			constants = host_constants(info, width, height, cfg["lights"])
			vis = oi.visibility(width, height, constants)
			ref = R.shade(cfg["entry"], width, height, cfg, constants, vis, oi.vks, oi.material_params, oi.noise, oi.ltc0, oi.ltc1, oi.shadow_tris, textures=oi.textures, light_textures=oi.light_textures)
			out["shader/%dx%d/%s" % (width, height, name)] = sha256(ref.tobytes())
	digests = []
	mismatches, compared, _ = fuzz_parity.run(with_reference=True, verbose=False, record_digests=digests, **F.REFERENCE_RUN)
	assert not any(mismatches.values()) and compared["reference vs oracle"] == len(digests)
	out["fuzz/reference_sha256"] = np.array([np.frombuffer(bytes.fromhex(d), dtype=np.uint8) for d in digests])


def main():
	if not R.available() or not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_host.so")):
		raise SystemExit("oracle/_ref is not built (python oracle/build_ref.py, needs the reference sources)")
	out = {}
	host_goldens(out)
	shader_goldens(out)
	path = os.path.join(ROOT, "tests", "golden", "ref_live.npz")
	np.savez_compressed(path, **out)
	print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
	main()
