#!/usr/bin/env python3
"""Freezes outputs of the REFERENCE's shader sources (compiled as C++ by oracle/build_ref.py) as golden fixtures.

  python tools/make_ref_golden.py        (needs /root/reference; run in the build container)

For every configuration in oracle/_ref/configs.json a 64x48 frame of a seeded synthetic scene is shaded by the
reference shader and kept as the SHA-256 of its float32 RGBA bytes; inputs are identified by sha256 of the scene file and the constant block is stored, so a drift
of the synthetic-data generator is detected instead of silently changing the fixture's meaning.
Output: tests/golden/ref_shader.npz (committed).
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import harness as H  # noqa: E402
from tests.ref_frames import WIDTH, HEIGHT, dataset_for, frame_sha256, host_constants  # noqa: E402
from oracle import ref_binding as R  # noqa: E402


def main():
	if not R.available():
		sys.path.insert(0, os.path.join(ROOT, "oracle"))
		import build_ref
		build_ref.build()
	out = {}
	for cfg in R.configs():
		name = dataset_for(cfg)
		info = H.dataset(name); oi = H.OracleInputs(info)
		constants = host_constants(info, WIDTH, HEIGHT, cfg["lights"], frame_bits=cfg.get("frame_bits", 0))
		vis = oi.visibility(WIDTH, HEIGHT, constants)
		ref = R.shade(cfg["entry"], WIDTH, HEIGHT, cfg, constants, vis, oi.vks, oi.material_params, oi.noise, oi.ltc0, oi.ltc1, oi.shadow_tris, textures=oi.textures, light_textures=oi.light_textures)
		key = cfg["name"]
		out[key + "/rgba_sha256"] = np.frombuffer(frame_sha256(ref), dtype=np.uint8)   # the frame itself: bit-identical or not, in 32 bytes
		out[key + "/visibility"] = vis
		out[key + "/constants"] = np.frombuffer(constants, dtype=np.uint8)
		out[key + "/vks_sha256"] = np.frombuffer(hashlib.sha256(open(info["vks"], "rb").read()).digest(), dtype=np.uint8)
		print(key, "mean radiance", float(ref[..., :3].mean()))
	np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ref_shader.npz"), **out)


if __name__ == "__main__":
	main()
