#!/usr/bin/env python3
"""Freezes stbi_write_jpg's output (the reference's stb_image_write.h, oracle/_ref/libref_jpeg.so from oracle/build_ref_jpeg.py) into
tests/golden/ref_jpeg.npz for tests/test_jpeg_on_host.py and tests/test_gpu_zzzzzzzzzzzz_jpeg.py.

Cases (tests/jpeg_cases.py): every small size x quality corner x content kind, the large sizes at a few qualities, and one ffpad image: the first
seed whose 16 x 16 noise at quality 50 ends its entropy-coded segment with a stuffed 0xFF in the padding byte (file tail FF 00 FF D9). Inputs are
regenerated from their seeds; full bytes are stored for images of at most FULL_BYTES_MAX_PIXELS pixels, length and SHA-256 for the others.

usage: python tools/make_ref_jpeg_golden.py
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import jpeg_cases as J  # noqa: E402


def main():
	stb = J.stb_encoder()
	if stb is None:
		raise SystemExit("oracle/_ref/libref_jpeg.so is missing: run `python oracle/build_ref_jpeg.py` where the reference is present")
	cases = [(k, w, h, q) for (w, h) in J.SMALL_SIZES for q in J.QUALITIES for k in J.KINDS] + J.LARGE_CASES
	rows = [dict(kind=k, width=w, height=h, quality=q, seed=J.case_seed(k, w, h, q)) for k, w, h, q in cases]
	for seed in range(100000):
		data = stb(J.make_image("ffpad", 16, 16, seed), 50)
		if data.endswith(b"\xff\x00\xff\xd9"):
			rows.append(dict(kind="ffpad", width=16, height=16, quality=50, seed=seed))
			break
	else:
		raise SystemExit("no ffpad seed found")
	arrays = {}
	for i, r in enumerate(rows):
		data = stb(J.make_image(r["kind"], r["width"], r["height"], r["seed"]), r["quality"])
		r.update(size=len(data), sha256=J.digest(data), full=r["width"] * r["height"] <= J.FULL_BYTES_MAX_PIXELS)
		if r["full"]:
			arrays["file_%d" % i] = np.frombuffer(data, dtype=np.uint8)
	os.makedirs(os.path.dirname(J.GOLDEN), exist_ok=True)
	np.savez_compressed(J.GOLDEN, cases=np.array(json.dumps(rows)), **arrays)
	print("%d cases (%d with full bytes, ffpad seed %d) -> %s, %d bytes" % (len(rows), len(arrays), rows[-1]["seed"], J.GOLDEN, os.path.getsize(J.GOLDEN)))


if __name__ == "__main__":
	main()
