#!/usr/bin/env python3
"""Compiles the REFERENCE's unchanged stb_image_write.h (v1.14, the JPEG writer of its screenshots) where it lies, together with oracle/ref_jpeg.c,
which writes into a memory buffer, into oracle/_ref/libref_jpeg.so (TEST INFRASTRUCTURE). tests/test_jpeg_on_host.py and
tools/make_ref_jpeg_golden.py hold csrc/vkr_jpeg.cuh against it byte for byte.

gcc on x86-64 with -ffp-contract=off and neither -mfma nor -ffast-math, so that stb's float arithmetic is plain IEEE binary32. Skipped where the
reference is absent, like the recipes of oracle/build_ref.py.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/src"
OUT = os.path.join(HERE, "_ref")


def build():
	if not os.path.exists(os.path.join(REF_SRC, "stb_image_write.h")):
		print("build_ref_jpeg: the reference's stb_image_write.h is not present; nothing to build")
		return None
	os.makedirs(OUT, exist_ok=True)
	lib = os.path.join(OUT, "libref_jpeg.so")
	subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-I", REF_SRC,
		os.path.join(HERE, "ref_jpeg.c"), "-lm", "-o", lib])
	print("build_ref_jpeg: stb_image_write's JPEG writer -> %s" % lib)
	return lib


if __name__ == "__main__":
	build()
