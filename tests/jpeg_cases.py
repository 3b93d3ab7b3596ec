"""The JPEG encoder's test images (tests/test_jpeg_on_host.py, tests/test_gpu_zzzzzzzzzzzz_jpeg.py, tools/make_ref_jpeg_golden.py): each image is made
from (kind, width, height, seed) with numpy's RandomState, whose stream numpy keeps stable across versions, so tests/golden/ref_jpeg.npz stores only
stb_image_write's outputs.

Kinds: flat (every block codes an EOB only), gradient (smooth ramps, short codes), noise (uniform noise: long codes, ZRL runs, many stuffed 0xFF),
saturated (every channel 0 or 255: extreme chroma), ffpad (noise chosen so that the byte holding the final 1-bit padding is 0xFF, see GOLDEN).
"""
import ctypes as C
import hashlib
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_jpeg.npz")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_jpeg.so")
HOST_LIB = os.path.join(ROOT, "tests", "build", "libjpeg_on_host.so")
KINDS = ("flat", "gradient", "noise", "saturated")
QUALITIES = (0, 1, 49, 50, 70, 90, 91, 100, -7)             # 90: the last subsampled quality; -7: clamped to 1
SMALL_SIZES = ((1, 1), (7, 5), (8, 8), (15, 17), (16, 16), (17, 33), (64, 48), (250, 130))
FULL_BYTES_MAX_PIXELS = 64 * 48                              # larger images: length and SHA-256 only
LARGE_CASES = [(k, w, h, q) for (w, h) in ((1920, 1080), (1921, 1081)) for q in (70, 91) for k in ("gradient", "noise", "saturated")] \
	+ [(k, 3840, 2160, 70) for k in ("gradient", "noise")]


def make_image(kind, width, height, seed):
	"""[height, width, 3] uint8"""
	rs = np.random.RandomState(seed)
	if kind == "flat":
		return np.broadcast_to(rs.randint(0, 256, 3).astype(np.uint8), (height, width, 3)).copy()
	if kind == "gradient":
		a, b, c = rs.randint(1, 8, 3)
		y, x = np.mgrid[0:height, 0:width]
		return np.stack([(a * x + 3 * y) % 256, (b * y + x // 2) % 256, (c * (x + y)) % 256], axis=-1).astype(np.uint8)
	if kind in ("noise", "ffpad"):
		return rs.randint(0, 256, (height, width, 3)).astype(np.uint8)
	if kind == "saturated":
		return (rs.randint(0, 2, (height, width, 3)) * 255).astype(np.uint8)
	raise ValueError(kind)


def case_seed(kind, width, height, quality):
	return (KINDS.index(kind) * 1000003 + width * 7919 + height * 104729 + (quality + 16) * 31) % (2 ** 31)


def digest(data):
	return hashlib.sha256(data).hexdigest()


def _encoder(lib, name):
	f = getattr(lib, name)
	f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
	f.restype = C.c_int

	def encode(image, quality):
		image = np.ascontiguousarray(image, dtype=np.uint8)
		height, width = image.shape[:2]
		capacity = 1024 + 8 * image.size
		out = np.empty(capacity, dtype=np.uint8)
		size = C.c_size_t(0)
		rc = f(image.ctypes.data, width, height, int(quality), out.ctypes.data, capacity, C.byref(size))
		return rc, out[:size.value].tobytes()
	return encode


def stb_encoder():
	"""stbi_write_jpg of the reference's stb_image_write.h (oracle/_ref/libref_jpeg.so, built by oracle/build_ref_jpeg.py), or None where it was not built"""
	if not os.path.exists(REF_LIB):
		return None
	encode = _encoder(C.CDLL(REF_LIB), "ref_write_jpg")

	def stb(image, quality):
		ok, data = encode(image, quality)
		assert ok == 1
		return data
	return stb


def host_library():
	if not os.path.exists(HOST_LIB):
		import __graft_entry__ as G
		G.build_device_on_host()
	return C.CDLL(HOST_LIB)


def host_encoder():
	"""vkr_jpeg.cuh compiled for the CPU (tests/jpeg_on_host.cpp): (image, quality) -> (return code, bytes)"""
	return _encoder(host_library(), "vkr_host_encode_jpg")


def load_golden():
	"""[(case dict, full bytes or None)]: case = kind, width, height, quality, seed, size, sha256"""
	with np.load(GOLDEN, allow_pickle=False) as z:
		cases = json.loads(str(z["cases"]))
		return [(c, z["file_%d" % i].tobytes() if c["full"] else None) for i, c in enumerate(cases)]
