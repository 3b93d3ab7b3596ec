"""The JPEG encoder (vulkan_renderer_b200/csrc/vkr_jpeg.cuh) compiled for the CPU (tests/jpeg_on_host.cpp: the kernels' stages as loops) against
stbi_write_jpg of the reference's stb_image_write.h, byte for byte, and the refusals of the C-ABI that come before any device work.

1. the host build writes every file of tests/golden/ref_jpeg.npz (stb's output, frozen by tools/make_ref_jpeg_golden.py) byte for byte.
2. where oracle/_ref/libref_jpeg.so was built: 2000 seeded random images of 1..96 pixels per side and 24 up to 1024, qualities -5..105, every
   content kind, byte-identical to stb.
3. refusals: zero and oversized sizes, NULL pointers, a capacity one byte short (nothing written, the size reported); vkr_encode_jpg and
   vkr_write_jpg refuse the same before touching the device, and vkr_write_jpg an unwritable path.
The -m gpu tests hold the kernels against this build (tests/test_gpu_zzzzzzzzzzzz_jpeg.py).
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests import jpeg_cases as J
from vulkan_renderer_b200 import api

RANDOM_IMAGES, LARGE_RANDOM_IMAGES = 2000, 24


@pytest.fixture(scope="module")
def host():
	return J.host_encoder()


@pytest.fixture(scope="module")
def golden():
	return J.load_golden()


def test_golden_covers_the_corners(golden):
	cases = [c for c, _ in golden]
	assert {c["quality"] for c in cases} >= set(J.QUALITIES)
	assert {c["kind"] for c in cases} == set(J.KINDS) | {"ffpad"}
	assert {(c["width"], c["height"]) for c in cases} >= set(J.SMALL_SIZES) | {(1920, 1080), (1921, 1081), (3840, 2160)}
	ffpad = [data for c, data in golden if c["kind"] == "ffpad"]
	assert len(ffpad) == 1 and ffpad[0].endswith(b"\xff\x00\xff\xd9")
	# uniform noise at quality 100 codes long runs of zeros (ZRL) and stuffs many 0xFF
	noisy = [data for c, data in golden if c["kind"] == "noise" and c["quality"] == 100 and data is not None and c["width"] == 64]
	assert noisy and noisy[0][607:-2].count(b"\xff\x00") > 20


def test_host_build_writes_the_golden_files(host, golden):
	for case, data in golden:
		rc, out = host(J.make_image(case["kind"], case["width"], case["height"], case["seed"]), case["quality"])
		assert rc == 0 and len(out) == case["size"], case
		if data is not None:
			assert out == data, case
		assert J.digest(out) == case["sha256"], case


def test_header_layout(host):
	"""SOI, JFIF 1.1, one DQT with both tables, SOF0 with 4:2:0 up to quality 90 and 4:4:4 above, one DHT, SOS; EOI at the end"""
	image = J.make_image("noise", 40, 24, 5)
	for quality, sampling in ((90, 0x22), (91, 0x11), (0, 0x22), (-3, 0x22)):
		_, out = host(image, quality)
		assert out[:20] == bytes([0xFF, 0xD8, 0xFF, 0xE0, 0, 16]) + b"JFIF\0" + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0])
		assert out[20:25] == bytes([0xFF, 0xDB, 0, 132, 0]) and out[89] == 1
		assert out[154:165] == bytes([0xFF, 0xC0, 0, 17, 8, 0, 24, 0, 40, 3, 1]) and out[165] == sampling
		assert out[173:177] == bytes([0xFF, 0xC4, 0x01, 0xA2]) and out[593:595] == bytes([0xFF, 0xDA])
		assert out[-2:] == bytes([0xFF, 0xD9])


@pytest.mark.skipif(not os.path.exists(J.REF_LIB), reason="oracle/_ref/libref_jpeg.so is built only where the reference is present")
def test_random_images_equal_stb(host):
	stb = J.stb_encoder()
	rs = np.random.RandomState(20261018)
	kinds = J.KINDS + ("ffpad",)
	mismatches = []
	for i in range(RANDOM_IMAGES + LARGE_RANDOM_IMAGES):
		top = 96 if i < RANDOM_IMAGES else 1024
		width, height = (int(v) for v in rs.randint(1, top + 1, 2))
		quality = int(rs.randint(-5, 106))
		kind = kinds[i % len(kinds)]
		image = J.make_image(kind, width, height, int(rs.randint(0, 2 ** 31 - 1)))
		rc, out = host(image, quality)
		if rc != 0 or out != stb(image, quality):
			mismatches.append((kind, width, height, quality))
	assert not mismatches, mismatches[:10]


def test_host_build_refusals(host):
	image = J.make_image("noise", 20, 12, 1)
	rc, out = host(image, 70)
	assert rc == 0
	lib = J.host_library()
	f = lib.vkr_host_encode_jpg
	buf = np.zeros(len(out) + 16, dtype=np.uint8)
	size = C.c_size_t(0)
	# one byte short: refused, nothing written, the size reported
	assert f(image.ctypes.data, 20, 12, 70, buf.ctypes.data, len(out) - 1, C.byref(size)) == 1
	assert size.value == len(out) and not buf.any()
	assert f(image.ctypes.data, 20, 12, 70, buf.ctypes.data, len(out), C.byref(size)) == 0 and buf[:len(out)].tobytes() == out
	for width, height in ((0, 12), (20, 0), (65536, 1), (1, 65536)):
		assert f(image.ctypes.data, width, height, 70, buf.ctypes.data, len(buf), C.byref(size)) == 1
	assert f(None, 20, 12, 70, buf.ctypes.data, len(buf), C.byref(size)) == 1
	assert f(image.ctypes.data, 20, 12, 70, None, len(buf), C.byref(size)) == 1
	assert f(image.ctypes.data, 20, 12, 70, buf.ctypes.data, len(buf), None) == 1


def test_c_abi_refuses_before_device_work(built_library, tmp_path):
	"""argument checks of vkr_encode_jpg and vkr_write_jpg run before the device is touched: a zeroed vkr_device_t is never used here"""
	lib = built_library
	device = api.Device()
	image = J.make_image("noise", 20, 12, 1)
	buf = np.zeros(4096, dtype=np.uint8)
	size = C.c_size_t(0)
	dev = C.byref(device)
	for width, height in ((0, 12), (20, 0), (65536, 1), (1, 65536)):
		assert lib.vkr_encode_jpg(dev, image.ctypes.data, width, height, 70, buf.ctypes.data, len(buf), C.byref(size)) == 1
		assert lib.vkr_write_jpg(dev, str(tmp_path / "a.jpg").encode(), width, height, image.ctypes.data, 70) == 1
	assert lib.vkr_encode_jpg(dev, None, 20, 12, 70, buf.ctypes.data, len(buf), C.byref(size)) == 1
	assert lib.vkr_encode_jpg(dev, image.ctypes.data, 20, 12, 70, None, len(buf), C.byref(size)) == 1
	assert lib.vkr_encode_jpg(dev, image.ctypes.data, 20, 12, 70, buf.ctypes.data, len(buf), None) == 1
	assert lib.vkr_encode_jpg(None, image.ctypes.data, 20, 12, 70, buf.ctypes.data, len(buf), C.byref(size)) == 1
	assert lib.vkr_write_jpg(dev, None, 20, 12, image.ctypes.data, 70) == 1
	assert lib.vkr_write_jpg(dev, str(tmp_path / "b.jpg").encode(), 20, 12, None, 70) == 1
	assert lib.vkr_write_jpg(None, str(tmp_path / "c.jpg").encode(), 20, 12, image.ctypes.data, 70) == 1
	assert lib.vkr_write_jpg(dev, str(tmp_path / "missing" / "d.jpg").encode(), 20, 12, image.ctypes.data, 70) == 1   # unwritable path
	assert not any(tmp_path.iterdir())
	assert lib.vkr_abi_version() == 1
