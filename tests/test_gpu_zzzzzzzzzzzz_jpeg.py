"""JPEG files encoded on the GPU (csrc/vkr_jpeg.cu): the kernels against stb_image_write's frozen output and against the host build of the same header
(tests/jpeg_on_host.cpp), byte for byte.

1. vkr_encode_jpg writes every file of tests/golden/ref_jpeg.npz and the host build's bytes; a second run writes the same bytes.
2. random 1920x1080, 1921x1081 and 3840x2160 images equal the host build.
3. vkr_take_screenshot_formats(png, jpg) on a Cornell frame: the *.png equals vkr_take_screenshot's byte for byte, the *.jpg is the host encoding of
   the *.png's pixels at quality 70, the *.hdr equals vkr_take_screenshot's; LDR and HDR cannot be mixed.
4. vkr_quantize_unorm8_device equals vkr_quantize_unorm8 on NaN, infinities, signed zeros, denormals, values above 1 and the floats one ulp either
   side of every rounding boundary (k + 0.5) / 255.
5. refusals through the device path: a capacity one byte short (nothing written, the size reported), bad sizes and NULL pointers.
"""
import ctypes as C

import numpy as np
import pytest

from tests import harness as H
from tests import jpeg_cases as J
from vulkan_renderer_b200 import api, jpeg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def device():
	import torch
	lib = api.load_library()
	dev = api.Device()
	assert lib.vkr_create_device(C.byref(dev), 0, None) == 0
	yield lib, dev, torch.device("cuda", 0)
	lib.vkr_destroy_device(C.byref(dev))


def device_encode(device, image, quality, capacity=None):
	"""(return code, bytes, reported size) of vkr_encode_jpg on a device copy of image"""
	import torch
	lib, dev, tdev = device
	d_image = torch.from_numpy(np.ascontiguousarray(image)).to(tdev)
	torch.cuda.synchronize(tdev)
	capacity = 1024 + 8 * image.size if capacity is None else capacity
	out = np.zeros(max(capacity, 1), dtype=np.uint8)
	size = C.c_size_t(0)
	rc = lib.vkr_encode_jpg(C.byref(dev), C.c_void_p(d_image.data_ptr()), image.shape[1], image.shape[0], int(quality), out.ctypes.data, capacity, C.byref(size))
	return rc, out, size.value


def test_device_writes_the_golden_files(device):
	host = J.host_encoder()
	for case, data in J.load_golden():
		image = J.make_image(case["kind"], case["width"], case["height"], case["seed"])
		rc, out, size = device_encode(device, image, case["quality"])
		assert rc == 0 and size == case["size"], case
		got = out[:size].tobytes()
		assert J.digest(got) == case["sha256"], case
		if data is not None:
			assert got == data, case
		assert got == host(image, case["quality"])[1], case
		rc, again, size = device_encode(device, image, case["quality"])
		assert rc == 0 and again[:size].tobytes() == got, case


@pytest.mark.parametrize("width,height,quality", [(1920, 1080, 70), (1921, 1081, 90), (1921, 1081, 95), (3840, 2160, 70)])
def test_large_random_images_equal_the_host_build(device, width, height, quality):
	host = J.host_encoder()
	for kind, seed in (("noise", 11), ("gradient", 12), ("saturated", 13)):
		image = J.make_image(kind, width, height, seed + width)
		rc, out, size = device_encode(device, image, quality)
		assert rc == 0
		assert out[:size].tobytes() == host(image, quality)[1], (kind, width, height, quality)


def test_python_wrappers(device, tmp_path):
	image = J.make_image("gradient", 100, 60, 3)
	expected = J.host_encoder()(image, 70)[1]
	assert jpeg.encode_jpg(image) == expected
	import torch
	assert jpeg.encode_jpg(torch.from_numpy(image).cuda(), quality=70) == expected
	assert jpeg.write_jpg(tmp_path / "a.jpg", image) == len(expected)
	assert (tmp_path / "a.jpg").read_bytes() == expected
	noise = J.make_image("noise", 300, 200, 4)    # larger than encode_jpg's first guess at quality 100
	assert jpeg.encode_jpg(noise, quality=100) == J.host_encoder()(noise, 100)[1]


def test_screenshot_formats(tmp_path):
	from tests.test_output import _read_png
	width, height = 160, 120
	info = H.dataset("cornell")
	frame = H.open_frame(info)
	targets = api.RenderTargets()
	try:
		frame.configure(sample_count=2, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)
		constants = frame.constants(width, height)
		_, gb = frame.gbuffer_host(width, height)
		assert frame.lib.vkr_create_render_targets(C.byref(targets), C.byref(frame.device), width, height) == 0
		assert frame.lib.vkr_upload_gbuffer(C.byref(targets), C.byref(frame.device), np.ascontiguousarray(gb, dtype=np.float32).ctypes.data_as(C.c_void_p)) == 0
		p = frame.create_pass(width, height)
		shot = lambda png, jpg, hdr: frame.lib.vkr_take_screenshot_formats(C.byref(p), C.byref(frame.device), constants, len(constants), targets.d_gbuffer,
			png and str(tmp_path / png).encode(), jpg and str(tmp_path / jpg).encode(), hdr and str(tmp_path / hdr).encode())
		old = lambda png, hdr: frame.lib.vkr_take_screenshot(C.byref(p), C.byref(frame.device), constants, len(constants), targets.d_gbuffer,
			png and str(tmp_path / png).encode(), hdr and str(tmp_path / hdr).encode())
		assert old("old.png", None) == 0 and old(None, "old.hdr") == 0
		assert shot("new.png", "new.jpg", None) == 0
		assert shot(None, "only.jpg", None) == 0
		assert shot(None, None, "new.hdr") == 0
		assert shot("x.png", None, "x.hdr") == 1 and shot(None, "x.jpg", "x.hdr") == 1 and shot("x.png", "x.jpg", "x.hdr") == 1   # LDR and HDR cannot be mixed
		assert shot(None, None, None) == 0
		assert p.desc.output_srgb == 0
	finally:
		frame.lib.vkr_destroy_render_targets(C.byref(targets), C.byref(frame.device)); frame.close()
	assert not any((tmp_path / n).exists() for n in ("x.png", "x.jpg", "x.hdr"))
	assert (tmp_path / "new.png").read_bytes() == (tmp_path / "old.png").read_bytes()
	assert (tmp_path / "new.hdr").read_bytes() == (tmp_path / "old.hdr").read_bytes()
	pixels = _read_png(str(tmp_path / "new.png"))
	assert pixels.max() > 32
	expected = J.host_encoder()(pixels, 70)[1]
	assert (tmp_path / "new.jpg").read_bytes() == expected
	assert (tmp_path / "only.jpg").read_bytes() == expected


def test_device_quantisation_equals_the_host(device):
	import torch
	lib, dev, tdev = device
	boundaries = ((np.arange(255, dtype=np.float64) + 0.5) / 255.0).astype(np.float32)
	special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, 1.17549435e-38, 1.0, 1.0000001, 2.0, 1e30, -1.0,
		0.99999994, np.float32(0.5) / np.float32(255)], dtype=np.float32)
	values = np.concatenate([special, boundaries, np.nextafter(boundaries, np.float32(0)), np.nextafter(boundaries, np.float32(2))]).astype(np.float32)
	values = np.concatenate([values, np.zeros((-len(values)) % 4, dtype=np.float32)])   # whole float4 pixels: alpha is a channel too, and ignored
	values = np.concatenate([values, values[::-1]])
	frame = values.reshape(-1, 4)
	width, height = frame.shape[0], 1
	expected = np.zeros(3 * width, dtype=np.uint8)
	lib.vkr_quantize_unorm8(frame.ctypes.data_as(C.c_void_p), width, height, expected.ctypes.data_as(C.c_void_p))
	d_frame = torch.from_numpy(frame.copy()).to(tdev)
	d_out = torch.zeros(3 * width, dtype=torch.uint8, device=tdev)
	torch.cuda.synchronize(tdev)
	assert lib.vkr_quantize_unorm8_device(C.byref(dev), C.c_void_p(d_frame.data_ptr()), width, height, C.c_void_p(d_out.data_ptr())) == 0
	assert lib.vkr_device_wait_idle(C.byref(dev)) == 0
	got = d_out.cpu().numpy()
	assert np.array_equal(got, expected), np.nonzero(got != expected)
	assert lib.vkr_quantize_unorm8_device(C.byref(dev), None, width, height, C.c_void_p(d_out.data_ptr())) == 1


def test_device_refusals(device):
	lib, dev, tdev = device
	image = J.make_image("noise", 33, 21, 9)
	rc, out, size = device_encode(device, image, 80)
	assert rc == 0
	rc, short, needed = device_encode(device, image, 80, capacity=size - 1)
	assert rc == 1 and needed == size and not short.any()
	rc, exact, _ = device_encode(device, image, 80, capacity=size)
	assert rc == 0 and exact[:size].tobytes() == out[:size].tobytes()
	import torch
	d_image = torch.from_numpy(image).to(tdev)
	buf = np.zeros(1 << 16, dtype=np.uint8)
	s = C.c_size_t(0)
	for width, height in ((0, 21), (33, 0), (65536, 21), (33, 65536)):
		assert lib.vkr_encode_jpg(C.byref(dev), C.c_void_p(d_image.data_ptr()), width, height, 80, buf.ctypes.data, len(buf), C.byref(s)) == 1
	assert lib.vkr_encode_jpg(C.byref(dev), None, 33, 21, 80, buf.ctypes.data, len(buf), C.byref(s)) == 1
	assert lib.vkr_encode_jpg(C.byref(dev), C.c_void_p(d_image.data_ptr()), 33, 21, 80, None, len(buf), C.byref(s)) == 1
	assert not buf.any()
