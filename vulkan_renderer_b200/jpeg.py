"""JPEG files encoded on the device (include/vkr_b200.h, vkr_encode_jpg / vkr_write_jpg; DESIGN.md §5 "JPEG screenshots").

encode_jpg() returns the bytes stbi_write_jpg (stb_image_write v1.14, the writer of the reference's *.jpg screenshots) writes for the same 8-bit RGB
image and quality, byte for byte; the encoder runs in libvkr_b200.so on a CUDA device and there is no CPU fallback. Only the file comes back from the
device. write_jpg() stores it. Screenshots of a shading pass in all three formats: vkr_take_screenshot_formats.
"""
import ctypes as C
import os

import numpy as np

from . import api

SCREENSHOT_QUALITY = 70   # stbi_write_jpg(..., 70) of the reference's screenshots (src/main.c:1745-1751)
HEADER_BYTES = 607        # SOI .. SOS (vkr_jpeg.cuh, kHeaderBytes)


def _device_image(rgb8, dev):
	"""[height, width, 3] uint8 from numpy or torch -> a contiguous uint8 tensor on dev"""
	import torch
	if not torch.is_tensor(rgb8):
		rgb8 = torch.from_numpy(np.ascontiguousarray(rgb8))
	if rgb8.dtype != torch.uint8 or rgb8.dim() != 3 or rgb8.shape[2] != 3:
		raise ValueError("rgb8 must be [height, width, 3] uint8, got %s %s" % (tuple(rgb8.shape), rgb8.dtype))
	return rgb8.to(dev).contiguous()


def encode_jpg(rgb8, quality=SCREENSHOT_QUALITY, cuda_device=0):
	"""The JPEG file of rgb8 ([height, width, 3] uint8, numpy or torch on any device) at quality (0 means 90, else clamped to 1..100), encoded
	on CUDA device cuda_device. Returns bytes."""
	import torch
	lib = api.load_library()
	dev = torch.device("cuda", cuda_device)
	image = _device_image(rgb8, dev)
	height, width = int(image.shape[0]), int(image.shape[1])
	torch.cuda.synchronize(dev)   # the library works on its own stream
	device = api.Device()
	if lib.vkr_create_device(C.byref(device), cuda_device, None) != 0:
		raise RuntimeError("vkr_create_device failed for CUDA device %d" % cuda_device)
	try:
		size = C.c_size_t(0)
		capacity = HEADER_BYTES + width * height + 4096
		for _ in range(2):   # the first call reports the size when the guess is too small
			out = np.empty(capacity, dtype=np.uint8)
			if lib.vkr_encode_jpg(C.byref(device), C.c_void_p(image.data_ptr()), width, height, int(quality), out.ctypes.data, capacity, C.byref(size)) == 0:
				return out[:size.value].tobytes()
			if size.value <= capacity:
				break
			capacity = size.value
		raise RuntimeError("vkr_encode_jpg failed (%d x %d, quality %d)" % (width, height, quality))
	finally:
		lib.vkr_destroy_device(C.byref(device))


def write_jpg(path, rgb8, quality=SCREENSHOT_QUALITY, cuda_device=0):
	"""Writes the JPEG file of the host image rgb8 ([height, width, 3] uint8) to path through vkr_write_jpg, which encodes it on CUDA device
	cuda_device. Returns the file's size."""
	rgb8 = np.ascontiguousarray(rgb8, dtype=np.uint8)
	if rgb8.ndim != 3 or rgb8.shape[2] != 3:
		raise ValueError("rgb8 must be [height, width, 3] uint8, got %s" % (rgb8.shape,))
	lib = api.load_library()
	device = api.Device()
	if lib.vkr_create_device(C.byref(device), cuda_device, None) != 0:
		raise RuntimeError("vkr_create_device failed for CUDA device %d" % cuda_device)
	try:
		if lib.vkr_write_jpg(C.byref(device), os.fspath(path).encode(), rgb8.shape[1], rgb8.shape[0], rgb8.ctypes.data, int(quality)) != 0:
			raise RuntimeError("vkr_write_jpg failed for %s" % path)
	finally:
		lib.vkr_destroy_device(C.byref(device))
	return os.path.getsize(path)
