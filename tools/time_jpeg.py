#!/usr/bin/env python3
"""Times the device JPEG encoder (vkr_encode_jpg) at 1920x1080 and 3840x2160 on synthetic and rendered content, and stb_image_write's encoder on the
host (oracle/_ref/libref_jpeg.so, where it was built) for the same images. Prints the card's name and power limit, then one JSON line per image:

  kernel_us   the encoder's kernels per call (torch.profiler, CUDA activities: jpeg_* kernels and the two scans), mean over the profiled calls
  call_ms     the whole synchronous vkr_encode_jpg call, host clock, median (allocations, two size read-backs and the file's copy included)
  host_stb_ms stbi_write_jpg on the host CPU, median (not a GPU number)
  bytes       the file's size; equal: the device file equals stb's byte for byte (where stb is available)

usage: python tools/time_jpeg.py [--calls N] [--quality Q] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
	try:
		out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True).stdout
		return out.strip().splitlines()[0]
	except (OSError, subprocess.CalledProcessError):
		return "unknown (nvidia-smi unavailable)"


def rendered(width, height):
	"""a Cornell frame as an 8-bit UNORM render target stores it (sRGB output, vkr_quantize_unorm8)"""
	from tests import harness as H
	from vulkan_renderer_b200 import api
	frame = H.open_frame(H.dataset("cornell"))
	try:
		frame.configure(sample_count=2, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)
		frame.output_srgb = 1
		_, gb = frame.gbuffer_host(width, height)
		out = np.ascontiguousarray(frame.shade_host(width, height, gb), dtype=np.float32)
	finally:
		frame.close()
	rgb = np.zeros((height, width, 3), dtype=np.uint8)
	api.load_library().vkr_quantize_unorm8(out.ctypes.data_as(C.c_void_p), width, height, rgb.ctypes.data_as(C.c_void_p))
	return rgb


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--calls", type=int, default=20)
	ap.add_argument("--quality", type=int, default=70)
	ap.add_argument("--out", default=None)
	args = ap.parse_args()
	import torch
	from torch.profiler import ProfilerActivity, profile
	from tests import jpeg_cases as J
	from vulkan_renderer_b200 import api
	if not torch.cuda.is_available():
		raise SystemExit("time_jpeg: no CUDA device; nothing is measured on the CPU")
	print("card, power limit: %s" % card())
	lib = api.load_library()
	dev = api.Device()
	assert lib.vkr_create_device(C.byref(dev), 0, None) == 0
	tdev = torch.device("cuda", 0)
	stb = J.stb_encoder()
	records = []
	try:
		for width, height in ((1920, 1080), (3840, 2160)):
			images = [("noise", J.make_image("noise", width, height, 1)), ("gradient", J.make_image("gradient", width, height, 2)), ("cornell", rendered(width, height))]
			for name, image in images:
				d_image = torch.from_numpy(image).to(tdev)
				torch.cuda.synchronize(tdev)
				capacity = 1024 + image.size * 2
				out = np.zeros(capacity, dtype=np.uint8)
				size = C.c_size_t(0)
				call = lambda: lib.vkr_encode_jpg(C.byref(dev), C.c_void_p(d_image.data_ptr()), width, height, args.quality, out.ctypes.data, capacity, C.byref(size))
				for _ in range(3):
					assert call() == 0
				times = []
				for _ in range(args.calls):
					t0 = time.perf_counter(); assert call() == 0; times.append(1e3 * (time.perf_counter() - t0))
				with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
					for _ in range(args.calls):
						assert call() == 0
				kernels = {}
				for e in prof.key_averages():
					t = getattr(e, "device_time_total", None)
					t = e.cuda_time_total if t is None else t
					m = re.search(r"jpeg_\w+|DeviceScan\w*", e.key)
					if m:
						kernels[m.group(0)] = kernels.get(m.group(0), 0.0) + t / args.calls
				data = out[:size.value].tobytes()
				record = dict(image=name, width=width, height=height, quality=args.quality, bytes=len(data), call_ms=statistics.median(times),
					kernel_us=sum(kernels.values()), kernels_us=kernels, frame_float4_mb=16.0 * width * height / 1e6)
				if stb is not None:
					host_times = []
					for _ in range(3):
						t0 = time.perf_counter(); ref = stb(image, args.quality); host_times.append(1e3 * (time.perf_counter() - t0))
					record.update(host_stb_ms=statistics.median(host_times), equal=ref == data)
				records.append(record)
				print(json.dumps(record))
	finally:
		lib.vkr_destroy_device(C.byref(dev))
	if args.out:
		os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
		with open(args.out, "w") as f:
			json.dump(dict(card=card(), records=records), f, indent=1)


if __name__ == "__main__":
	main()
