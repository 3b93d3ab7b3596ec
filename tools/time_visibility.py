"""Times the two visibility buffers on the GPU in one process: the primary-ray cast (vkr_run_visibility_pass) and the rasteriser
(vkr_rasterize_visibility), alternating call by call, at the C3 shape (city, 1920x1080) and the C4 shape (room, 3840x2160).

Whole calls: CUDA events around each call, median and spread of --calls calls after --warmup calls of each. Stages of the rasteriser: torch.profiler
CUDA activities over --profile-calls calls in a separate run, summed per kernel and divided by the number of calls. Also reports build_seconds of the
C3 scene loaded with and without acceleration structure (what a user who renders without shadow rays saves), and the card's name and power limit.
Prints one JSON document; --out also writes it to a file.

    python tools/time_visibility.py [--calls 60] [--warmup 10] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tests import harness as H  # noqa: E402
from vulkan_renderer_b200 import api  # noqa: E402

SHAPES = [("C3", "city", 1920, 1080), ("C4", "room", 3840, 2160)]


def card():
	out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
	return out.stdout.strip()


def time_shape(name, width, height, calls, warmup, profile_calls):
	info = H.dataset(name)
	frame = H.open_frame(info)
	lib, dev, scene = frame.lib, C.byref(frame.device), C.byref(frame.scene)
	try:
		constants = frame.constants(width, height)[:256]
		vis = torch.empty((height, width), dtype=torch.int32, device="cuda:0")
		r = api.Rasterizer()
		frame._check(lib.vkr_create_rasterizer(C.byref(r), dev, width, height, frame.scene.triangle_count), "vkr_create_rasterizer")
		ray = lambda: lib.vkr_run_visibility_pass(dev, scene, constants, width, height, vis.data_ptr())
		raster = lambda: lib.vkr_rasterize_visibility(C.byref(r), dev, scene, constants, vis.data_ptr(), None)
		stream = torch.cuda.ExternalStream(frame.device.stream)
		times = {"ray": [], "raster": []}
		for i in range(warmup + calls):
			for key, fn in (("ray", ray), ("raster", raster)):
				begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
				begin.record(stream)
				assert fn() == 0
				end.record(stream)
				end.synchronize()
				if i >= warmup:
					times[key].append(begin.elapsed_time(end) * 1e3)
		drawn = {}
		for key, fn in (("ray", ray), ("raster", raster)):
			assert fn() == 0
			lib.vkr_device_wait_idle(dev)
			drawn[key] = float((vis.cpu().numpy() != -1).mean())
		from torch.profiler import ProfilerActivity, profile
		with profile(activities=[ProfilerActivity.CUDA]) as prof:
			for _ in range(profile_calls):
				assert raster() == 0
			lib.vkr_device_wait_idle(dev)
		stages = {}
		for e in prof.key_averages():
			if e.device_type == torch.autograd.DeviceType.CUDA:
				m = re.search(r"raster_\w+_kernel|DeviceScan\w*Kernel|Memset|Memcpy", e.key)
				label = m.group(0) if m else e.key[:60]
				stages[label] = stages.get(label, 0.0) + e.device_time_total / profile_calls
		lib.vkr_destroy_rasterizer(C.byref(r), dev)
		summary = lambda v: dict(median_us=float(np.median(v)), p10_us=float(np.percentile(v, 10)), p90_us=float(np.percentile(v, 90)))
		return dict(triangles=int(frame.scene.triangle_count), ray=summary(times["ray"]), raster=summary(times["raster"]), raster_stages_us=stages,
			drawn_fraction=drawn, build_seconds_with_acceleration_structure=float(frame.scene.build_seconds))
	finally:
		frame.close()


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--calls", type=int, default=60)
	ap.add_argument("--warmup", type=int, default=10)
	ap.add_argument("--profile-calls", type=int, default=20)
	ap.add_argument("--out")
	args = ap.parse_args()
	if not torch.cuda.is_available():
		raise SystemExit("no CUDA device: this tool measures the GPU")
	result = dict(card=card(), shapes={})
	for label, name, width, height in SHAPES:
		result["shapes"][label] = dict(dataset=name, width=width, height=height, **time_shape(name, width, height, args.calls, args.warmup, args.profile_calls))
	frame = H.open_frame(H.dataset("city"), request_acceleration_structure=False)
	result["shapes"]["C3"]["build_seconds_without_acceleration_structure"] = float(frame.scene.build_seconds)
	frame.close()
	text = json.dumps(result, indent=1)
	print(text)
	if args.out:
		with open(args.out, "w") as f:
			f.write(text)


if __name__ == "__main__":
	main()
