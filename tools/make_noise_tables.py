#!/usr/bin/env python3
"""Generates the blue-noise and Ahmed-Wonka noise tables on the GPU and writes them as the .blob files vkr_load_noise_table reads (and
tools/run_experiments.py --noise ROOT, and Frame(noise_type=..., noise_root=ROOT)).

  python tools/make_noise_tables.py --out ROOT [--type blue|ahmed|both] [--seed 0]

Writes ROOT/data/noise/blue_noise_rgba_64x64_64.blob and ROOT/data/noise/ahmed_2d_rgba_256x256_64.blob at the reference's default resolutions and
prints one JSON line per table: the device's name and power limit, the generating kernel's time (CUDA events) and, for the dither arrays, how many
relaxations stopped at the iteration limit. These are this project's tables, not the files of the paper's data download (DESIGN.md §5).
Needs a GPU (no CPU fallback).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from vulkan_renderer_b200 import noise_gen  # noqa: E402


def power_limit(cuda_device):
	try:
		out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(cuda_device)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
		return out.stdout.strip() or None
	except (OSError, subprocess.TimeoutExpired):
		return None


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--out", required=True, metavar="ROOT", help="the tables go to ROOT/data/noise/")
	ap.add_argument("--type", choices=["blue", "ahmed", "both"], default="both")
	ap.add_argument("--seed", type=int, default=0)
	ap.add_argument("--cuda-device", type=int, default=0)
	args = ap.parse_args()
	for name in (["blue", "ahmed"] if args.type == "both" else [args.type]):
		noise_type = noise_gen.NAMES[name]
		texels, stats = noise_gen.generate_noise_table(noise_type, seed=args.seed, cuda_device=args.cuda_device)
		path = noise_gen.write_noise_table(args.out, noise_type, texels)
		layers, height, width, _ = texels.shape
		record = dict(type=name, device=stats["device"], power_limit=power_limit(args.cuda_device), kernel_ms=round(stats["kernel_ms"], 3),
			timed="generating kernel, CUDA events", width=width, height=height, layers=layers, seed=args.seed, path=path)
		if name == "blue":
			record["relaxation_limit_hits"] = stats["relaxation_limit_hits"]
		print(json.dumps(record), flush=True)


if __name__ == "__main__":
	main()
