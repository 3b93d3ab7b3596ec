#!/usr/bin/env python3
"""Runs the reference's experiment list (src/experiment_list.c) on the CUDA path and writes the timing matrix as JSON.

  python tools/run_experiments.py --out gpurun_out/experiments [--select timings_central_4] [--width 1920 --height 1080] [--frames 12] [--no-screenshots]

Needs a GPU (no CPU fallback). See vulkan_renderer_b200/experiments.py.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from vulkan_renderer_b200 import experiments  # noqa: E402


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--out", default="gpurun_out/experiments")
	ap.add_argument("--data", default="/tmp/vkr_b200_data/experiments")
	ap.add_argument("--select", default="", help="run only experiments whose name contains this string")
	ap.add_argument("--width", type=int, default=None); ap.add_argument("--height", type=int, default=None)
	ap.add_argument("--frames", type=int, default=12); ap.add_argument("--warmup", type=int, default=3)
	ap.add_argument("--no-figs", action="store_true"); ap.add_argument("--no-timings", action="store_true"); ap.add_argument("--no-screenshots", action="store_true")
	args = ap.parse_args()
	todo = [e for e in experiments.experiment_list(all_figs=not args.no_figs, all_timings=not args.no_timings) if args.select in e["name"]]
	print("%d experiments" % len(todo))
	experiments.run(todo, args.data, args.out, json_path=os.path.join(args.out, "timings.json"), frames=args.frames, warmup=args.warmup,
		width=args.width, height=args.height, screenshot=not args.no_screenshots)


if __name__ == "__main__":
	main()
