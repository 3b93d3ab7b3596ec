#!/usr/bin/env python3
"""Runs the reference's experiment list (src/experiment_list.c) on the CUDA path and writes the timing matrix as JSON.

  python tools/run_experiments.py --out gpurun_out/experiments [--select timings_central_4] [--width 1920 --height 1080] [--frames 12] [--no-screenshots]
      [--convergence M [--variance-frames K]] [--ltc DIR] [--noise ROOT]

--convergence M also measures the error of the selected figure experiments against converged references (M animated frames of each reference's
settings averaged on the device) and their noise level (mean per-frame variance over K animated frames), and writes convergence.json next to
timings.json (experiments.convergence_groups, experiments.run_convergence).

--ltc DIR shades every experiment with the LTC table in DIR (fit<i>.dat, e.g. written by tools/fit_ltc.py) instead of the datasets' synthetic one.

--noise ROOT shades every experiment and every convergence reference with the Ahmed-Wonka noise table ROOT/data/noise/ahmed_2d_rgba_256x256_64.blob
(e.g. written by tools/make_noise_tables.py), the noise type the reference's experiment list names, instead of white noise.

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
	ap.add_argument("--convergence", type=int, default=0, metavar="M", help="frames averaged into each reference; 0: no convergence measurement")
	ap.add_argument("--variance-frames", type=int, default=16, metavar="K", help="animated frames per member for its mean variance (with --convergence)")
	ap.add_argument("--ltc", default=None, metavar="DIR", help="directory of fit<i>.dat files to shade with instead of the synthetic LTC table")
	ap.add_argument("--noise", default=None, metavar="ROOT", help="directory holding data/noise/ahmed_2d_rgba_256x256_64.blob to shade with instead of white noise")
	args = ap.parse_args()
	todo = [e for e in experiments.experiment_list(all_figs=not args.no_figs, all_timings=not args.no_timings) if args.select in e["name"]]
	print("%d experiments" % len(todo))
	experiments.run(todo, args.data, args.out, json_path=os.path.join(args.out, "timings.json"), frames=args.frames, warmup=args.warmup,
		width=args.width, height=args.height, screenshot=not args.no_screenshots, ltc_dir=args.ltc, noise_root=args.noise)
	if args.convergence:
		selected = {e["name"] for e in todo}
		groups = [dict(g, members=[m for m in g["members"] if m in selected]) for g in experiments.convergence_groups()]
		groups = [g for g in groups if g["members"]]
		print("%d convergence groups" % len(groups))
		experiments.run_convergences(groups, args.data, args.out, os.path.join(args.out, "convergence.json"), args.convergence, args.variance_frames,
			width=args.width, height=args.height, ltc_dir=args.ltc, noise_root=args.noise)


if __name__ == "__main__":
	main()
