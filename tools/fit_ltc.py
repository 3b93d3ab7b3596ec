#!/usr/bin/env python3
"""Fits the specular BRDF's LTC table on the GPU and writes it as fit<i>.dat files that vkr_load_ltc_table (and tools/run_experiments.py --ltc) read.

  python tools/fit_ltc.py --out DIR [--resolution 64] [--fresnel-count 51] [--quadrature 32] [--iteration-limit 400] [--l1-cells 64]

Prints one JSON line: the device's name and power limit, the fit kernel's time (CUDA events), cells, objective evaluations, the L3 error summary of
the fit and, for --l1-cells cells drawn with a fixed seed, the L1 distance between the lobe and the LTC the shader evaluates from the quantised
table, next to that of the synthetic stand-in table (vulkan_renderer_b200.synth.write_ltc_fits). Needs a GPU (no CPU fallback).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from vulkan_renderer_b200 import ltc_fit, synth  # noqa: E402


def power_limit(cuda_device):
	try:
		out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(cuda_device)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
		return out.stdout.strip() or None
	except (OSError, subprocess.TimeoutExpired):
		return None


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--out", required=True, help="directory for fit0.dat ... fit<F-1>.dat")
	ap.add_argument("--resolution", type=int, default=64); ap.add_argument("--fresnel-count", type=int, default=51)
	ap.add_argument("--quadrature", type=int, default=32); ap.add_argument("--iteration-limit", type=int, default=400)
	ap.add_argument("--l1-cells", type=int, default=64, help="cells whose L1 distance is measured (0: none)")
	ap.add_argument("--cuda-device", type=int, default=0)
	args = ap.parse_args()
	fits, stats = ltc_fit.fit_ltc_table(args.resolution, args.fresnel_count, args.quadrature, args.iteration_limit, args.cuda_device)
	ltc_fit.write_ltc_fits(args.out, fits)
	record = dict(device=stats["device"], power_limit=power_limit(args.cuda_device), fit_ms=round(stats["fit_ms"], 3), timed="fit kernel, CUDA events",
		resolution=args.resolution, fresnel_count=args.fresnel_count, quadrature_size=args.quadrature, iteration_limit=args.iteration_limit,
		cells=stats["cell_count"], objective_evaluations=stats["objective_evaluations"], iteration_limit_hits=stats["iteration_limit_hits"],
		l3_error=dict(max=stats["max_error"], median=stats["median_error"], mean=stats["mean_error"]), out=args.out)
	if args.l1_cells:
		rng = np.random.default_rng(1)
		n, f = args.resolution, args.fresnel_count
		cells = [(int(rng.integers(f)), int(rng.integers(n)), int(rng.integers(1, n))) for _ in range(args.l1_cells)]   # column 0 (alpha = 1e-3) is finer than the grid
		with tempfile.TemporaryDirectory() as tmp:
			synth.write_ltc_fits(tmp, n, f)
			synthetic = ltc_fit.read_ltc_fits(tmp, f)
		grid = ltc_fit.hemisphere_grid()
		fitted_l1 = [ltc_fit.l1_distance(fits, n, f, *c, grid=grid) for c in cells]
		synthetic_l1 = [ltc_fit.l1_distance(synthetic, n, f, *c, grid=grid) for c in cells]
		record["l1"] = dict(cells=len(cells), fitted_median=float(np.median(fitted_l1)), fitted_max=float(np.max(fitted_l1)),
			synthetic_median=float(np.median(synthetic_l1)), synthetic_max=float(np.max(synthetic_l1)),
			cells_better_than_synthetic=int(sum(a < b for a, b in zip(fitted_l1, synthetic_l1))))
	print(json.dumps(record))


if __name__ == "__main__":
	main()
