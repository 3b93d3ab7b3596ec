#!/usr/bin/env python3
"""Summarises an ncu capture of the shading megakernel into profiles/ (run here, no GPU needed).

  python tools/summarize_ncu.py gpurun_out/r01_prof.ncu-rep gpurun_out/r01_launches.csv profiles/r01_v1 [workload]

Writes <out>_summary.md: launch list (share of the step per kernel), key metrics of the top kernel (duration, DRAM
bytes, occupancy, issue utilisation, lanes per instruction), warp stall reasons and the hottest source lines
(SASS profile joined with nvdisasm line info of the in-tree library).
"""
import collections
import csv
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
	"sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
	"sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
	"gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
	"sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "launch__waves_per_multiprocessor", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic"]


def launches(path):
	rows = [r for r in csv.reader(l for l in open(path) if not l.startswith("=="))]
	hdr = rows[0]; ki = hdr.index("Kernel Name"); vi = hdr.index("Metric Value")
	d = collections.defaultdict(list)
	for r in rows[1:]:
		if len(r) > vi:
			d[r[ki]].append(float(r[vi].replace(",", "")))
	total = sum(sum(v) for v in d.values())
	return sorted(((k, len(v), sum(v), sum(v) / total) for k, v in d.items()), key=lambda t: -t[2])


def raw_metrics(rep):
	out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
	rows = list(csv.reader(out.splitlines()))
	hdr, units, vals = rows[0], rows[1], rows[2]
	return {h: (vals[i], units[i]) for i, h in enumerate(hdr)}, vals[hdr.index("Kernel Name")]


def sass_profile(rep):
	out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], stdout=subprocess.PIPE, text=True).stdout
	rows = list(csv.reader(out.splitlines()))
	hi = [i for i, r in enumerate(rows) if "Instructions Executed" in r][0]
	hdr = rows[hi]
	idx = {n: hdr.index(n) for n in ("Address", "Instructions Executed", "Thread Instructions Executed", "# Samples")}
	stalls = [i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
	prof = []; stall_tot = collections.Counter()
	for r in rows[hi + 1:]:
		try:
			prof.append((int(r[idx["Address"]], 16), float(r[idx["Instructions Executed"]]), float(r[idx["Thread Instructions Executed"]]), float(r[idx["# Samples"]])))
		except (ValueError, IndexError):
			continue
		for i in stalls:
			try: stall_tot[hdr[i]] += float(r[i])
			except ValueError: pass
	return prof, stall_tot


def line_info(kernel_mangled_regex, maxp):
	"""SASS line table of the kernel from the in-tree object of its vertex bound (build/vkr_shading_kernel_v<maxp - 1>.cu.o)."""
	obj = os.path.join(ROOT, "vulkan_renderer_b200", "build", "vkr_shading_kernel_v%d.cu.o" % (int(maxp) - 1))
	if not os.path.exists(obj):
		return []
	tmp = tempfile.mkdtemp()
	subprocess.run(["cuobjdump", "-xelf", "all", obj], cwd=tmp, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
	text, start = [], []
	for name in sorted(os.listdir(tmp)):
		if not name.endswith(".cubin"):
			continue
		text = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, name)], stdout=subprocess.PIPE, text=True).stdout.split("\n")
		start = [i for i, l in enumerate(text) if re.match(r"\.text\." + kernel_mangled_regex + ":", l)]
		if start:
			break
	if not start:
		return []
	insts = []; cur = ("?", 0)
	for l in text[start[0] + 1:]:
		if l.startswith("\t.section") or l.startswith(".text."):
			break
		m = re.search(r'//## File "([^"]+)", line (\d+)', l)
		if m:
			cur = (os.path.basename(m.group(1)), int(m.group(2))); continue
		if re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+\S", l):
			insts.append(cur)
	return insts


def main():
	rep, launch_csv, out = sys.argv[1:4]
	lines = ["# ncu summary: %s" % os.path.basename(rep), ""]
	lines += ["## Launch list (`--metrics gpu__time_duration.sum --clock-control none`, serialised, cold cache: compare shares)", "", "| kernel | launches | total ns | share |", "|---|---|---|---|"]
	for k, n, t, s in launches(launch_csv)[:8]:
		lines.append("| `%s` | %d | %.0f | %.4f |" % (k[:90], n, t, s))
	m, kernel = raw_metrics(rep)
	lines += ["", "## Top kernel `%s` (`--set full --clock-control none`)" % kernel, "", "| metric | value | unit |", "|---|---|---|"]
	for name in METRICS:
		if name in m:
			lines.append("| %s | %s | %s |" % (name, m[name][0], m[name][1]))
	prof, stalls = sass_profile(rep)
	tot_s = sum(stalls.values())
	lines += ["", "## Warp stall reasons (share of samples)", "", "| reason | share |", "|---|---|"]
	for k, v in stalls.most_common(8):
		lines.append("| %s | %.1f%% |" % (k, 100 * v / tot_s))
	mm = re.search(r"shading_kernel<([^>]*)>", kernel)
	insts = []
	if mm:
		args = re.findall(r"\d+", re.sub(r"\((int|bool)\)", "", mm.group(1)))
		mangled = "".join("L%s%sE" % ("i" if k < 2 else "b", a) for k, a in enumerate(args))
		insts = line_info(r"_ZN3vkr14shading_kernelI%sEEvNS_21shading_kernel_paramsE" % mangled, args[1])
	if insts and len(insts) == len(prof):
		by = collections.defaultdict(lambda: [0.0, 0.0, 0.0]); byfile = collections.defaultdict(lambda: [0.0, 0.0, 0.0])
		for (a, c, t, s), key in zip(prof, insts):
			for d in (by[key], byfile[key[0]]):
				d[0] += c; d[1] += t; d[2] += s
		tot = sum(v[0] for v in byfile.values()); tots = sum(v[2] for v in byfile.values())
		lines += ["", "## Instructions by source file", "", "| file | warp instructions | active lanes / instruction | stall samples |", "|---|---|---|---|"]
		for f, v in sorted(byfile.items(), key=lambda kv: -kv[1][0]):
			lines.append("| %s | %.1f%% | %.1f | %.1f%% |" % (f, 100 * v[0] / tot, v[1] / max(v[0], 1), 100 * v[2] / max(tots, 1)))
		lines += ["", "## Hottest source lines", "", "| share | lanes | where | source |", "|---|---|---|---|"]
		cache = {}
		for (f, ln), v in sorted(by.items(), key=lambda kv: -kv[1][0])[:30]:
			if f not in cache:
				p = os.path.join(ROOT, "vulkan_renderer_b200", "csrc", f)
				cache[f] = open(p).read().split("\n") if os.path.exists(p) else []
			src = cache[f][ln - 1].strip()[:90].replace("|", "\\|") if 0 < ln <= len(cache[f]) else ""
			lines.append("| %.2f%% | %.1f | %s:%d | `%s` |" % (100 * v[0] / tot, v[1] / max(v[0], 1), f, ln, src))
	else:
		lines += ["", "(source correlation skipped: the in-tree library does not match the profiled binary: %d vs %d instructions)" % (len(insts), len(prof))]
	with open(out + "_summary.md", "w") as f:
		f.write("\n".join(lines) + "\n")
	if len(sys.argv) > 4:   # workload name: record the counters bench.py quotes in its roofline object
		import json
		def num(name): return float(m[name][0].replace(",", "")) if name in m else None
		def in_bytes(name):
			scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
			return num(name) * scale.get(m[name][1], 1.0) if name in m else 0.0
		path = os.path.join(ROOT, "profiles", "kernel_counters.json")
		data = json.load(open(path)) if os.path.exists(path) else {}
		def frac(name): return round(num(name) / 100.0, 4) if num(name) is not None else None
		git = subprocess.run(["git", "-C", ROOT, "rev-parse", "--short", "HEAD"], stdout=subprocess.PIPE, text=True).stdout.strip()
		data[sys.argv[4]] = {"source": os.path.basename(out) + "_summary.md (ncu --set full --clock-control none, one launch)",
			"git": os.environ.get("VKR_CAPTURE_GIT", git),   # the commit whose kernel was captured (the commit of the tree the capture ran on)
			"warp_instructions": int(num("smsp__inst_executed.sum")) if num("smsp__inst_executed.sum") is not None else None,
			"lanes_per_instruction": num("smsp__thread_inst_executed_per_inst_executed.ratio"),
			"pipe_fma_frac": frac("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active"), "pipe_alu_frac": frac("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"),
			"pipe_xu_frac": frac("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active"), "pipe_lsu_frac": frac("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active"),
			"l1_hit_frac": frac("l1tex__t_sector_hit_rate.pct"), "l2_hit_frac": frac("lts__t_sector_hit_rate.pct"), "warps_active_frac": frac("sm__warps_active.avg.pct_of_peak_sustained_active"),
			"dram_bytes_per_launch": int(in_bytes("dram__bytes_read.sum") + in_bytes("dram__bytes_write.sum")),
			"issue_active_frac": round(num("smsp__issue_active.avg.pct_of_peak_sustained_active") / 100.0, 4),
			"l1_data_pipe_frac": round(num("l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed") / 100.0, 4) if num("l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed") is not None else None,
			"kernel_ms_under_ncu": round(num("gpu__time_duration.sum") * {"ms": 1.0, "us": 1e-3, "ns": 1e-6, "s": 1e3}.get(m["gpu__time_duration.sum"][1], 1.0), 3)}
		with open(path, "w") as f:
			json.dump(data, f, indent=1)
	print("\n".join(lines[:40]))


if __name__ == "__main__":
	main()
