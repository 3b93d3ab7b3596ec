#!/usr/bin/env python3
"""Writes profiles/<tag>_sass_excerpt.md: the parts of the benchmark kernel's SASS that show what it is built from (run here, no GPU needed).

  python tools/sass_excerpt.py r02

shading_kernel<3,5,0,0,1> (quad lights, diffuse + specular MIS, shadow rays) from the in-tree object: resource usage, the instruction mix, the bulk copy of
the constant block (UBLKCP) with its mbarrier, the register hand-over between trace and shading warps (USETMAXREG) and the trace warps' node loop
(four 128-bit node fetches, the slab test on the FMA pipe, its min / max as VIMNMX3 + VIMNMX)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN3vkr14shading_kernelILi3ELi5ELb0ELb0ELb1EEEvNS_21shading_kernel_paramsE"
OBJ = os.path.join(ROOT, "vulkan_renderer_b200", "build", "vkr_shading_kernel_v4.cu.o")


def main():
	tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
	sass = subprocess.run(["cuobjdump", "-sass", "-fun", KERNEL, OBJ], stdout=subprocess.PIPE, text=True).stdout
	lines = [re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", l).rstrip() for l in sass.split("\n") if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
	usage = subprocess.run(["cuobjdump", "-res-usage", "-fun", KERNEL, OBJ], stdout=subprocess.PIPE, text=True).stdout
	usage = [l.strip() for l in usage.split("\n") if "REG:" in l]
	ops = collections.Counter(re.sub(r"^@!?U?P\d\s+", "", l.split("*/", 1)[1].strip()).split()[0].rstrip(";") for l in lines)
	def family(prefixes): return sum(v for k, v in ops.items() if k.split(".")[0] in prefixes)
	git = subprocess.run(["git", "-C", ROOT, "rev-parse", "--short", "HEAD"], stdout=subprocess.PIPE, text=True).stdout.strip()
	out = ["# SASS of `shading_kernel<3,5,0,0,1>` (sm_90a), commit %s" % git, "",
		"`cuobjdump -sass -fun %s vulkan_renderer_b200/build/vkr_shading_kernel_v4.cu.o`, excerpts." % KERNEL, "",
		"* resource usage: `%s`" % (usage[0] if usage else "?"),
		"* %d instructions; FFMA / FMUL / FADD %d, FMNMX %d, VIMNMX3 / VIMNMX %d, MUFU %d, LDG %d (of them 128-bit: %d), LDS / STS %d, LDL / STL (spills) %d, VOTE / SHFL %d" % (
			len(lines), family({"FFMA", "FMUL", "FADD"}), family({"FMNMX"}), family({"VIMNMX3", "VIMNMX"}), family({"MUFU"}), family({"LDG"}), sum(v for k, v in ops.items() if k.startswith("LDG") and ".128" in k),
			family({"LDS", "STS"}), family({"LDL", "STL"}), family({"VOTE", "VOTEU", "SHFL"})),
		"* no tensor-core or tensor-map instructions (HMMA / HGMMA / UTMALDG count: %d): the path has no contraction" % family({"HMMA", "HGMMA", "UTMALDG"}), ""]
	def excerpt(title, pattern, before, after, limit=1):
		hits = [i for i, l in enumerate(lines) if re.search(pattern, l)][:limit]
		for i in hits:
			out.extend(["## %s" % title, "", "```"] + lines[max(0, i - before):i + after + 1] + ["```", ""])
	excerpt("Constant block: one bulk asynchronous copy into shared memory, completion on an mbarrier", r"UBLKCP", 6, 8)
	excerpt("Role split: trace warps give registers to the shading warps", r"USETMAXREG", 2, 3, limit=2)
	excerpt("Trace warps: the node loop (one node pair = four 128-bit loads; slab test as FFMA + VIMNMX3 / VIMNMX; shared-memory stack)", r"VIMNMX3", 40, 40)
	excerpt("Trace warps: ticket draw (one shared-memory atomic per warp refill)", r"ATOMS\.ADD", 8, 6)
	path = os.path.join(ROOT, "profiles", "%s_sass_excerpt.md" % tag)
	os.makedirs(os.path.dirname(path), exist_ok=True)
	with open(path, "w") as f:
		f.write("\n".join(out) + "\n")
	print("wrote", path, "(%d instructions)" % len(lines))


if __name__ == "__main__":
	main()
