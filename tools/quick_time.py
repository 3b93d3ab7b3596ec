#!/usr/bin/env python3
"""Quick kernel timing experiments on the bench scene (developer tool): python tools/quick_time.py [spp] [lights] [rays]"""
import ctypes as C, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from vulkan_renderer_b200 import Frame, api, synth
spp = int(sys.argv[1]) if len(sys.argv) > 1 else 64
lights = int(sys.argv[2]) if len(sys.argv) > 2 else 8
rays = int(sys.argv[3]) if len(sys.argv) > 3 else 1
strategy = int(sys.argv[4]) if len(sys.argv) > 4 else 3
width, height = 1920, 1080
info = synth.build_dataset("/tmp/vkr_b200_data/city", "city")
dev = torch.device("cuda", 0); stream = torch.cuda.Stream(dev); torch.cuda.set_stream(stream)
frame = Frame(info["vks"], info["textures"], info["save"], info["ltc"], cuda_device=0, stream=stream.cuda_stream)
frame.configure(sample_count=spp, strategy=strategy, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=rays, show_lights=1, light_count=lights)
lib = frame.lib
print("BVH: %d node pairs, depth %d, built in %.3f s (%s)" % (frame.scene.shadow_node_count, frame.scene.shadow_max_depth, frame.scene.build_seconds, os.environ.get("VKR_BVH_BUILDER", "sah on the host")), flush=True)
constants = frame.constants(width, height)
vis = torch.empty((height, width), dtype=torch.int32, device=dev); gb = torch.empty((4, height, width, 4), dtype=torch.float32, device=dev); out = torch.zeros((height, width, 4), dtype=torch.float32, device=dev)
lib.vkr_run_visibility_pass(C.byref(frame.device), C.byref(frame.scene), constants, width, height, vis.data_ptr())
lib.vkr_run_gbuffer_pass(C.byref(frame.device), C.byref(frame.scene), constants, width, height, vis.data_ptr(), gb.data_ptr())
p = frame.create_pass(width, height, timing=True)
for i in range(3):
	lib.vkr_shading_pass_run(C.byref(p), C.byref(frame.device), constants, len(constants), gb.data_ptr(), out.data_ptr())
	lib.vkr_shading_pass_wait(C.byref(p), C.byref(frame.device))
	print("spp %d lights %d rays %d strategy %d: kernel %.3f ms -> %.1f Msamples/s" % (spp, lights, rays, strategy, p.last_kernel_ms, width * height * spp / p.last_kernel_ms / 1e3), flush=True)
if os.environ.get("VKR_COUNTERS"):   # what the trace warps did (the counters edition of the kernel; same frame)
	counters = (C.c_uint64 * api.TRACE_COUNTER_COUNT)()
	assert lib.vkr_shading_pass_run_with_counters(C.byref(p), C.byref(frame.device), constants, len(constants), gb.data_ptr(), out.data_ptr(), counters) == 0
	c = dict(zip(api.TRACE_COUNTER_NAMES, [int(v) for v in counters]))
	rays = max(1, c["rays"])
	print("counters", c)
	print("per ray: %.2f node visits, %.2f leaves, %.2f triangle tests; occluded %.3f, cache hits %.3f; lanes per node step %.2f; counters-edition kernel %.1f ms" % (
		c["node_visits"] / rays, c["leaf_visits"] / rays, c["triangle_tests"] / rays, c["occluded"] / rays, c["cache_hits"] / rays, c["node_visits"] / max(1, c["warp_node_steps"]), p.last_kernel_ms))
import hashlib
print("valid fraction", float((gb[1, :, :, 3] != 0).float().mean()), "mean radiance", float(out[..., :3].mean()),
	"frame sha256", hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()[:16])   # builders and traversal variants must leave the frame bit-identical
