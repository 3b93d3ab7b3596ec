"""Frame set-up shared by tools/make_ref_golden.py and tests/test_ref_shader.py (host-only, no GPU)."""
import ctypes as C
import hashlib

import numpy as np

from vulkan_renderer_b200 import api

WIDTH, HEIGHT = 64, 48


def frame_sha256(frame):
	"""What tests/golden/ref_shader.npz keeps of a frame of the reference shader (`<name>/rgba_sha256`): the SHA-256 of its float32 RGBA bytes."""
	return hashlib.sha256(np.ascontiguousarray(frame, dtype=np.float32).tobytes()).digest()


def assert_matches_fixture(golden, name, frame):
	"""Bit for bit: the frame equals the reference shader's fixture `name`."""
	assert frame_sha256(frame) == bytes(golden[name + "/rgba_sha256"]), "%s: the frame differs from the reference shader's" % name


def dataset_for(cfg):
	if cfg.get("textured", 0):
		return "mini_textured"
	if cfg.get("light_textures", 0):
		return "mini_lit"
	if cfg["materials"] == 3:
		return "cornell"
	if cfg["lights"] > 3:
		return "mini_room"
	if cfg["max_vertices"] >= 5:
		vmin = cfg.get("min_vertices", cfg["max_vertices"])
		return "mini_poly" if vmin != cfg["max_vertices"] else "mini_v%d" % cfg["max_vertices"]
	if cfg["max_vertices"] == 3:
		return "mini_tri"
	return "mini_mixed" if cfg.get("min_vertices", cfg["max_vertices"]) != cfg["max_vertices"] else "mini_city"


def host_constants(info, width, height, lights, sample_count=1, frame_bits=0):
	"""Constant block through the library's host-only loaders (device = NULL)."""
	lib = api.load_library()
	scene = api.Scene(); ltc = api.LtcTable(); noise = api.NoiseTable(); spec = api.SceneSpecification(); st = api.RenderSettings()
	assert lib.vkr_load_scene(C.byref(scene), None, info["vks"].encode(), info["textures"].encode(), 0) == 0
	assert lib.vkr_load_ltc_table(C.byref(ltc), None, info["ltc"].encode(), 51) == 0
	assert lib.vkr_load_noise_table(C.byref(noise), None, 256, 256, 64, api.NOISE_WHITE) == 0
	assert lib.vkr_quick_load(C.byref(spec), info["save"].encode()) == 0
	assert lights <= spec.polygonal_light_count
	assert lib.vkr_create_and_assign_light_textures(None, None, C.byref(spec)) == 0   # texture indices only (src/main.c:2167)
	spec_count = spec.polygonal_light_count
	spec.polygonal_light_count = lights
	lib.vkr_specify_default_render_settings(C.byref(st)); st.animate_noise = 0; st.exposure_factor = 1.0; st.sample_count = sample_count
	size = lib.vkr_get_constants_size(C.byref(spec)); buf = (C.c_uint8 * size)()
	lib.vkr_write_constants(buf, C.byref(spec), C.byref(st), C.byref(scene), C.byref(ltc), C.byref(noise), width, height)
	if frame_bits:
		lib.vkr_set_frame_bits(buf, frame_bits)
	spec.polygonal_light_count = spec_count
	lib.vkr_destroy_scene_specification(C.byref(spec)); lib.vkr_destroy_noise_table(C.byref(noise), None); lib.vkr_destroy_ltc_table(C.byref(ltc), None); lib.vkr_destroy_scene(C.byref(scene), None)
	return bytes(buf)


def oracle_cfg(cfg, width=WIDTH, height=HEIGHT):
	return dict(width=width, height=height, light_count=cfg["lights"], max_light_vertex_count=cfg["max_vertices"], min_light_vertex_count=cfg.get("min_vertices", cfg["max_vertices"]),
		sample_count=cfg["samples"], sampling_strategies=cfg["strategy"], mis_heuristic=cfg["heuristic"], biased_sampling=cfg["biased"],
		trace_shadow_rays=cfg["trace"], show_polygonal_lights=cfg["show_lights"], output_srgb=cfg.get("srgb", 0), polygon_sampling_technique=cfg.get("technique", 11), error_display=cfg.get("error_display", 0))
