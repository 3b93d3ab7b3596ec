"""Boundary B1 (SURVEY 8b): the reference's UNCHANGED loader and host-maths sources, compiled against shim/, load the synthetic datasets; what
they upload through the shim must equal, byte for byte, what libvkr_b200.so's own loaders produce. Also pins the host maths
(update_polygonal_light, camera matrices, matrix_inverse) of vkr_host.cpp against the reference's code. What the reference's code produced
is frozen in tests/golden/ref_live.npz (tools/make_ref_live_golden.py; arrays, or SHA-256 digests of the large ones), so these tests need
nothing outside the repository."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from tests import harness as H
from vulkan_renderer_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_live.npz")
LOAD_SCENE_DATASETS = ["cornell", "mini_city"]
CONSTANT_BLOCK_FRAMES = [("cornell", 1, 128, 96), ("mini_city", 3, 320, 192), ("mini_room", 32, 64, 48)]


@pytest.fixture(scope="module")
def ref():
	return np.load(GOLDEN)


def sha256(data):
	return np.frombuffer(hashlib.sha256(bytes(data)).digest(), dtype=np.uint8)


def light_trials():
	"""The polygonal lights of test_host_maths_matches_the_reference_bit_for_bit (seeded): (light with its 160 bytes of parameters set, vertex count,
	plane-space vertices)."""
	rng = np.random.default_rng(11)
	for trial in range(200):
		n = int(rng.integers(3, 8))
		light = api.PolygonalLight()
		for i in range(3):
			light.rotation_angles[i] = rng.uniform(-3.2, 3.2); light.translation[i] = rng.uniform(-50, 50); light.radiant_flux[i] = rng.uniform(0.1, 100)
		light.scaling_x = rng.uniform(0.1, 5); light.scaling_y = rng.uniform(0.1, 5)
		ang = np.sort(rng.uniform(0, 2 * np.pi, n))
		if trial % 2: ang = ang[::-1]                       # both windings (the plane gets flipped for clockwise polygons)
		vp = np.zeros((n, 4), dtype=np.float32); vp[:, 0] = np.cos(ang) * rng.uniform(0.5, 1.5); vp[:, 1] = np.sin(ang) * rng.uniform(0.5, 1.5)
		yield light, n, vp
	for trial in range(200):
		cam = api.Camera()
		for i in range(3): cam.position_world_space[i] = rng.uniform(-100, 100)
		cam.rotation_z = rng.uniform(-7, 7); cam.rotation_x = rng.uniform(0, 3.14); cam.vertical_fov = rng.uniform(0.3, 2.0); cam.near_plane = 0.05; cam.far_plane = 1000.0
		aspect = np.float32(rng.uniform(0.5, 2.5))
		yield cam, aspect, None


def world_to_projection_for_the_inverse():
	"""The matrix test_constant_block_pixel_to_ray_uses_the_reference_inverse hands to the reference's matrix_inverse."""
	from tests.ref_frames import host_constants
	cb = host_constants(H.dataset("mini_city"), 320, 200, 3)
	w2p = np.frombuffer(cb[32:96], dtype=np.float32).reshape(4, 4).copy()
	w2p[:3, 3] = 0.0
	return cb, w2p


def test_struct_sizes(ref):
	assert list(ref["struct_sizes"]) == [C.sizeof(api.Camera), C.sizeof(api.PolygonalLight), 88, 160, C.sizeof(api.LtcConstants)]


@pytest.mark.parametrize("name", LOAD_SCENE_DATASETS)
def test_reference_load_scene_through_the_shim_equals_our_loader(ref, name):
	info = H.dataset(name)
	g = lambda key: ref["load_scene/%s/%s" % (name, key)]
	lib = api.load_library()
	scene = api.Scene()
	assert lib.vkr_load_scene(C.byref(scene), None, info["vks"].encode(), info["textures"].encode(), 1) == 0
	n = int(g("counts")[0])
	assert n == scene.triangle_count == info["triangle_count"] and int(g("counts")[1]) == scene.material_count
	assert g("factor_summand").tobytes() == np.array(list(scene.dequantization_factor) + list(scene.dequantization_summand), dtype=np.float32).tobytes()
	vks = H.read_vks(info["vks"])
	assert np.array_equal(g("positions_sha256"), sha256(np.ascontiguousarray(vks["positions"], dtype=np.uint32)))
	assert np.array_equal(g("normals_uv_sha256"), sha256(np.ascontiguousarray(vks["normals_uv"], dtype=np.uint16)))
	assert np.array_equal(g("material_indices_sha256"), sha256(np.ascontiguousarray(vks["material_indices"], dtype=np.uint8)))
	# the triangle soup handed to vkCmdBuildAccelerationStructuresKHR (scene.c:175-209) == what our shadow BVH is built from
	ours = H.oracle.dequantize_for_bvh(vks["positions"], vks["factor"], vks["summand"])
	assert np.array_equal(g("soup_sha256"), sha256(np.ascontiguousarray(ours, dtype=np.float32)))
	# materials: names and the texel our constant-material model takes from each *.vkt
	mp = np.ctypeslib.as_array(scene.material_params, (scene.material_count, 8))
	names = bytes(g("material_names")).split(b"\0")
	texels = g("material_texels")
	for m in range(scene.material_count):
		assert names[m] == scene.material_names[m]
		for t, cols in ((0, (0, 1, 2)), (1, (None, 3, 4)), (2, (5, 6, None))):
			half = texels[m, t].view(np.float16)[:4].astype(np.float32)
			for k, col in enumerate(cols):
				if col is not None:
					assert half[k] == mp[m, col]
	lib.vkr_destroy_scene(C.byref(scene), None)


def test_reference_ltc_and_noise_tables_through_the_shim(ref):
	info = H.dataset("cornell")
	lib = api.load_library()
	ltc = api.LtcTable()
	assert lib.vkr_load_ltc_table(C.byref(ltc), None, info["ltc"].encode(), 51) == 0
	r = int(ref["ltc/resolution"][0])
	assert r == ltc.roughness_count == 64
	assert np.array_equal(ref["ltc/table0_sha256"], sha256(np.ctypeslib.as_array(ltc.h_table0, (51, r, r, 4))))
	assert np.array_equal(ref["ltc/table1_sha256"], sha256(np.ctypeslib.as_array(ltc.h_table1, (51, r, r, 2))))
	assert ref["ltc/constants"].tobytes() == bytes(ltc.constants)
	lib.vkr_destroy_ltc_table(C.byref(ltc), None)
	for animate in (0, 1):
		noise = api.NoiseTable()
		assert lib.vkr_load_noise_table(C.byref(noise), None, 256, 256, 64, api.NOISE_WHITE) == 0
		assert np.array_equal(ref["noise/texels_sha256"], sha256(np.ctypeslib.as_array(noise.h_noise, (64 * 256 * 256 * 4,))))
		masks = (C.c_uint32 * 2)(); layer = C.c_uint32(); rnd = (C.c_uint32 * 4)()
		lib.vkr_set_noise_constants(masks, C.byref(layer), rnd, C.byref(noise), animate)
		assert list(ref["noise/constants_animate%d" % animate]) == list(masks) + [layer.value] + list(rnd)
		lib.vkr_destroy_noise_table(C.byref(noise), None)


def test_host_maths_matches_the_reference_bit_for_bit(ref):
	lib = api.load_library()
	lights = cameras = 0
	for a, b, vp in light_trials():
		if vp is not None:
			light, n = a, b
			lib.vkr_set_polygonal_light_vertex_count(C.byref(light), n)
			C.memmove(light.vertices_plane_space, vp.ctypes.data, vp.nbytes)
			lib.vkr_update_polygonal_light(C.byref(light))
			g = lambda key: ref["host_maths/light%03d/%s" % (lights, key)]
			assert bytes(light)[:160] == g("parameters").tobytes(), lights
			assert np.array_equal(np.ctypeslib.as_array(light.vertices_world_space, (n, 4)).view(np.uint32), g("vertices_world_space").view(np.uint32))
			assert np.array_equal(np.ctypeslib.as_array(light.fan_areas, (n - 2, 4)).view(np.uint32), g("fan_areas").view(np.uint32))
			lib.vkr_destroy_polygonal_light(C.byref(light))
			lights += 1
		else:
			cam, aspect = a, b
			m = (C.c_float * 16)()
			lib.vkr_get_world_to_projection_space(m, C.byref(cam), C.c_float(aspect))
			assert bytes(m) == ref["host_maths/world_to_projection"][cameras].tobytes(), cameras
			cameras += 1
	assert lights == cameras == 200


def test_constant_block_pixel_to_ray_uses_the_reference_inverse(ref):
	"""vkr_write_constants inverts the projection with the reference's cofactor expansion (math_utilities.h:24-46)."""
	cb, w2p = world_to_projection_for_the_inverse()
	assert w2p.tobytes() == ref["matrix_inverse/input"].tobytes(), "the world-to-projection matrix drifted: regenerate with tools/make_ref_live_golden.py"
	inv = ref["matrix_inverse/output"].reshape(4, 4)
	vt = np.array([np.float32(2.0) / np.float32(320), np.float32(2.0) / np.float32(200)], dtype=np.float32)
	p2p = np.array([[vt[0], 0, np.float32(0.5) * vt[0] - np.float32(1)], [0, vt[1], np.float32(0.5) * vt[1] - np.float32(1)], [0, 0, 1], [0, 0, 1]], dtype=np.float32)
	expect = np.zeros((3, 4), dtype=np.float32)
	for i in range(3):
		for j in range(3):
			acc = np.float32(0)
			for k in range(4):
				acc = np.float32(acc + np.float32(inv[i, k] * p2p[k, j]))
			expect[i, j] = acc
	got = np.frombuffer(cb[96:144], dtype=np.float32).reshape(3, 4)
	assert np.array_equal(got.view(np.uint32), expect.view(np.uint32))


@pytest.mark.parametrize("name,lights,width,height", CONSTANT_BLOCK_FRAMES)
def test_constant_block_equals_the_reference_host_code(ref, name, lights, width, height):
	"""vkr_write_constants against quick_load + write_constants of the reference (restated over its own structs and functions in oracle/ref_host_probe.c)."""
	from tests.ref_frames import host_constants
	info = H.dataset(name)
	ours = host_constants(info, width, height, lights, sample_count=4)
	theirs = ref["constants/%s_%d_%dx%d" % (name, lights, width, height)].tobytes()
	assert len(ours) == len(theirs)
	assert ours == theirs


def test_noise_blob_files_are_read_as_the_reference_lays_them_out(tmp_path, monkeypatch):
	"""The *.blob branch of load_noise_table (src/noise_table.c:76-107; the reference's timing runs use noise_type_ahmed, src/experiment_list.c:371): raw uint16 RGBA
	cells, layer-major, under data/noise/<type>_<w>x<h>_<layers>.blob. The reference's own loader cannot be the judge here: it formats the path with
	sprintf(file_path, file_path, ...) onto itself (noise_table.c:96, undefined behaviour; with this C library the path comes out empty and the load fails),
	so a synthetic blob is compared with what vkr_load_noise_table hands to the device; a missing file fails."""
	lib = api.load_library()
	monkeypatch.chdir(tmp_path)
	os.makedirs("data/noise")
	w, h, layers = 16, 8, 4
	rng = np.random.default_rng(3)
	cells = rng.integers(0, 65536, w * h * layers * 4, dtype=np.uint16)
	for noise_type, pattern in ((api.NOISE_AHMED, "data/noise/ahmed_2d_rgba_%02dx%02d_%02d.blob"), (api.NOISE_BLUE, "data/noise/blue_noise_rgba_%02dx%02d_%02d.blob")):
		noise = api.NoiseTable()
		assert lib.vkr_load_noise_table(C.byref(noise), None, w, h, layers, noise_type) != 0    # no file yet
		cells.tofile(pattern % (w, h, layers))
		assert lib.vkr_load_noise_table(C.byref(noise), None, w, h, layers, noise_type) == 0
		assert (noise.width, noise.height, noise.layers) == (w, h, layers)
		assert np.array_equal(np.ctypeslib.as_array(noise.h_noise, (len(cells),)), cells)
		masks = (C.c_uint32 * 2)(); layer = C.c_uint32(); rnd = (C.c_uint32 * 4)()
		lib.vkr_set_noise_constants(masks, C.byref(layer), rnd, C.byref(noise), 0)
		assert list(masks) == [w - 1, h - 1] and layer.value == layers - 1
		lib.vkr_destroy_noise_table(C.byref(noise), None)
