"""The rasterised visibility buffer on the GPU (csrc/vkr_raster.cu, vkr_rasterize_visibility; DESIGN.md §5 "Rasterised visibility").

1. It equals the brute-force oracle (tests/raster_oracle.h) on the scenes, sizes and random cameras of tests/test_raster_on_host.py: visibility and depth.
2. At the C3 shape (city, 1920x1080) and the C4 shape (room, 3840x2160) it equals the device code run on the CPU; two C3 runs are identical.
3. A scene loaded without acceleration structure rasterises to the same buffer; vkr_run_visibility_pass still refuses that scene.
4. A whole mini_city frame (raster visibility, G-buffer pass, shading with shadow rays) equals the oracle's shading of the same visibility buffer.
5. NULL arguments, a rasterizer that was not created, a scene larger than the capacity and missing positions are refused; nothing is written.
"""
import ctypes as C

import numpy as np
import pytest

from tests import harness as H
from tests import raster_cases as R
from vulkan_renderer_b200 import api

pytestmark = pytest.mark.gpu


def _rasterize(frame, constants, width, height, rasterizer=None):
	"""(visibility, depth) of vkr_rasterize_visibility on frame's device scene"""
	import torch
	lib = frame.lib
	dev = torch.device("cuda", frame.device.cuda_device)
	own = rasterizer is None
	if own:
		rasterizer = api.Rasterizer()
		assert lib.vkr_create_rasterizer(C.byref(rasterizer), C.byref(frame.device), width, height, max(frame.scene.triangle_count, 1)) == 0
	try:
		vis = torch.full((height, width), 7, dtype=torch.int32, device=dev)
		depth = torch.full((height, width), 7.0, dtype=torch.float32, device=dev)
		torch.cuda.synchronize(dev)
		assert lib.vkr_rasterize_visibility(C.byref(rasterizer), C.byref(frame.device), C.byref(frame.scene), constants, vis.data_ptr(), depth.data_ptr()) == 0
		assert lib.vkr_device_wait_idle(C.byref(frame.device)) == 0
		return vis.cpu().numpy().view(np.uint32), depth.cpu().numpy()
	finally:
		if own:
			lib.vkr_destroy_rasterizer(C.byref(rasterizer), C.byref(frame.device))


def _assert_equal(a, b):
	assert np.array_equal(a[0], b[0]), "%d pixels differ in visibility" % int((a[0] != b[0]).sum())
	assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)), "%d pixels differ in depth" % int((a[1].view(np.uint32) != b[1].view(np.uint32)).sum())


@pytest.mark.parametrize("name", R.SCENES)
def test_rasterizer_equals_the_oracle(name):
	sc = R.SceneConstants(name)
	frame = H.open_frame(sc.info)
	try:
		for width, height in R.SIZES:
			constants = sc.constants(width, height)
			ref = R.oracle(width, height, constants, sc.q)
			_assert_equal(_rasterize(frame, constants, width, height), ref)
		rng = np.random.default_rng(11)
		r = api.Rasterizer()
		assert frame.lib.vkr_create_rasterizer(C.byref(r), C.byref(frame.device), 48, 27, frame.scene.triangle_count) == 0
		try:
			for cam in R.random_cameras(sc, rng, 40):
				constants = sc.constants(48, 27, cam)
				_assert_equal(_rasterize(frame, constants, 48, 27, r), R.oracle(48, 27, constants, sc.q))
		finally:
			frame.lib.vkr_destroy_rasterizer(C.byref(r), C.byref(frame.device))
	finally:
		frame.close(); sc.close()


@pytest.mark.parametrize("name,width,height", [("city", 1920, 1080), ("room", 3840, 2160)])
def test_full_shapes_equal_the_device_code_on_the_cpu(name, width, height):
	sc = R.SceneConstants(name)
	frame = H.open_frame(sc.info, request_acceleration_structure=False)
	try:
		constants = sc.constants(width, height)
		first = _rasterize(frame, constants, width, height)
		_assert_equal(first, R.device_code(width, height, constants, sc.q))
		assert (first[0] != 0xFFFFFFFF).mean() > 0.3
		if name == "city":
			_assert_equal(_rasterize(frame, constants, width, height), first)
	finally:
		frame.close(); sc.close()


def test_a_scene_without_acceleration_structure_rasterizes_and_the_ray_cast_still_refuses_it():
	import torch
	width, height = 160, 90
	sc = R.SceneConstants("mini_city")
	with_as = H.open_frame(sc.info)
	without = H.open_frame(sc.info, request_acceleration_structure=False)
	try:
		constants = sc.constants(width, height)
		_assert_equal(_rasterize(without, constants, width, height), _rasterize(with_as, constants, width, height))
		vis = torch.empty((height, width), dtype=torch.int32, device="cuda:0")
		assert without.lib.vkr_run_visibility_pass(C.byref(without.device), C.byref(without.scene), constants, width, height, vis.data_ptr()) != 0
	finally:
		with_as.close(); without.close(); sc.close()


def test_whole_frame_on_raster_visibility_equals_the_oracle():
	width, height = 160, 90
	info = H.dataset("mini_city")
	oi = H.OracleInputs(info)
	frame = H.open_frame(info)
	try:
		frame.configure(sample_count=2, strategy=api.STRATEGY_DIFFUSE_SPECULAR_MIS, heuristic=api.MIS_OPTIMAL_CLAMPED, trace_shadow_rays=1)
		constants = frame.constants(width, height)
		vis, gb = frame.gbuffer_host(width, height, visibility="raster")
		out = frame.shade_host(width, height, gb)
		ref_gb = oi.gbuffer(width, height, constants, vis)
		ref, _ = oi.shade(H.oracle_config(frame, width, height), constants, ref_gb)
	finally:
		frame.close()
	assert (vis != 0xFFFFFFFF).mean() > 0.3
	assert np.array_equal(gb.view(np.uint32), np.asarray(ref_gb, dtype=np.float32).view(np.uint32))
	assert H.compare_radiance(out, ref)["bit_exact"]


def test_error_cases_are_refused_and_launch_nothing():
	import torch
	width, height = 32, 16
	sc = R.SceneConstants("cornell")
	frame = H.open_frame(sc.info)
	lib = frame.lib
	try:
		constants = sc.constants(width, height)
		r = api.Rasterizer()
		assert lib.vkr_create_rasterizer(C.byref(r), C.byref(frame.device), 0, height, 100) != 0
		assert lib.vkr_create_rasterizer(C.byref(r), C.byref(frame.device), width, 40000, 100) != 0
		assert lib.vkr_create_rasterizer(C.byref(r), C.byref(frame.device), width, height, 0) != 0
		assert lib.vkr_create_rasterizer(None, C.byref(frame.device), width, height, 100) != 0
		assert r.d_keys is None
		lib.vkr_destroy_rasterizer(C.byref(r), C.byref(frame.device))   # a zeroed struct
		vis = torch.full((height, width), 7, dtype=torch.int32, device="cuda:0")
		dev, scene = C.byref(frame.device), C.byref(frame.scene)
		assert lib.vkr_rasterize_visibility(C.byref(r), dev, scene, constants, vis.data_ptr(), None) != 0   # not created
		assert lib.vkr_create_rasterizer(C.byref(r), dev, width, height, frame.scene.triangle_count - 1) == 0
		assert lib.vkr_rasterize_visibility(C.byref(r), dev, scene, constants, vis.data_ptr(), None) != 0   # scene larger than the capacity
		lib.vkr_destroy_rasterizer(C.byref(r), dev)
		assert lib.vkr_create_rasterizer(C.byref(r), dev, width, height, frame.scene.triangle_count) == 0
		try:
			assert lib.vkr_rasterize_visibility(C.byref(r), dev, scene, None, vis.data_ptr(), None) != 0
			assert lib.vkr_rasterize_visibility(C.byref(r), dev, scene, constants, None, None) != 0
			assert lib.vkr_rasterize_visibility(C.byref(r), dev, None, constants, vis.data_ptr(), None) != 0
			assert lib.vkr_rasterize_visibility(C.byref(r), None, scene, constants, vis.data_ptr(), None) != 0
			assert lib.vkr_rasterize_visibility(None, dev, scene, constants, vis.data_ptr(), None) != 0
			no_positions = api.Scene(); C.memmove(C.byref(no_positions), scene, C.sizeof(api.Scene)); no_positions.d_quantized_positions = None
			assert lib.vkr_rasterize_visibility(C.byref(r), dev, C.byref(no_positions), constants, vis.data_ptr(), None) != 0
			assert lib.vkr_device_wait_idle(dev) == 0
			assert (vis.cpu().numpy() == 7).all()
			assert lib.vkr_rasterize_visibility(C.byref(r), dev, scene, constants, vis.data_ptr(), None) == 0
			assert lib.vkr_device_wait_idle(dev) == 0
			assert (vis.cpu().numpy() != 7).all()
		finally:
			lib.vkr_destroy_rasterizer(C.byref(r), dev)
	finally:
		frame.close(); sc.close()
