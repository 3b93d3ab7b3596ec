"""Inputs of the rasterised-visibility tests (tests/test_raster_on_host.py, tests/test_gpu_zzzzzzzzzzzzzz_raster_visibility.py): constant blocks for
the synthetic scenes under their own and random cameras, hand-made scenes in quantised positions, and the CPU builds of the rasteriser and its oracle
(tests/raster_on_host.cpp)."""
import ctypes as C
import os
import struct

import numpy as np

from tests import harness as H
from vulkan_renderer_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libraster_on_host.so")
SCENES = ["cornell", "mini_city", "mini_room", "shadowed_plane", "roughness_planes"]
SIZES = [(61, 37), (160, 90), (257, 129)]
P = lambda a: a.ctypes.data_as(C.c_void_p)


def lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	return C.CDLL(LIB_PATH)


def _u32(n):
	return np.zeros(n, dtype=np.uint32)


def device_code(width, height, constants, q):
	"""vkr_raster.cuh run on the CPU: (visibility, depth)"""
	vis = _u32(width * height); depth = np.zeros(width * height, dtype=np.float32)
	q = np.ascontiguousarray(q, dtype=np.uint32)
	lib().vkr_raster_on_host_visibility(C.c_uint32(width), C.c_uint32(height), C.c_char_p(constants), P(q), C.c_uint64(len(q) // 3), P(vis), P(depth))
	return vis.reshape(height, width), depth.reshape(height, width)


def fragments(width, height, constants, q):
	"""The device code with the depth test off: fragments per pixel and per triangle"""
	q = np.ascontiguousarray(q, dtype=np.uint32)
	per_pixel = _u32(width * height); per_triangle = _u32(len(q) // 3)
	lib().vkr_raster_on_host_fragments(C.c_uint32(width), C.c_uint32(height), C.c_char_p(constants), P(q), C.c_uint64(len(q) // 3), P(per_pixel), P(per_triangle))
	return per_pixel.reshape(height, width), per_triangle


def oracle(width, height, constants, q):
	"""tests/raster_oracle.h: (visibility, depth, fragments per pixel with the depth test off)"""
	vis = _u32(width * height); depth = np.zeros(width * height, dtype=np.float32); frags = _u32(width * height)
	q = np.ascontiguousarray(q, dtype=np.uint32)
	lib().vkr_raster_oracle_visibility(C.c_uint32(width), C.c_uint32(height), C.c_char_p(constants), P(q), C.c_uint64(len(q) // 3), P(vis), P(depth), P(frags))
	return vis.reshape(height, width), depth.reshape(height, width), frags.reshape(height, width)


class SceneConstants:
	"""Constant blocks of one synthetic dataset through the library's host-only loaders, under its own or any other camera."""

	def __init__(self, name):
		self.info = H.dataset(name)
		self.vks = H.read_vks(self.info["vks"])
		self.q = np.ascontiguousarray(self.vks["positions"], dtype=np.uint32)
		self.lib = api.load_library()
		self.scene = api.Scene(); self.ltc = api.LtcTable(); self.noise = api.NoiseTable(); self.spec = api.SceneSpecification(); self.settings = api.RenderSettings()
		assert self.lib.vkr_load_scene(C.byref(self.scene), None, self.info["vks"].encode(), self.info["textures"].encode(), 0) == 0
		assert self.lib.vkr_load_ltc_table(C.byref(self.ltc), None, self.info["ltc"].encode(), 51) == 0
		assert self.lib.vkr_load_noise_table(C.byref(self.noise), None, 256, 256, 64, api.NOISE_WHITE) == 0
		assert self.lib.vkr_quick_load(C.byref(self.spec), self.info["save"].encode()) == 0
		assert self.lib.vkr_create_and_assign_light_textures(None, None, C.byref(self.spec)) == 0
		self.lib.vkr_specify_default_render_settings(C.byref(self.settings)); self.settings.animate_noise = 0; self.settings.exposure_factor = 1.0
		self.camera = api.Camera(); C.memmove(C.byref(self.camera), C.byref(self.spec.camera), C.sizeof(api.Camera))

	def positions(self):
		"""World-space vertices (float64) of the shader's decode, for choosing cameras and for normals."""
		v = self.vks
		x = (self.q[:, 0] & 0x1FFFFF).astype(np.float64)
		y = (((self.q[:, 0] & 0xFFE00000) >> 21) | ((self.q[:, 1] & 0x3FF) << 11)).astype(np.float64)
		z = ((self.q[:, 1] & 0x7FFFFC00) >> 10).astype(np.float64)
		return np.stack([x, y, z], axis=1) * v["factor"].astype(np.float64) + v["summand"].astype(np.float64)

	def constants(self, width, height, camera=None):
		"""camera: None (the quicksave's) or dict(position, rotation_z, rotation_x)"""
		c = self.spec.camera
		C.memmove(C.byref(c), C.byref(self.camera), C.sizeof(api.Camera))
		if camera is not None:
			for i in range(3):
				c.position_world_space[i] = camera["position"][i]
			c.rotation_z = camera["rotation_z"]; c.rotation_x = camera["rotation_x"]
		size = self.lib.vkr_get_constants_size(C.byref(self.spec)); buf = (C.c_uint8 * size)()
		self.lib.vkr_write_constants(buf, C.byref(self.spec), C.byref(self.settings), C.byref(self.scene), C.byref(self.ltc), C.byref(self.noise), width, height)
		return bytes(buf)[:256]

	def close(self):
		self.lib.vkr_destroy_scene_specification(C.byref(self.spec)); self.lib.vkr_destroy_noise_table(C.byref(self.noise), None)
		self.lib.vkr_destroy_ltc_table(C.byref(self.ltc), None); self.lib.vkr_destroy_scene(C.byref(self.scene), None)


def random_cameras(sc, rng, count):
	"""Cameras anywhere in the scene's box (inside geometry too), and cameras looking at a triangle from closer than the effective near plane
	2 f n / (f + n) ~ 0.1, so that clipping cuts triangles."""
	p = sc.positions()
	lo, hi = p.min(axis=0), p.max(axis=0)
	cams = []
	for k in range(count):
		if k % 2 == 0:
			cams.append(dict(position=tuple(rng.uniform(lo, hi)), rotation_z=float(rng.uniform(0.0, 2.0 * np.pi)), rotation_x=float(rng.uniform(0.1, np.pi - 0.1))))
		else:
			t = int(rng.integers(len(p) // 3))
			a, b, c = p[3 * t], p[3 * t + 1], p[3 * t + 2]
			n = np.cross(b - a, c - a); n /= max(np.linalg.norm(n), 1e-30)
			centre = (a + b + c) / 3.0
			eye = centre + n * rng.uniform(0.02, 0.15) + rng.normal(0.0, 0.02, 3)
			cam = synth.look_at_camera(eye, centre + rng.normal(0.0, 0.1, 3))
			cams.append(dict(position=cam["position"], rotation_z=cam["rotation_z"], rotation_x=cam["rotation_x"]))
	return cams


# ---- hand-made scenes: positions are integers q with dequantisation factor 1 and summand 0; with a power-of-two viewport W, H the matrix
#      x_clip = q_x / (128 W) - 1, y_clip = q_y / (128 H) - 1, w = 1 puts vertex q at framebuffer position q / 256 exactly (no rounding anywhere)

def pack(points):
	"""points [n, 3] of non-negative integers < 2^21 -> quantised positions [n, 2]"""
	pts = np.asarray(points, dtype=np.uint64)
	x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
	q = np.zeros((len(pts), 2), dtype=np.uint32)
	q[:, 0] = (x | ((y & 0x7FF) << 21)) & 0xFFFFFFFF
	q[:, 1] = ((y >> 11) | (z << 10)) & 0xFFFFFFFF
	return q


def screen_constants(width, height, z_scale=0.0, z_bias=0.5, factor=(1.0, 1.0, 1.0), summand=(0.0, 0.0, 0.0), matrix=None):
	m = np.zeros((4, 4), dtype=np.float32)
	if matrix is None:
		m[0, 0] = 1.0 / (128.0 * width); m[0, 3] = -1.0
		m[1, 1] = 1.0 / (128.0 * height); m[1, 3] = -1.0
		m[2, 2] = z_scale; m[2, 3] = z_bias
		m[3, 3] = 1.0
	else:
		m[:] = matrix
	buf = bytearray(256)
	struct.pack_into("<3f", buf, 0, *factor); struct.pack_into("<3f", buf, 16, *summand)
	buf[32:96] = m.astype("<f4").tobytes()
	return bytes(buf)


def front_facing(tri):
	"""Orders a screen-space triangle (3 x [X, Y, ...]) so that it is front-facing: Vulkan's a > 0, i.e. (v1 - v0) x (v2 - v0) < 0 with y down."""
	(x0, y0), (x1, y1), (x2, y2) = [(int(v[0]), int(v[1])) for v in tri]
	c = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0)
	return [tri[0], tri[2], tri[1]] if c > 0 else list(tri)


def stand_in(width, height, constants, q):
	"""The ray-cast stand-in: the body of visibility_kernel (tests/device_on_host.cpp, vkr_device_on_host_visibility) over the primary BVH the library
	builds from the shader-decoded vertices. Also returns those vertices (float32, [n, 3, 3])."""
	from tests.test_device_on_host import _lib as device_on_host
	dev = device_on_host()
	q = np.ascontiguousarray(q, dtype=np.uint32)
	n = len(q) // 3
	verts = np.zeros((3 * n, 3), dtype=np.float32)
	dev.vkr_device_on_host_decode_positions(C.c_char_p(constants), P(q), C.c_uint64(3 * n), P(verts))
	lib_ = api.load_library()
	nodes = C.POINTER(C.c_float)(); tris = C.POINTER(C.c_float)(); ids = C.POINTER(C.c_uint32)(); count = C.c_uint64(); depth = C.c_uint32()
	assert lib_.vkr_bvh_build_probe(P(verts), n, C.byref(nodes), C.byref(count), C.byref(tris), C.byref(ids), C.byref(depth)) == 0
	vis = _u32(width * height)
	try:
		dev.vkr_device_on_host_visibility(C.c_uint32(width), C.c_uint32(height), C.c_char_p(constants), nodes, tris, ids, C.c_uint32(n), P(vis))
	finally:
		lib_.vkr_bvh_free_probe(nodes, tris, ids)
	return vis.reshape(height, width), verts.reshape(n, 3, 3)


# ---- where the raster and the stand-in may differ (DESIGN.md §5 "Rasterised visibility", "Against the stand-in")

SNAP_PIXELS = 2.0 ** -0.5 / 256.0 * 2.0 + 2.0 ** -10   # a vertex moves by at most sqrt(2) / 512 pixel when snapped; x2 for both triangles' edges, plus fp32 slack
DEPTH_ULPS = 2.0 ** -20                                # 16 binary32 ulps of a depth below 1.0


def _pixel_geometry(constants, xs, ys):
	m = np.frombuffer(constants[96:144], dtype="<f4").reshape(3, 4)[:, :3].astype(np.float64)
	d = np.stack([xs, ys, np.ones_like(xs)], axis=-1).astype(np.float64) @ m.T
	return d / np.linalg.norm(d, axis=-1, keepdims=True)


def explain_differences(constants, raster, stand, verts):
	"""Classifies every pixel where the raster's and the stand-in's primitive differ. Returns (differing, unexplained, counts per reason)."""
	camera = np.frombuffer(constants[144:156], dtype="<f4").astype(np.float64)
	w2p = np.frombuffer(constants[32:96], dtype="<f4").reshape(4, 4).astype(np.float64)
	ys, xs = np.nonzero(raster != stand)
	counts = dict(edge=0, back_facing=0, near_or_far=0, depth=0)
	unexplained = []
	if len(xs) == 0:
		return 0, unexplained, counts
	v = verts.astype(np.float64)
	d = _pixel_geometry(constants, xs, ys)
	# angle between neighbouring pixel rays: converts angular distances to pixels
	pixel_angle = np.linalg.norm(np.cross(d, _pixel_geometry(constants, xs + 1.0, ys)), axis=-1)

	def edge_pixels(prim, k):
		"""signed distance (pixels) of each ray to the triangle's boundary, positive inside the triangle's cone seen from the camera"""
		a, b, c = (v[prim, i] - camera for i in range(3))
		orient = np.sign(np.einsum("ij,ij->i", a, np.cross(b, c)))
		dist = []
		for p, q in ((a, b), (b, c), (c, a)):
			n = np.cross(p, q)
			dist.append(orient * np.einsum("ij,ij->i", d[k], n) / np.maximum(np.linalg.norm(n, axis=-1), 1e-300) / pixel_angle[k])
		return np.min(np.stack(dist), axis=0)

	def hit(prim, k):
		"""ray parameter and clip coordinates of the ray's intersection with the triangle's plane"""
		a, b, c = v[prim, 0], v[prim, 1], v[prim, 2]
		n = np.cross(b - a, c - a)
		t = np.einsum("ij,ij->i", a - camera, n) / np.einsum("ij,ij->i", d[k], n)
		h = camera + t[:, None] * d[k]
		clip = np.concatenate([h, np.ones((len(h), 1))], axis=1) @ w2p.T
		return t, clip, n

	for k in range(len(xs)):
		r, s = int(raster[ys[k], xs[k]]), int(stand[ys[k], xs[k]])
		kk = np.array([k])
		near_edge = any(abs(edge_pixels(np.array([p]), kk)[0]) <= SNAP_PIXELS for p in (r, s) if p != 0xFFFFFFFF)
		if near_edge:
			counts["edge"] += 1; continue
		if s != 0xFFFFFFFF:
			_, clip_s, n_s = hit(np.array([s]), kk)
			if np.dot(n_s[0], camera - v[s, 0]) <= 0.0:
				counts["back_facing"] += 1; continue
			if not (0.0 <= clip_s[0, 2] <= clip_s[0, 3]):
				counts["near_or_far"] += 1; continue
			if r != 0xFFFFFFFF:
				_, clip_r, _ = hit(np.array([r]), kk)
				z_s, z_r = clip_s[0, 2] / clip_s[0, 3], clip_r[0, 2] / clip_r[0, 3]
				# the depth a snapped vertex moves: its slope per pixel times the snap, for both triangles
				slope = 0.0
				for p in (r, s):
					_, c1, _ = hit(np.array([p]), kk)
					dx = _pixel_geometry(constants, xs[k:k + 1] + 1.0, ys[k:k + 1]); dy = _pixel_geometry(constants, xs[k:k + 1], ys[k:k + 1] + 1.0)
					for dd in (dx, dy):
						a, b, c = v[p, 0], v[p, 1], v[p, 2]
						n = np.cross(b - a, c - a)
						t = np.dot(a - camera, n) / np.dot(dd[0], n)
						c2 = np.append(camera + t * dd[0], 1.0) @ w2p.T
						slope = max(slope, abs(c2[2] / c2[3] - c1[0, 2] / c1[0, 3]))
				if abs(z_s - z_r) <= DEPTH_ULPS + 2.0 * SNAP_PIXELS * slope:
					counts["depth"] += 1; continue
		unexplained.append((int(xs[k]), int(ys[k]), r, s))
	return len(xs), unexplained, counts
