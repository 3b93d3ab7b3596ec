"""Seeded synthetic inputs in the reference's own file formats (SURVEY 8d).

The reference ships no data (README.md:8-12), so scenes, material textures, LTC fits and quicksaves
are synthesised here and written as *.vks / *.vkt / fit*.dat / *.save files that the unchanged
reference loaders (and this library's loaders) read. Format sources:
  *.vks   reader src/scene.c:419-483, writer tools/io_export_vulkan_blender28.py:470-531
  *.vkt   src/textures.c:111-169
  fit.dat src/ltc_table.c:46-84
  *.save  src/main.c:49-130
This is authoring tooling (like the reference's Blender exporter), not part of the timed path.
"""
import os
import struct

import contextlib

import numpy as np


@contextlib.contextmanager
def _atomic_write(path):
	"""Writes to a temporary file and renames it: another process reading (or writing) the same data set never sees a truncated file."""
	tmp = "%s.%d.tmp" % (path, os.getpid())
	with open(tmp, "wb") as f:
		yield f
	os.replace(tmp, path)

# ---------------------------------------------------------------------------------------------
# geometry helpers: everything is a list of (triangles[n,3,3], normals[n,3,3], material_id)
# ---------------------------------------------------------------------------------------------

def _grid_quad(origin, edge_u, edge_v, nu, nv, flip=False):
	"""Tessellates the parallelogram origin + s*edge_u + t*edge_v into nu*nv*2 triangles."""
	origin, edge_u, edge_v = (np.asarray(a, dtype=np.float64) for a in (origin, edge_u, edge_v))
	s = np.linspace(0.0, 1.0, nu + 1)
	t = np.linspace(0.0, 1.0, nv + 1)
	S, T = np.meshgrid(s, t, indexing="ij")
	P = origin[None, None, :] + S[..., None] * edge_u[None, None, :] + T[..., None] * edge_v[None, None, :]
	p00, p10, p01, p11 = P[:-1, :-1], P[1:, :-1], P[:-1, 1:], P[1:, 1:]
	t0 = np.stack([p00, p10, p11], axis=2).reshape(-1, 3, 3)
	t1 = np.stack([p00, p11, p01], axis=2).reshape(-1, 3, 3)
	tris = np.concatenate([t0, t1], axis=0)
	if flip:
		tris = tris[:, ::-1, :]
	return tris


def _box(lo, hi, n=1, inward=False):
	"""Axis-aligned box as 6 tessellated faces (n x n quads each); outward normals unless inward."""
	lo = np.asarray(lo, dtype=np.float64); hi = np.asarray(hi, dtype=np.float64)
	d = hi - lo
	ex, ey, ez = np.array([d[0], 0, 0]), np.array([0, d[1], 0]), np.array([0, 0, d[2]])
	faces = [
		_grid_quad(lo, ey, ex, n, n),                    # z = lo (normal -z)
		_grid_quad(lo + ez, ex, ey, n, n),               # z = hi (+z)
		_grid_quad(lo, ex, ez, n, n),                    # y = lo (-y)
		_grid_quad(lo + ey, ez, ex, n, n),               # y = hi (+y)
		_grid_quad(lo, ez, ey, n, n),                    # x = lo (-x)
		_grid_quad(lo + ex, ey, ez, n, n),               # x = hi (+x)
	]
	tris = np.concatenate(faces, axis=0)
	if inward:
		tris = tris[:, ::-1, :]
	return tris


def _flat_normals(tris):
	n = np.cross(tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0])
	n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-30)
	return np.repeat(n[:, None, :], 3, axis=1)


class Mesh:
	def __init__(self):
		self.tris, self.mats = [], []

	def add(self, tris, material):
		self.tris.append(np.asarray(tris, dtype=np.float64))
		self.mats.append(np.full(len(tris), material, dtype=np.uint8))

	def finish(self):
		tris = np.concatenate(self.tris, axis=0)
		mats = np.concatenate(self.mats, axis=0)
		return tris, _flat_normals(tris), mats


# ---------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------

def scene_cornell():
	"""1x1x1 m box open towards -y, two blocks: 5 walls * 2 + 2 boxes * 12 = 34 triangles, 3 materials."""
	m = Mesh()
	m.add(_grid_quad([0, 0, 0], [1, 0, 0], [0, 1, 0], 1, 1), 0)            # floor (+z)
	m.add(_grid_quad([0, 0, 1], [0, 1, 0], [1, 0, 0], 1, 1), 0)            # ceiling (-z)
	m.add(_grid_quad([0, 1, 0], [1, 0, 0], [0, 0, 1], 1, 1), 0)            # back wall (-y)
	m.add(_grid_quad([0, 0, 0], [0, 1, 0], [0, 0, 1], 1, 1), 1)            # left wall (+x), red
	m.add(_grid_quad([1, 0, 0], [0, 0, 1], [0, 1, 0], 1, 1), 2)            # right wall (-x), green
	m.add(_box([0.15, 0.5, 0.0], [0.45, 0.8, 0.6]), 0)
	m.add(_box([0.55, 0.2, 0.0], [0.85, 0.5, 0.3]), 0)
	materials = [
		dict(name="white", base=(0.73, 0.73, 0.73), roughness=0.7, metal=0.0),
		dict(name="red", base=(0.65, 0.05, 0.05), roughness=0.7, metal=0.0),
		dict(name="green", base=(0.12, 0.45, 0.15), roughness=0.7, metal=0.0),
	]
	return m.finish(), materials


def _city_block(m, rng, x0, y0, size, detail, n_mat):
	"""One jittered block: building, awning, poles and clutter. detail scales the tessellation."""
	w = size * rng.uniform(0.45, 0.7); d = size * rng.uniform(0.45, 0.7); h = rng.uniform(4.0, 14.0)
	bx = x0 + rng.uniform(0.05, 0.25) * size; by = y0 + rng.uniform(0.05, 0.25) * size
	mat = int(rng.integers(1, n_mat))
	m.add(_box([bx, by, 0.0], [bx + w, by + d, h], n=max(1, detail)), mat)
	# awning: a slanted quad in front of the building, double sided
	a0 = np.array([bx, by - 1.5, 2.6]); au = np.array([w, 0.0, 0.0]); av = np.array([0.0, 1.5, 0.5])
	na = max(1, detail // 2)
	m.add(_grid_quad(a0, au, av, na, na), int(rng.integers(1, n_mat)))
	m.add(_grid_quad(a0, au, av, na, na, flip=True), int(rng.integers(1, n_mat)))
	# poles
	for k in range(4):
		px = x0 + rng.uniform(0.0, size); py = y0 + rng.uniform(0.0, size)
		m.add(_box([px, py, 0.0], [px + 0.12, py + 0.12, rng.uniform(2.5, 5.0)], n=max(1, detail // 4)), int(rng.integers(1, n_mat)))
	# clutter: small boxes on the ground and on the roof
	for k in range(6 * max(1, detail // 2)):
		cx = x0 + rng.uniform(0.0, size); cy = y0 + rng.uniform(0.0, size); s = rng.uniform(0.15, 0.6)
		on_roof = bx < cx < bx + w - s and by < cy < by + d - s
		z = h if on_roof else 0.0
		m.add(_box([cx, cy, z], [cx + s, cy + s, z + s * rng.uniform(0.5, 2.0)]), int(rng.integers(1, n_mat)))


def scene_city(seed=1, blocks=24, extent=200.0, detail=16, ground_cells=256, n_mat=64):
	"""'bistro_like' stand-in: ground plane + blocks x blocks jittered buildings. Defaults give ~2.8 M triangles."""
	rng = np.random.default_rng(seed)
	m = Mesh()
	m.add(_grid_quad([0, 0, 0], [extent, 0, 0], [0, extent, 0], ground_cells, ground_cells), 0)
	size = extent / blocks
	# an open plaza (the "bistro terrace") in front of the camera: no buildings, but tables, chairs and parasols
	px0, px1, py0, py1 = 0.5 * extent - 22.0, 0.5 * extent + 16.0, 0.5 * extent - 44.0, 0.5 * extent + 2.0
	for i in range(blocks):
		for j in range(blocks):
			x0, y0 = i * size, j * size
			if x0 + size > px0 and x0 < px1 and y0 + size > py0 and y0 < py1:
				continue
			_city_block(m, rng, x0, y0, size, detail, n_mat)
	prng = np.random.default_rng(seed + 500)
	nd = max(1, detail // 4)
	for k in range(40 * max(1, detail // 2)):
		cx = prng.uniform(px0 + 1.0, px1 - 2.0); cy = prng.uniform(py0 + 8.0, py1 - 2.0)
		kind = k % 3
		if kind == 0:   # table: top + leg
			m.add(_box([cx, cy, 0.72], [cx + 0.9, cy + 0.9, 0.78], n=nd), int(prng.integers(1, n_mat)))
			m.add(_box([cx + 0.4, cy + 0.4, 0.0], [cx + 0.5, cy + 0.5, 0.72], n=nd), int(prng.integers(1, n_mat)))
		elif kind == 1: # chair: seat + back
			m.add(_box([cx, cy, 0.42], [cx + 0.45, cy + 0.45, 0.47], n=nd), int(prng.integers(1, n_mat)))
			m.add(_box([cx, cy, 0.47], [cx + 0.45, cy + 0.05, 0.95], n=nd), int(prng.integers(1, n_mat)))
		else:           # parasol: pole + slanted canopy
			m.add(_box([cx, cy, 0.0], [cx + 0.06, cy + 0.06, 2.3], n=nd), int(prng.integers(1, n_mat)))
			m.add(_grid_quad([cx - 1.2, cy - 1.2, 2.2], [2.4, 0.0, 0.2], [0.0, 2.4, 0.1], 2 * nd, 2 * nd), int(prng.integers(1, n_mat)))
			m.add(_grid_quad([cx - 1.2, cy - 1.2, 2.2], [2.4, 0.0, 0.2], [0.0, 2.4, 0.1], 2 * nd, 2 * nd, flip=True), int(prng.integers(1, n_mat)))
	mrng = np.random.default_rng(seed + 1000)
	materials = []
	for k in range(n_mat):
		materials.append(dict(name="mat%03d" % k, base=tuple(mrng.uniform(0.05, 0.9, 3)), roughness=float(np.sqrt(mrng.uniform(0.1, 0.9))),
			metal=float(mrng.random() < 0.2)))
	return m.finish(), materials


def scene_roughness_planes():
	"""Three 4 m x 4 m planes side by side with roughness 0.15 / 0.4 / 0.8 on a dark floor: the stand-in for the reference's
	'roughness planes' scene of the timing experiments (src/experiment_list.c:218-409; the asset itself is not in the repository)."""
	m = Mesh()
	materials = [dict(name="floor", base=(0.2, 0.2, 0.2), roughness=0.9, metal=0.0)]
	m.add(_grid_quad([-40.0, -30.0, 0.0], [80.0, 0.0, 0.0], [0.0, 90.0, 0.0], 16, 18), 0)
	for i, r in enumerate((0.15, 0.4, 0.8)):
		materials.append(dict(name="plane_%d" % i, base=(0.7, 0.7, 0.7), roughness=r, metal=1.0 if i == 0 else 0.0))
		m.add(_grid_quad([-6.5 + 4.5 * i, -2.0, 0.05], [4.0, 0.0, 0.0], [0.0, 4.0, 0.0], 8, 8), 1 + i)
	return m.finish(), materials


def scene_shadowed_plane():
	"""A ground plane with a bollard and a block that cast shadows: stand-in for the reference's 'mis plane' and 'shadowed plane' scenes
	(src/experiment_list.c:170-220, 268-292; the assets are not in the repository)."""
	m = Mesh()
	materials = [dict(name="ground", base=(0.6, 0.6, 0.6), roughness=0.35, metal=0.0), dict(name="occluder", base=(0.3, 0.25, 0.2), roughness=0.6, metal=0.0)]
	m.add(_grid_quad([-20.0, -20.0, 0.0], [40.0, 0.0, 0.0], [0.0, 40.0, 0.0], 20, 20), 0)
	m.add(_box([-0.15, 0.6, 0.0], [0.15, 0.9, 1.1]), 1)
	m.add(_box([1.2, 1.5, 0.0], [2.0, 2.1, 0.6]), 1)
	return m.finish(), materials


def roughness_planes_lights(vertex_count, central, light_count):
	"""Lights of the timing experiments (src/experiment_list.c:366-409): regular polygons with 3 to 7 vertices, either close above the
	planes and facing down (central: the surface normal passes through the polygon for most pixels) or standing beside them
	(decentral), one big light or 128 small ones with the same total flux."""
	rng = np.random.default_rng(1000 * vertex_count + 10 * int(central) + (light_count > 1))
	polygon = [(0.5 + 0.5 * float(np.cos(0.4 + 2.0 * np.pi * k / vertex_count)), 0.5 + 0.5 * float(np.sin(0.4 + 2.0 * np.pi * k / vertex_count))) for k in range(vertex_count)]
	lights = []
	for k in range(light_count):
		scale = 14.0 if light_count == 1 else 1.6
		if central:
			# plane normal = rotation column 2; a rotation about x by pi makes the light face down
			centre = (0.0, 0.0, 1.2) if light_count == 1 else (rng.uniform(-7.0, 7.0), rng.uniform(-5.0, 5.0), rng.uniform(0.9, 1.5))
			angles = (np.pi, 0.0, 0.0) if light_count == 1 else (np.pi + rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.0, 2.0 * np.pi))
			translation = (centre[0] - 0.5 * scale, centre[1] + 0.5 * scale, centre[2]) if light_count == 1 else centre
		else:
			# a rotation about x by pi/2 turns the normal towards -y: an upright light behind the planes
			scale = 6.0 if light_count == 1 else 1.2
			translation = (-3.0, 5.5, 0.3) if light_count == 1 else (rng.uniform(-8.0, 7.0), rng.uniform(4.5, 6.0), rng.uniform(0.2, 3.0))
			angles = (0.5 * np.pi, 0.0, 0.0) if light_count == 1 else (0.5 * np.pi + rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(-0.3, 0.3))
		flux = 40.0 / light_count
		lights.append(make_light(translation, angles, (scale, scale), (flux, flux, flux), polygon))
	return lights


def scene_room(seed=2, detail=48, clutter=2500, n_mat=32):
	"""'attic_like' stand-in: closed 12 x 8 x 4 m room with slanted beams and clutter. Defaults give ~1.0 M triangles."""
	rng = np.random.default_rng(seed)
	m = Mesh()
	m.add(_box([0, 0, 0], [12, 8, 4], n=detail, inward=True), 0)
	for k in range(10):
		x = 1.0 + k * 1.1
		m.add(_box([x, 0.0, 3.4], [x + 0.2, 8.0, 3.7], n=max(1, detail // 6)), 1)
	for k in range(clutter):
		c = np.array([rng.uniform(0.3, 11.4), rng.uniform(0.3, 7.4), 0.0]); s = rng.uniform(0.1, 0.7)
		m.add(_box(c, c + np.array([s, s * rng.uniform(0.5, 1.5), s * rng.uniform(0.5, 3.0)]), n=max(1, detail // 12)), int(rng.integers(1, n_mat)))
	mrng = np.random.default_rng(seed + 1000)
	materials = [dict(name="room%03d" % k, base=tuple(mrng.uniform(0.05, 0.9, 3)), roughness=float(np.sqrt(mrng.uniform(0.1, 0.9))), metal=float(mrng.random() < 0.2)) for k in range(n_mat)]
	return m.finish(), materials


# ---------------------------------------------------------------------------------------------
# *.vks writer
# ---------------------------------------------------------------------------------------------

def _part_1_by_2(x):
	x = x & 0x3FF
	x = (x ^ (x << 16)) & 0xFF0000FF
	x = (x ^ (x << 8)) & 0x0300F00F
	x = (x ^ (x << 4)) & 0x030C30C3
	x = (x ^ (x << 2)) & 0x09249249
	return x


def _encode_octahedral(normal):
	l1 = np.abs(normal).sum(axis=-1, keepdims=True)
	o = normal[..., 0:2] / np.maximum(l1, 1e-30)
	sign_not_zero = np.where(o >= 0.0, 1.0, -1.0)
	o = np.where(normal[..., 2:3] <= 0.0, (1.0 - np.abs(o[..., ::-1])) * sign_not_zero, o)
	factor = float(2 ** 15 - 1)
	return np.asarray(o * factor + (factor + 1.5), dtype=np.uint16)


def write_vks(path, mesh, materials, sort_triangles=True):
	tris, normals, mats = mesh
	n = len(tris)
	if sort_triangles:
		centroids = tris.mean(axis=1).astype(np.float32)
		lo, hi = centroids.min(axis=0), centroids.max(axis=0)
		q = np.minimum(1023, ((centroids - lo) / np.maximum(hi - lo, 1e-30) * 1024.0).astype(np.uint64)).astype(np.uint64)
		morton = _part_1_by_2(q[:, 0]) | (_part_1_by_2(q[:, 1]) << np.uint64(1)) | (_part_1_by_2(q[:, 2]) << np.uint64(2))
		perm = np.argsort(morton, kind="stable")
		tris, normals, mats = tris[perm], normals[perm], mats[perm]
	pos = tris.reshape(-1, 3)
	box_min = pos.min(axis=0); box_max = pos.max(axis=0)
	span = np.maximum(box_max - box_min, 1e-6)
	quantization_factor = 2.0 ** 21 / span
	qp = np.minimum(2 ** 21 - 1, np.asarray(pos * quantization_factor - box_min * quantization_factor, dtype=np.uint32))
	dequantization_factor = (1.0 / quantization_factor).astype(np.float32)
	dequantization_summand = (box_min + 0.5 / quantization_factor).astype(np.float32)
	packed = np.zeros((len(pos), 2), dtype=np.uint32)
	packed[:, 0] = qp[:, 0] + ((qp[:, 1] & 0x7FF) << 21)
	packed[:, 1] = ((qp[:, 1] & 0x1FF800) >> 11) + (qp[:, 2] << 10)
	nuv = np.zeros((len(pos), 4), dtype=np.uint16)
	nuv[:, 0:2] = _encode_octahedral(normals.reshape(-1, 3))
	# planar uv: unit square per triangle
	uv = np.tile(np.array([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0]]), (n, 1))
	nuv[:, 2:4] = np.clip(uv * ((2.0 ** 16 - 1.0) / 8.0) + 0.5, 0.0, 65535.0).astype(np.uint16)
	with _atomic_write(path) as f:
		f.write(struct.pack("<II", 0x00ABCABC, 1))
		f.write(struct.pack("<QQ", len(materials), n))
		f.write(struct.pack("<fff", *dequantization_factor))
		f.write(struct.pack("<fff", *dequantization_summand))
		for mat in materials:
			name = mat["name"].encode("utf-8")
			f.write(struct.pack("<Q", len(name))); f.write(name); f.write(b"\0")
		f.write(packed.astype("<u4").tobytes())
		f.write(nuv.astype("<u2").tobytes())
		f.write(mats.astype(np.uint8).tobytes())
		f.write(struct.pack("<I", 0x00E0FE0F))
	return dict(triangle_count=n, dequantization_factor=dequantization_factor, dequantization_summand=dequantization_summand,
		quantized_positions=packed, normals_and_tex_coords=nuv, material_indices=mats.astype(np.uint8))


# ---------------------------------------------------------------------------------------------
# *.vkt constant textures (RGBA16F, 4x4 with a full mip chain)
# ---------------------------------------------------------------------------------------------

def write_vkt_constant(path, rgba):
	texel = np.asarray(rgba, dtype=np.float16)
	mips = [(4, 4), (2, 2), (1, 1)]
	payload = b""; headers = b""
	for (w, h) in mips:
		data = np.tile(texel, w * h).astype("<f2").tobytes()
		headers += struct.pack("<IIQQ", w, h, len(data), len(payload))
		payload += data
	with _atomic_write(path) as f:
		f.write(struct.pack("<IIIIIIQ", 0x00BC1BC1, 1, len(mips), 4, 4, 97, len(payload)))
		f.write(headers); f.write(payload)
		f.write(struct.pack("<I", 0x00E0FE0F))


def mip_chain(level0):
	"""Box-filtered mip chain of an [H, W, C] array down to 1x1 (what the reference's converter produces with stb's resizer, in spirit)."""
	levels = [np.asarray(level0, dtype=np.float32)]
	while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
		a = levels[-1]; h, w = a.shape[:2]
		if h > 1: a = 0.5 * (a[0:2 * (h // 2):2] + a[1:2 * (h // 2):2])
		if w > 1: a = 0.5 * (a[:, 0:2 * (w // 2):2] + a[:, 1:2 * (w // 2):2])
		levels.append(a.astype(np.float32))
	return levels


def _encode_bc1_block(rgb):
	"""One 4x4 block [4, 4, 3] in [0,1] -> 8 bytes (4-colour mode: endpoints = the extremes along the main diagonal of the colour box)."""
	flat = rgb.reshape(16, 3)
	lo, hi = flat.min(0), flat.max(0)
	def pack(c): return (int(round(c[0] * 31)) << 11) | (int(round(c[1] * 63)) << 5) | int(round(c[2] * 31))
	c0, c1 = pack(hi), pack(lo)
	if c0 == c1:   # one colour: three-colour mode with every index 0
		return struct.pack("<HHI", c0, c1, 0)
	if c0 < c1: c0, c1 = c1, c0
	def unpack(c): return np.array([((c >> 11) & 31) / 31.0, ((c >> 5) & 63) / 63.0, (c & 31) / 31.0])
	a, b = unpack(c0), unpack(c1)
	palette = np.stack([a, b, (2 * a + b) / 3, (a + 2 * b) / 3])
	idx = np.argmin(((flat[:, None, :] - palette[None]) ** 2).sum(-1), axis=1)
	bits = 0
	for t in range(16): bits |= int(idx[t]) << (2 * t)
	return struct.pack("<HHI", c0, c1, bits)


def _encode_bc4_block(values):
	"""One 4x4 block of one channel in [0,1] -> 8 bytes (8-value mode)."""
	flat = values.reshape(16)
	r0, r1 = int(round(float(flat.max()) * 255)), int(round(float(flat.min()) * 255))
	if r0 == r1:
		return struct.pack("<BB", r0, r1) + bytes(6)
	palette = np.array([r0, r1] + [((8 - i) * r0 + (i - 1) * r1) / 7.0 for i in range(2, 8)]) / 255.0
	idx = np.argmin(np.abs(flat[:, None] - palette[None]), axis=1)
	bits = 0
	for t in range(16): bits |= int(idx[t]) << (3 * t)
	return struct.pack("<BB", r0, r1) + bits.to_bytes(6, "little")


def write_vkt(path, level0, vk_format=97):
	"""Writes a *.vkt with a full mip chain (src/textures.c:111-169). level0: [H, W, >=3] floats in [0,1] for the block formats.
	vk_format: 97 R16G16B16A16_SFLOAT, 109 R32G32B32A32_SFLOAT, 131 BC1_RGB_UNORM, 141 BC5_UNORM."""
	levels = mip_chain(level0)
	payload = b""; headers = b""
	for a in levels:
		h, w = a.shape[:2]
		if vk_format in (97, 109):
			rgba = np.concatenate([a[..., :3], np.ones((h, w, 1), dtype=np.float32) if a.shape[-1] < 4 else a[..., 3:4]], axis=-1)
			data = rgba.astype("<f2" if vk_format == 97 else "<f4").tobytes()
		else:
			pad = np.pad(a, ((0, (-h) % 4), (0, (-w) % 4), (0, 0)), mode="edge")
			data = b""
			for by in range(pad.shape[0] // 4):
				for bx in range(pad.shape[1] // 4):
					blk = pad[4 * by:4 * by + 4, 4 * bx:4 * bx + 4]
					data += _encode_bc1_block(blk[..., :3]) if vk_format == 131 else (_encode_bc4_block(blk[..., 0]) + _encode_bc4_block(blk[..., 1]))
		headers += struct.pack("<IIQQ", w, h, len(data), len(payload))
		payload += data
	with _atomic_write(path) as f:
		f.write(struct.pack("<IIIIIIQ", 0x00BC1BC1, 1, len(levels), level0.shape[1], level0.shape[0], vk_format, len(payload)))
		f.write(headers); f.write(payload)
		f.write(struct.pack("<I", 0x00E0FE0F))


def write_light_textures(directory):
	"""Three light textures: [0] an area texture (coloured checker with a soft spot, BC1), [1] a light probe in the theta-phi layout the
	shader expects (u = azimuth / 2 pi, v = polar angle / pi; RGBA16F, values above 1), [2] an IES-like profile (rotationally
	asymmetric lobe, RGBA16F). Returns the three paths."""
	os.makedirs(directory, exist_ok=True)
	paths = [os.path.join(directory, n) for n in ("area.vkt", "probe.vkt", "ies.vkt")]
	v, u = np.meshgrid((np.arange(16) + 0.5) / 16.0, (np.arange(16) + 0.5) / 16.0, indexing="ij")
	checker = ((np.floor(u * 4) + np.floor(v * 4)) % 2)[..., None]
	area = np.clip(checker * np.array([0.9, 0.5, 0.1]) + (1.0 - checker) * np.array([0.1, 0.4, 0.9]) + 0.3 * np.exp(-8.0 * ((u - 0.5) ** 2 + (v - 0.5) ** 2))[..., None], 0.0, 1.0)
	write_vkt(paths[0], area.astype(np.float32), vk_format=131)
	v, u = np.meshgrid((np.arange(16) + 0.5) / 16.0, (np.arange(32) + 0.5) / 32.0, indexing="ij")
	sky = np.stack([0.4 + 0.6 * v, 0.6 + 0.3 * np.cos(2.0 * np.pi * u), 1.2 - 0.8 * v], axis=-1) + 6.0 * np.exp(-40.0 * ((u - 0.3) ** 2 + (v - 0.35) ** 2))[..., None]
	write_vkt(paths[1], sky.astype(np.float32), vk_format=97)
	lobe = (np.cos(np.pi * v) ** 2 * (1.0 + 0.5 * np.cos(4.0 * np.pi * u)))[..., None] * np.array([1.0, 0.95, 0.8])   # bright towards both poles of the light's normal, dark sideways
	write_vkt(paths[2], lobe.astype(np.float32), vk_format=97)
	return paths


def write_material_textures(directory, materials):
	os.makedirs(directory, exist_ok=True)
	for m in materials:
		write_vkt_constant(os.path.join(directory, m["name"] + "_BaseColor.vkt"), list(m["base"]) + [1.0])
		write_vkt_constant(os.path.join(directory, m["name"] + "_Specular.vkt"), [1.0, m["roughness"], m["metal"], 1.0])
		write_vkt_constant(os.path.join(directory, m["name"] + "_Normal.vkt"), [0.5, 0.5, 1.0, 1.0])


def write_patterned_material_textures(directory, materials, seed=5):
	"""Material textures that are not constant, in the formats real assets use (tools/texture_conversion: BC1 base colour, BC5 normals; the
	specular texture as RGBA16F and not square): tiles in the base colour, roughness stripes, a metallic checker for some materials, bumps."""
	os.makedirs(directory, exist_ok=True)
	rng = np.random.default_rng(seed)
	for k, m in enumerate(materials):
		yy, xx = np.mgrid[0:64, 0:64]
		tiles = (((xx // 8) + (yy // 8)) % 2).astype(np.float32)
		base = np.clip(np.asarray(m["base"], dtype=np.float32)[None, None, :] * (0.55 + 0.6 * tiles[..., None]) + 0.05 * rng.random((64, 64, 3)), 0.0, 1.0)
		write_vkt(os.path.join(directory, m["name"] + "_BaseColor.vkt"), base.astype(np.float32), 131)
		yy, xx = np.mgrid[0:16, 0:32]
		roughness = np.clip(m["roughness"] * (0.6 + 0.8 * ((xx // 4) % 2)), 0.05, 1.0)
		metal = ((xx // 8 + yy // 8) % 2) * (1.0 if k % 3 == 0 else 0.0)
		write_vkt(os.path.join(directory, m["name"] + "_Specular.vkt"), np.stack([np.ones((16, 32)), roughness, metal], -1).astype(np.float32), 97)
		yy, xx = np.mgrid[0:32, 0:32]
		normal = np.stack([0.5 + 0.25 * np.sin(xx * 2.0 * np.pi / 8.0), 0.5 + 0.25 * np.cos(yy * 2.0 * np.pi / 16.0), np.ones((32, 32))], -1)
		write_vkt(os.path.join(directory, m["name"] + "_Normal.vkt"), normal.astype(np.float32), 141)


def material_params(materials):
	"""The 8 floats per material the G-buffer producer consumes, after the RGBA16F round trip of the *.vkt files."""
	out = np.zeros((len(materials), 8), dtype=np.float32)
	for i, m in enumerate(materials):
		h = lambda v: np.float32(np.float16(v))
		out[i] = [h(m["base"][0]), h(m["base"][1]), h(m["base"][2]), h(m["roughness"]), h(m["metal"]), h(0.5), h(0.5), 0.0]
	return out


# ---------------------------------------------------------------------------------------------
# LTC fits: a smooth synthetic stand-in, NOT a GGX fit (the real fit*.dat files are not in the repo)
# ---------------------------------------------------------------------------------------------

def write_ltc_fits(directory, resolution=64, fresnel_count=51):
	os.makedirs(directory, exist_ok=True)
	alpha = (np.arange(resolution, dtype=np.float64) / (resolution - 1)) ** 2      # column = sqrt(roughness)
	incl = np.arange(resolution, dtype=np.float64) / (resolution - 1) * (0.5 * np.pi)  # row = inclination
	A, I = np.meshgrid(alpha, incl, indexing="xy")
	for i in range(fresnel_count):
		f0 = i / (fresnel_count - 1)
		a = np.clip(A, 0.01, 1.0)
		m00 = 0.25 + 0.75 * a * (1.0 - 0.3 * np.sin(I))
		m11 = 0.25 + 0.75 * a
		m02 = -0.35 * np.sin(I) * (1.0 - a)
		m20 = 0.15 * np.sin(I) * (1.0 - a) * a
		albedo = np.clip((0.04 + 0.96 * f0) * (1.0 - 0.5 * a) + 0.3 * (1.0 - f0) * (1.0 - np.cos(I)) ** 3, 0.0, 1.0)
		data = np.stack([m00, m02, m11, m20, albedo], axis=-1).astype("<f4")
		with _atomic_write(os.path.join(directory, "fit%d.dat" % i)) as f:
			f.write(struct.pack("<Q", resolution))
			f.write(data.tobytes())


# ---------------------------------------------------------------------------------------------
# quicksaves
# ---------------------------------------------------------------------------------------------

def make_light(translation, rotation_angles, scaling, flux, vertices_plane_space=None):
	if vertices_plane_space is None:
		vertices_plane_space = [(0.0, 0.0), (1.0, 0.0), (1.0, 1.0), (0.0, 1.0)]
	return dict(translation=tuple(float(t) for t in translation), rotation_angles=tuple(float(r) for r in rotation_angles),
		scaling=(float(scaling[0]), float(scaling[1])), flux=tuple(float(f) for f in flux), vertices=[(float(x), float(y)) for x, y in vertices_plane_space])


def write_quicksave(path, camera, lights):
	"""camera: dict(position, rotation_z, rotation_x, vertical_fov, near, far, speed)"""
	with _atomic_write(path) as f:
		f.write(struct.pack("<3f3f2ffi2f", *camera["position"], camera["rotation_z"], camera["rotation_x"], camera["vertical_fov"],
			camera["near"], camera["far"], camera.get("speed", 2.0), 0, 0.0, 0.0))
		f.write(struct.pack("<II", 0, len(lights)))
		for L in lights:
			n = len(L["vertices"])
			# the first 88 bytes of polygonal_light_t: 20 floats + vertex_count + texturing_technique
			f.write(struct.pack("<3ff3ff3ff3ff4f", *L["rotation_angles"], L["scaling"][0], *L["translation"], L["scaling"][1], *L["flux"], 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0))
			f.write(struct.pack("<II", n, int(L.get("texturing_technique", 0))))
			path = L.get("texture_file_path", "").encode()
			f.write(struct.pack("<Q", len(path) + 1 if path else 0))   # texture path with its terminator, 0 = none (src/main.c:94-100)
			if path: f.write(path + b"\0")
			f.write(struct.pack("<QQ", 0, 0))    # legacy NULL pointers
			for (x, y) in L["vertices"]:
				f.write(struct.pack("<4f", x, y, 0.0, 0.0))


def look_at_camera(position, target):
	"""First-person camera at position looking at target: forward = (-sin z, -cos z) horizontally (camera.c:123-129),
	rotation_x = angle from straight down (camera.h:28-30)."""
	d = np.asarray(target, dtype=np.float64) - np.asarray(position, dtype=np.float64)
	d /= np.linalg.norm(d)
	return default_camera(position, float(np.arctan2(-d[0], -d[1])), float(np.arccos(np.clip(-d[2], -1.0, 1.0))))


def default_camera(position, rotation_z, rotation_x):
	return dict(position=tuple(float(p) for p in position), rotation_z=float(rotation_z), rotation_x=float(rotation_x), vertical_fov=float(0.33 * np.pi), near=0.05, far=1.0e3, speed=2.0)


# ---------------------------------------------------------------------------------------------
# named configurations (BASELINE.json configs; synthetic stand-ins, SURVEY 8d)
# ---------------------------------------------------------------------------------------------

def _ceiling_lights(rng, count, x_range, y_range, z_range, scale_range=(0.5, 2.0), flux=10.0):
	lights = []
	for k in range(count):
		s = rng.uniform(*scale_range, size=2)
		pos = (rng.uniform(*x_range), rng.uniform(*y_range), rng.uniform(*z_range))
		# plane normal = rotation column 2; rotate about x by ~pi so that the light faces down, +- 30 degrees
		angles = (np.pi + rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(0.0, 2.0 * np.pi))
		lights.append(make_light(pos, angles, s, (flux, flux, flux)))
	return lights


def build_dataset(directory, name, **overrides):
	"""Writes <name>.vks, <name>_textures/, <name>.save and ggx_ltc_fit/ into directory; returns paths and metadata."""
	os.makedirs(directory, exist_ok=True)
	rng = np.random.default_rng({"cornell": 0, "city": 1, "room": 2, "mini_city": 3, "mini_textured": 3, "mini_lit": 3, "mini_tri": 3, "mini_mixed": 3, "mini_room": 4, "mini_v5": 3, "mini_v6": 3, "mini_v7": 3, "mini_poly": 3}.get(name, 9))
	if name == "cornell":
		mesh, materials = scene_cornell()
		camera = look_at_camera((0.5, -1.2, 0.5), (0.5, 0.5, 0.5))
		lights = [make_light((0.35, 0.35, 0.995), (np.pi, 0.0, 0.0), (0.3, 0.3), (1.0, 1.0, 1.0))]
		lights[0]["translation"] = (0.35, 0.65, 0.995)
		if overrides.get("tilted"):   # cornell_box_tilted_light.save (src/experiment_list.c:247-259)
			lights = [make_light((0.3, 0.75, 0.93), (np.pi + 0.6, 0.25, 0.0), (0.4, 0.3), (1.0, 1.0, 1.0))]
	elif name == "city":
		mesh, materials = scene_city(**{k: v for k, v in overrides.items() if k in ("seed", "blocks", "extent", "detail", "ground_cells", "n_mat")})
		extent = overrides.get("extent", 200.0)
		camera = look_at_camera((0.5 * extent - 3.0, 0.5 * extent - 42.0, 4.5), (0.5 * extent - 3.0, 0.5 * extent - 18.0, 1.0))
		n_lights = overrides.get("lights", 8)
		lights = _ceiling_lights(rng, n_lights, (0.5 * extent - 16.0, 0.5 * extent + 10.0), (0.5 * extent - 34.0, 0.5 * extent - 6.0), (2.6, 4.5), flux=60.0)
		if overrides.get("light_size"):   # "small" / "tiny": one distant light (the reference's Bistro_outside_<size>_light.save, src/experiment_list.c:129-168)
			size = {"small": 0.5, "tiny": 0.08}[overrides["light_size"]]
			lights = [make_light((0.5 * extent - 6.0, 0.5 * extent - 20.0, 9.0), (np.pi + 0.2, 0.1, 0.3), (size, size), (400.0, 400.0, 400.0))]
	elif name == "mini_city":
		mesh, materials = scene_city(seed=3, blocks=4, extent=32.0, detail=2, ground_cells=8, n_mat=8)
		camera = look_at_camera((14.0, 1.0, 5.0), (16.0, 14.0, 1.5))
		lights = _ceiling_lights(rng, overrides.get("lights", 3), (10.0, 22.0), (8.0, 20.0), (2.0, 4.0))
	elif name == "mini_textured":
		# the mini_city scene with material textures that need filtering (SURVEY 8 f1): BC1 base colour, RGBA16F specular, BC5 normals
		mesh, materials = scene_city(seed=3, blocks=4, extent=32.0, detail=2, ground_cells=8, n_mat=8)
		camera = look_at_camera((14.0, 1.0, 5.0), (16.0, 14.0, 1.5))
		lights = _ceiling_lights(rng, overrides.get("lights", 3), (10.0, 22.0), (8.0, 20.0), (2.0, 4.0))
	elif name == "mini_lit":
		# the mini_city scene under textured lights (get_polygon_radiance, shading_pass.frag.glsl:151-185): an area texture (BC1), a light probe seen
		# through a portal and an IES profile (both RGBA16F, theta-phi parametrisation); polygon_texturing_technique_t 1, 2, 3
		mesh, materials = scene_city(seed=3, blocks=4, extent=32.0, detail=2, ground_cells=8, n_mat=8)
		camera = look_at_camera((14.0, 1.0, 5.0), (16.0, 14.0, 1.5))
		lights = _ceiling_lights(rng, overrides.get("lights", 3), (10.0, 22.0), (8.0, 20.0), (2.0, 4.0))
		light_texture_directory = os.path.join(directory, name + "_light_textures")
		paths = write_light_textures(light_texture_directory)
		for i, light in enumerate(lights):
			light["texturing_technique"] = 1 + i % 3
			light["texture_file_path"] = paths[i % 3]
			if overrides.get("vertices"):   # regular polygons of 3 .. 7 vertices instead of quads, as in mini_v5
				n = int(overrides["vertices"]); phase = 0.3 * n
				light["vertices"] = [(0.5 + 0.5 * float(np.cos(phase + 2.0 * np.pi * k / n)), 0.5 + 0.5 * float(np.sin(phase + 2.0 * np.pi * k / n))) for k in range(n)]
	elif name in ("mini_tri", "mini_mixed"):
		# the mini_city scene lit by triangles (MAX_POLYGONAL_LIGHT_VERTEX_COUNT = 3) or by a triangle, a quad and a
		# triangle (MIN_POLYGON_VERTEX_COUNT_BEFORE_CLIPPING = 3 < MAX = 4, main.c:730-732)
		mesh, materials = scene_city(seed=3, blocks=4, extent=32.0, detail=2, ground_cells=8, n_mat=8)
		camera = look_at_camera((14.0, 1.0, 5.0), (16.0, 14.0, 1.5))
		lights = _ceiling_lights(rng, overrides.get("lights", 3), (10.0, 22.0), (8.0, 20.0), (2.0, 4.0))
		triangle = [(0.0, 0.0), (1.0, 0.0), (0.3, 1.0)]
		for i, light in enumerate(lights):
			if name == "mini_tri" or i != 1:
				light["vertices"] = [(float(x), float(y)) for x, y in triangle]
	elif name in ("mini_v5", "mini_v6", "mini_v7", "mini_poly"):
		# the mini_city scene lit by convex pentagons / hexagons / heptagons (MAX_POLYGONAL_LIGHT_VERTEX_COUNT up to 7), or by
		# one of each in one frame
		mesh, materials = scene_city(seed=3, blocks=4, extent=32.0, detail=2, ground_cells=8, n_mat=8)
		camera = look_at_camera((14.0, 1.0, 5.0), (16.0, 14.0, 1.5))
		lights = _ceiling_lights(rng, overrides.get("lights", 3), (10.0, 22.0), (8.0, 20.0), (2.0, 4.0))
		counts = {"mini_v5": [5, 5, 5], "mini_v6": [6, 6, 6], "mini_v7": [7, 7, 7], "mini_poly": [5, 7, 6]}[name]
		for light, n in zip(lights, counts * (len(lights) // 3 + 1)):
			phase = 0.3 * n
			light["vertices"] = [(0.5 + 0.5 * float(np.cos(phase + 2.0 * np.pi * k / n)), 0.5 + 0.5 * float(np.sin(phase + 2.0 * np.pi * k / n))) for k in range(n)]
	elif name == "mini_room":
		# small closed room with 32 lights: the many-lights shape of BASELINE config 4 (constant block of 10 KB)
		mesh, materials = scene_room(seed=4, detail=6, clutter=60, n_mat=8)
		camera = look_at_camera((0.7, 0.7, 1.65), (8.0, 5.0, 1.0))
		lights = _ceiling_lights(rng, overrides.get("lights", 32), (1.0, 11.0), (1.0, 7.0), (2.4, 3.3), scale_range=(0.3, 1.0))
	elif name == "shadowed_plane":
		mesh, materials = scene_shadowed_plane()
		camera = look_at_camera((0.0, -4.0, 2.2), (0.3, 1.0, 0.0))
		lights = [make_light((-1.0, 3.0, 0.4), (0.5 * np.pi + 0.25, 0.0, 0.0), (2.0, 1.2), (25.0, 25.0, 25.0))]
	elif name == "roughness_planes":
		# scene of the reference's timing experiments; overrides: vertices (3..7), central (0/1), lights (1 or 128)
		mesh, materials = scene_roughness_planes()
		camera = look_at_camera((0.0, -6.0, 7.5), (0.0, 0.0, 0.0))
		lights = roughness_planes_lights(int(overrides.get("vertices", 4)), bool(overrides.get("central", 1)), int(overrides.get("lights", 1)))
		if overrides.get("screen"):   # roughness_planes_screen.save (src/experiment_list.c:341-362): an upright rectangular emitter showing a picture
			lights = [make_light((-4.0, 5.5, 0.3), (0.5 * np.pi, 0.0, 0.0), (8.0, 4.5), (60.0, 60.0, 60.0))]
			lights[0]["texturing_technique"] = 1
			lights[0]["texture_file_path"] = write_light_textures(os.path.join(directory, name + "_light_textures"))[0]
	elif name == "room":
		mesh, materials = scene_room(**{k: v for k, v in overrides.items() if k in ("seed", "detail", "clutter", "n_mat")})
		camera = look_at_camera((0.7, 0.7, 1.65), (8.0, 5.0, 1.0))
		lights = _ceiling_lights(rng, overrides.get("lights", 32), (1.0, 11.0), (1.0, 7.0), (2.4, 3.3), scale_range=(0.3, 1.0))
		if overrides.get("ies_profile"):   # attic_ies_profile.save (src/experiment_list.c:294-314): one rectangular ceiling light with an IES profile
			lights = [make_light((5.2, 3.4, 3.6), (np.pi, 0.0, 0.3), (1.6, 0.8), (120.0, 120.0, 120.0))]
			lights[0]["texturing_technique"] = 3
			lights[0]["texture_file_path"] = write_light_textures(os.path.join(directory, name + "_light_textures"))[2]
	else:
		raise ValueError(name)
	vks = os.path.join(directory, name + ".vks")
	tex = os.path.join(directory, name + "_textures")
	save = os.path.join(directory, name + ".save")
	ltc = os.path.join(directory, "ggx_ltc_fit")
	info = write_vks(vks, mesh, materials)
	if name == "mini_textured": write_patterned_material_textures(tex, materials)
	else: write_material_textures(tex, materials)
	write_quicksave(save, camera, lights)
	if not os.path.exists(os.path.join(ltc, "fit50.dat")):
		write_ltc_fits(ltc)
	info.update(textured=(name == "mini_textured"), vks=vks, textures=tex, save=save, ltc=ltc, materials=materials, material_params=material_params(materials), camera=camera, lights=lights)
	return info
