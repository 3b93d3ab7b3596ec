"""The rasterised visibility buffer on the CPU (DESIGN.md §5 "Rasterised visibility"): the device code of csrc/vkr_raster.cuh, compiled for the host
by tests/raster_on_host.cpp, against the brute-force oracle (tests/raster_oracle.h) and against the invariants Vulkan's rules imply: watertight
coverage with the top-left rule, facing tied to the scenes' counter-clockwise winding, clipping at the effective near plane, ties in draw order."""
import numpy as np
import pytest

from tests import raster_cases as R


def _assert_equal(a, b):
	va, da = a[0], a[1]
	vb, db = b[0], b[1]
	assert np.array_equal(va, vb), "%d pixels differ in visibility" % int((va != vb).sum())
	assert np.array_equal(da.view(np.uint32), db.view(np.uint32)), "%d pixels differ in depth" % int((da.view(np.uint32) != db.view(np.uint32)).sum())


@pytest.mark.parametrize("size", R.SIZES, ids=["%dx%d" % s for s in R.SIZES])
@pytest.mark.parametrize("name", R.SCENES)
def test_device_code_equals_the_oracle(name, size):
	width, height = size
	sc = R.SceneConstants(name)
	try:
		constants = sc.constants(width, height)
		dev = R.device_code(width, height, constants, sc.q)
		ref = R.oracle(width, height, constants, sc.q)
	finally:
		sc.close()
	_assert_equal(dev, ref)
	drawn = dev[0] != 0xFFFFFFFF
	assert drawn.mean() > 0.2
	assert (dev[1][drawn] < 1.0).all() and (dev[1][drawn] >= 0.0).all() and (dev[1][~drawn] == 1.0).all()


def test_device_code_equals_the_oracle_under_random_cameras():
	"""200 cameras: anywhere in each scene's box, inside geometry too, and closer to a triangle than the effective near plane."""
	rng = np.random.default_rng(11)
	width, height = 48, 27
	clipped = 0
	for name in R.SCENES:
		sc = R.SceneConstants(name)
		try:
			for cam in R.random_cameras(sc, rng, 40):
				constants = sc.constants(width, height, cam)
				dev = R.device_code(width, height, constants, sc.q)
				ref = R.oracle(width, height, constants, sc.q)
				_assert_equal(dev, ref)
				clipped += int(_near_plane_cuts_a_visible_triangle(constants, sc.positions()))
		finally:
			sc.close()
	assert clipped >= 20


def _near_plane_cuts_a_visible_triangle(constants, positions):
	"""Some triangle has a vertex in front of the plane z_clip = 0 and inside the view, and another vertex behind it (float64, approximately)."""
	m = np.frombuffer(constants[32:96], dtype="<f4").reshape(4, 4).astype(np.float64)
	c = np.concatenate([positions, np.ones((len(positions), 1))], axis=1) @ m.T
	c = c.reshape(-1, 3, 4)
	in_view = (c[..., 2] > 0) & (c[..., 2] < c[..., 3]) & (np.abs(c[..., 0]) < c[..., 3]) & (np.abs(c[..., 1]) < c[..., 3])
	behind = c[..., 2] < 0
	return bool((in_view.any(axis=1) & behind.any(axis=1)).any())


def _grid_scene(rng, nx, ny, x0, y0, x1, y1, jitter):
	"""A rectangle [x0, x1] x [y0, y1] (sub-pixel units) tessellated into nx * ny quads, inner vertices moved by up to `jitter`; every triangle front-facing."""
	xs = np.linspace(x0, x1, nx + 1); ys = np.linspace(y0, y1, ny + 1)
	P = np.zeros((nx + 1, ny + 1, 2), dtype=np.int64)
	for i in range(nx + 1):
		for j in range(ny + 1):
			dx = rng.integers(-jitter, jitter + 1) if 0 < i < nx else 0
			dy = rng.integers(-jitter, jitter + 1) if 0 < j < ny else 0
			P[i, j] = (int(round(xs[i])) + dx, int(round(ys[j])) + dy)
	tris = []
	for i in range(nx):
		for j in range(ny):
			a, b, c, d = P[i, j], P[i + 1, j], P[i + 1, j + 1], P[i, j + 1]
			split = rng.integers(2)
			for t in ([a, b, c], [a, c, d]) if split else ([a, b, d], [b, c, d]):
				tris.append(R.front_facing([(int(v[0]), int(v[1]), 0) for v in t]))
	return R.pack([v for t in tris for v in t])


def _centres(width, height):
	y, x = np.mgrid[0:height, 0:width]
	return x * 256 + 128, y * 256 + 128


@pytest.mark.parametrize("seed", range(6))
def test_tessellated_grids_are_watertight(seed):
	"""Depth test off: every pixel centre strictly inside the rectangle is covered exactly once, every one outside not at all."""
	rng = np.random.default_rng(seed)
	width = height = 64
	x0, y0 = int(rng.integers(256, 2048)), int(rng.integers(256, 2048))
	x1, y1 = int(rng.integers(10000, 15000)), int(rng.integers(10000, 15000))
	q = _grid_scene(rng, int(rng.integers(2, 12)), int(rng.integers(2, 12)), x0, y0, x1, y1, jitter=int(rng.integers(0, 300)))
	constants = R.screen_constants(width, height)
	per_pixel, _ = R.fragments(width, height, constants, q)
	px, py = _centres(width, height)
	inside = (px > x0) & (px < x1) & (py > y0) & (py < y1)
	outside = (px < x0) | (px > x1) | (py < y0) | (py > y1)
	assert (per_pixel[inside] == 1).all(), int((per_pixel[inside] != 1).sum())
	assert (per_pixel[outside] == 0).all()
	assert np.array_equal(per_pixel, R.oracle(width, height, constants, q)[2])


@pytest.mark.parametrize("seed", range(6))
def test_fans_are_watertight(seed):
	"""A convex polygon fanned around an inner vertex at a random sub-pixel position; centres strictly inside are covered exactly once."""
	rng = np.random.default_rng(100 + seed)
	width = height = 64
	n = int(rng.integers(3, 24))
	# convex by construction: every angular gap is below pi (at most 1 / (1 + 0.6 (n - 1)) <= 0.455 of the turn), so the ring also keeps the
	# circle's centre at least r cos(0.455 pi) = 0.14 r inside
	gaps = rng.uniform(0.6, 1.0, n)
	angles = np.cumsum(gaps / gaps.sum() * 2.0 * np.pi) + rng.uniform(0.0, 2.0 * np.pi)
	cx, cy, r = 8192 + int(rng.integers(-500, 500)), 8192 + int(rng.integers(-500, 500)), 6000
	ring = [(int(cx + r * np.cos(a)), int(cy + r * np.sin(a))) for a in angles]
	centre = (cx + int(rng.integers(-200, 200)), cy + int(rng.integers(-200, 200)))
	tris = [R.front_facing([(centre[0], centre[1], 0), (ring[i][0], ring[i][1], 0), (ring[(i + 1) % n][0], ring[(i + 1) % n][1], 0)]) for i in range(n)]
	q = R.pack([v for t in tris for v in t])
	constants = R.screen_constants(width, height)
	per_pixel, _ = R.fragments(width, height, constants, q)
	px, py = _centres(width, height)
	# strictly inside the ring polygon (counter-clockwise in y-up terms: the sorted angles), exactly
	inside = np.ones_like(px, dtype=bool); outside = np.zeros_like(px, dtype=bool)
	for i in range(n):
		(ax, ay), (bx, by) = ring[i], ring[(i + 1) % n]
		e = (bx - ax) * (py - ay) - (by - ay) * (px - ax)
		inside &= e > 0; outside |= e < 0
	assert (per_pixel[inside] == 1).all()
	assert (per_pixel[outside] == 0).all()


def test_centres_on_edges_and_vertices_follow_the_top_left_rule():
	"""Vertices on pixel centres: a square cut along either diagonal, grids whose every edge and vertex passes through pixel centres."""
	width = height = 64
	constants = R.screen_constants(width, height)
	c = lambda i: 256 * i + 128   # centre of pixel i
	px, py = _centres(width, height)
	for diagonal in (0, 1):
		a, b, cc, d = (c(10), c(12)), (c(30), c(12)), (c(30), c(40)), (c(10), c(40))
		quads = ([a, b, cc], [a, cc, d]) if diagonal else ([a, b, d], [b, cc, d])
		q = R.pack([v for t in quads for v in R.front_facing([tuple(p) + (0,) for p in t])])
		per_pixel, per_tri = R.fragments(width, height, constants, q)
		# top and left edges are in, bottom and right edges out: columns 10..29, rows 12..39
		expected = (px >= c(10)) & (px < c(30)) & (py >= c(12)) & (py < c(40))
		assert np.array_equal(per_pixel, expected.astype(np.uint32))
		assert per_tri.sum() == 20 * 28
	# a single triangle: its horizontal top edge is in, its sloped right edge (centres on it at every second row) is out, its left edge is in
	tri = R.front_facing([(c(4), c(4), 0), (c(20), c(4), 0), (c(4), c(36), 0)])
	per_pixel, _ = R.fragments(width, height, constants, R.pack(tri))
	assert per_pixel[4, 4] == 1 and per_pixel[4, 19] == 1 and per_pixel[4, 20] == 0 and per_pixel[36, 4] == 0
	assert per_pixel[6, 19] == 0 and per_pixel[6, 18] == 1    # (19, 6) lies on the hypotenuse from (20, 4) to (4, 36): a right edge
	# grids with vertices on centres, spacing two pixels: every edge and vertex passes through centres
	rng = np.random.default_rng(3)
	q = _grid_scene(rng, 8, 6, c(8), c(8), c(24), c(20), jitter=0)
	per_pixel, _ = R.fragments(width, height, constants, q)
	expected = (px >= c(8)) & (px < c(24)) & (py >= c(8)) & (py < c(20))
	assert np.array_equal(per_pixel, expected.astype(np.uint32))


@pytest.mark.parametrize("name", R.SCENES)
def test_exactly_one_of_a_triangle_and_its_reverse_is_drawn_and_it_faces_the_camera(name):
	"""Ties the sign convention to the scenes' counter-clockwise winding (synth._grid_quad): the drawn one of each pair has its geometric normal
	(v1 - v0) x (v2 - v0) towards the camera."""
	width, height = 160, 90
	sc = R.SceneConstants(name)
	try:
		constants = sc.constants(width, height)
		p = sc.positions()
	finally:
		sc.close()
	n = len(sc.q) // 3
	reversed_q = sc.q.reshape(n, 3, 2)[:, ::-1, :].reshape(-1, 2)
	_, per_tri = R.fragments(width, height, constants, np.concatenate([sc.q, reversed_q]))
	fwd, rev = per_tri[:n], per_tri[n:]
	assert not ((fwd > 0) & (rev > 0)).any()
	camera = np.frombuffer(constants[144:156], dtype="<f4").astype(np.float64)
	t = p.reshape(n, 3, 3)
	normal = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
	towards = np.einsum("ij,ij->i", normal, camera - t[:, 0])
	assert (towards[fwd > 0] > 0).all()
	assert (towards[rev > 0] < 0).all()
	assert (fwd > 0).sum() > 0.05 * n


# ---- clipping: an identity view (camera at the origin looking down -z) and camera.c's projection, n = 0.05, f = 1000

_N, _F = 0.05, 1000.0


def _projection(width, height, fov=1.0367255756846319):
	top = np.tan(0.5 * fov); right = width / height * top
	return np.array([[-1.0 / right, 0, 0, 0], [0, 1.0 / top, 0, 0], [0, 0, -(_F + _N) / (_F - _N), -2.0 * _F * _N / (_F - _N)], [0, 0, -1.0, 0]], dtype=np.float32)


def _view_scene(tris_view, width=64, height=48):
	"""Triangles in view space (metres, 1/1024 m steps within +-1024 m) -> quantised positions and constants"""
	factor = 1.0 / 1024.0; summand = -1024.0
	pts = [tuple(int(round((c - summand) / factor)) for c in v) for t in tris_view for v in t]
	constants = R.screen_constants(width, height, factor=(factor,) * 3, summand=(summand,) * 3, matrix=_projection(width, height))
	return R.pack(pts), constants


def _facing_triangle(depth, size):
	"""A triangle facing the camera at view depth `depth` (z = -depth), counter-clockwise seen from the camera"""
	return [(-size, -size, -depth), (size, -size, -depth), (0.0, size, -depth)]


def test_clipping_at_the_effective_near_plane_and_the_far_plane():
	width, height = 64, 48
	near_effective = 2.0 * _F * _N / (_F + _N)   # ~0.1: where camera.c's z_clip = 0
	cases = [
		(0.075, 0.0),                 # between n and 2fn/(f+n): clipped away, the quirk of the OpenGL-style projection under Vulkan's clip volume
		(near_effective * 1.05, 1.0), # just beyond it: drawn
		(10.0, 1.0),
		(_F * 1.01, 0.0),             # beyond f
	]
	for depth, drawn in cases:
		size = depth * 0.2
		q, constants = _view_scene([_facing_triangle(depth, size)], width, height)
		vis, d, _ = R.oracle(width, height, constants, q)
		dev = R.device_code(width, height, constants, q)
		_assert_equal(dev, (vis, d))
		assert ((vis == 0).any()) == bool(drawn), depth
	# behind the camera: nothing; crossing w = 0: only the part in front, which reaches the screen's edge
	q, constants = _view_scene([[(-1.0, -1.0, 2.0), (1.0, -1.0, 2.0), (0.0, 1.0, 2.0)]], width, height)
	assert (R.device_code(width, height, constants, q)[0] == 0xFFFFFFFF).all()
	q, constants = _view_scene([[(0.0, 0.3, 3.0), (0.5, -0.3, -2.0), (-0.5, -0.3, -2.0)]], width, height)
	dev = R.device_code(width, height, constants, q)
	_assert_equal(dev, R.oracle(width, height, constants, q)[:2])
	assert (dev[0] == 0).sum() > 0


def test_a_screen_filling_triangle_covers_what_the_same_plane_cut_into_pieces_covers():
	"""Far-off vertices cross the guard band (and the screen's edges by far): clipped, it covers every pixel, as the plane's pieces do."""
	width, height = 64, 48
	depth = 5.0
	big = [(-900.0, -900.0, -depth), (900.0, -900.0, -depth), (0.0, 900.0, -depth)]
	q, constants = _view_scene([big], width, height)
	vis, _ = R.device_code(width, height, constants, q)
	pieces = []
	xs = np.linspace(-6.0, 6.0, 5); ys = np.linspace(-6.0, 6.0, 4)
	for i in range(4):
		for j in range(3):
			a, b, c, d = (xs[i], ys[j], -depth), (xs[i + 1], ys[j], -depth), (xs[i + 1], ys[j + 1], -depth), (xs[i], ys[j + 1], -depth)
			pieces += [[a, b, c], [a, c, d]]
	q2, constants2 = _view_scene(pieces, width, height)
	vis2, _ = R.device_code(width, height, constants2, q2)
	assert (vis == 0).all()
	assert (vis2 != 0xFFFFFFFF).all()


def test_ties_go_to_the_lower_primitive_and_zero_area_draws_nothing():
	width = height = 64
	constants = R.screen_constants(width, height)
	tri = R.front_facing([(1000, 1000, 0), (12000, 2000, 0), (5000, 14000, 0)])
	degenerate = [(1000, 1000, 0), (6000, 6000, 0), (11000, 11000, 0)]
	q = R.pack(degenerate + tri + tri + degenerate[::-1])
	vis, depth = R.device_code(width, height, constants, q)
	_assert_equal((vis, depth), R.oracle(width, height, constants, q)[:2])
	assert set(np.unique(vis)) == {1, 0xFFFFFFFF}
	_, per_tri = R.fragments(width, height, constants, q)
	assert per_tri[0] == 0 and per_tri[3] == 0 and per_tri[1] == per_tri[2] > 0


def test_every_pixel_where_the_raster_and_the_ray_cast_stand_in_differ_is_explained():
	"""Against the stand-in (the body of visibility_kernel on the CPU, over the library's primary BVH), on the scenes, sizes and random cameras above.
	Each differing pixel's centre lies within SNAP_PIXELS of an edge of either chosen triangle, or the stand-in's triangle faces away, or its hit lies
	outside 0 <= z <= w (nearer than 2fn/(f+n) or beyond f), or the two depths agree within DEPTH_ULPS plus what snapping moves. The same raster
	flipped upside down leaves most of its differences unexplained: this ties the raster's viewport to the pixel rays the G-buffer pass intersects."""
	rng = np.random.default_rng(11)
	report = {}
	for name in R.SCENES:
		sc = R.SceneConstants(name)
		try:
			cases = [(w, h, None) for w, h in R.SIZES] + [(48, 27, cam) for cam in R.random_cameras(sc, rng, 40)]
			for w, h, cam in cases:
				constants = sc.constants(w, h, cam)
				raster, _ = R.device_code(w, h, constants, sc.q)
				stand, verts = R.stand_in(w, h, constants, sc.q)
				differing, unexplained, counts = R.explain_differences(constants, raster, stand, verts)
				assert not unexplained, (name, w, h, cam, unexplained[:8])
				key = (name, "own camera" if cam is None else "random cameras")
				acc = report.setdefault(key, dict(pixels=0, differing=0, edge=0, back_facing=0, near_or_far=0, depth=0))
				acc["pixels"] += w * h; acc["differing"] += differing
				for k, v in counts.items():
					acc[k] += v
				if cam is None and (w, h) == R.SIZES[1]:
					assert len(R.explain_differences(constants, raster[::-1].copy(), stand, verts)[1]) > 0.05 * w * h
		finally:
			sc.close()
	for key, acc in sorted(report.items()):
		print("%s, %s: %.3f %% of %d pixels differ %s" % (key[0], key[1], 100.0 * acc["differing"] / acc["pixels"], acc["pixels"],
			{k: acc[k] for k in ("edge", "back_facing", "near_or_far", "depth")}))
	own = [acc for key, acc in report.items() if key[1] == "own camera"]
	assert sum(a["differing"] for a in own) < 0.01 * sum(a["pixels"] for a in own)
