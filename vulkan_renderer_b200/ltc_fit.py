"""Fitting the specular BRDF's LTC table on the device (include/vkr_b200.h, vkr_fit_ltc_table / vkr_write_ltc_fits; DESIGN.md §5).

fit_ltc_table() runs the fit through libvkr_b200.so (float64 on the device, bit-identical from run to run; there is no CPU fallback) and returns
the table as the files hold it; write_ltc_fits() writes it as fit<i>.dat, which vkr_load_ltc_table (and Frame) then load. The numpy functions
below restate, in float64, what the shader evaluates from a loaded table, so that a table's fit can be measured where it is used:
quantise() is vkr_load_ltc_table's storage, table_density() evaluate_ltc_density of get_ltc_coefficients' matrix (ltc_utility.glsl:58-108) at a
texel centre, target_lobe() the specular BRDF of brdfs.glsl:74-87 times cos(theta_i).
"""
import ctypes as C
import os

import numpy as np

from . import api

ALPHA_MIN = 1.0e-3          # vkr_ltc_fit.cuh, kAlphaMin
THETA_MAX_DEGREES = 89.5    # vkr_ltc_fit.cuh, kThetaMaxDegrees


def default_desc():
	desc = api.LtcFitDesc()
	api.load_library().vkr_ltc_fit_default_desc(C.byref(desc))
	return desc


def fit_ltc_table(resolution=64, fresnel_count=51, quadrature_size=32, iteration_limit=400, cuda_device=0):
	"""Fits the table on CUDA device cuda_device. Returns (fits [F, N, N, 5] float32 {m00, m02, m11, m20, albedo}, stats dict with the per-cell
	L3 errors [F, N, N] under "cell_errors")."""
	lib = api.load_library()
	desc = api.LtcFitDesc(resolution, fresnel_count, quadrature_size, iteration_limit)
	fits = np.zeros((fresnel_count, resolution, resolution, 5), dtype=np.float32)
	errors = np.zeros((fresnel_count, resolution, resolution), dtype=np.float64)
	stats = api.LtcFitStats()
	stats.cell_errors = errors.ctypes.data_as(C.POINTER(C.c_double))
	device = api.Device()
	if lib.vkr_create_device(C.byref(device), cuda_device, None) != 0:
		raise RuntimeError("vkr_create_device failed for CUDA device %d" % cuda_device)
	try:
		if lib.vkr_fit_ltc_table(C.byref(device), C.byref(desc), fits.ctypes.data, C.byref(stats)) != 0:
			raise RuntimeError("vkr_fit_ltc_table failed (resolution %d, Fresnel count %d, quadrature %d, iteration limit %d)" % (resolution, fresnel_count, quadrature_size, iteration_limit))
		name = device.name.decode(errors="replace")
	finally:
		lib.vkr_destroy_device(C.byref(device))
	return fits, dict(device=name, cell_count=int(stats.cell_count), objective_evaluations=int(stats.objective_evaluations),
		iteration_limit_hits=int(stats.iteration_limit_hits), max_error=stats.max_error, median_error=stats.median_error, mean_error=stats.mean_error,
		fit_ms=float(stats.fit_ms), cell_errors=errors)


def write_ltc_fits(directory, fits):
	"""Writes fits [F, N, N, 5] as directory/fit<i>.dat (created if missing)."""
	fits = np.ascontiguousarray(fits, dtype=np.float32)
	if fits.ndim != 4 or fits.shape[1] != fits.shape[2] or fits.shape[3] != 5:
		raise ValueError("fits must be [F, N, N, 5], got %s" % (fits.shape,))
	os.makedirs(directory, exist_ok=True)
	if api.load_library().vkr_write_ltc_fits(directory.encode(), fits.shape[1], fits.shape[0], fits.ctypes.data) != 0:
		raise RuntimeError("vkr_write_ltc_fits failed for %s" % directory)


def read_ltc_fits(directory, fresnel_count):
	"""The fit<i>.dat files of a directory as [F, N, N, 5] float32."""
	layers = []
	for i in range(fresnel_count):
		with open(os.path.join(directory, "fit%d.dat" % i), "rb") as f:
			n = int(np.frombuffer(f.read(8), dtype="<u8")[0])
			layers.append(np.frombuffer(f.read(n * n * 20), dtype="<f4").reshape(n, n, 5))
	return np.stack(layers)


# ---- what the shader evaluates, in float64
def cell(resolution, fresnel_count, layer, row, column):
	"""(theta, alpha, f0) of a cell as the fit uses it: the texel centre's parameters, clamped at the degenerate ends."""
	theta = min(row / (resolution - 1) * (0.5 * np.pi), np.deg2rad(THETA_MAX_DEGREES))
	return theta, max((column / (resolution - 1)) ** 2, ALPHA_MIN), layer / (fresnel_count - 1)


def quantise(fits):
	"""vkr_load_ltc_table's storage (src/ltc_table.c:86-116) in float32: fits [..., 5] -> (table0 [..., 4], table1 [..., 2]) uint16."""
	m = np.asarray(fits, dtype=np.float32)
	inv = np.stack([m[..., 2], -(m[..., 1] * m[..., 2]), m[..., 0] - m[..., 1] * m[..., 3], -(m[..., 2] * m[..., 3]), m[..., 0] * m[..., 2]], axis=-1)
	inv = inv / np.abs(inv).max(axis=-1, keepdims=True)
	entries = np.stack([inv[..., 0], -inv[..., 1], inv[..., 2], inv[..., 3], inv[..., 4], m[..., 4]], axis=-1).astype(np.float32)
	q = (np.clip(entries, np.float32(0.0), np.float32(1.0)) * np.float32(65535.0) + np.float32(0.5)).astype(np.uint16)
	return q[..., :4], q[..., 4:]


def unclamped_entries(fits):
	"""The six values vkr_load_ltc_table clamps to [0, 1] before quantising, and get_ltc_coefficients' determinant from them (float64)."""
	m = np.asarray(fits, dtype=np.float64)
	inv = np.stack([m[..., 2], -(m[..., 1] * m[..., 2]), m[..., 0] - m[..., 1] * m[..., 3], -(m[..., 2] * m[..., 3]), m[..., 0] * m[..., 2]], axis=-1)
	inv = inv / np.abs(inv).max(axis=-1, keepdims=True)
	entries = np.stack([inv[..., 0], -inv[..., 1], inv[..., 2], inv[..., 3], inv[..., 4], m[..., 4]], axis=-1)
	return entries, entries[..., 2] * (entries[..., 0] * entries[..., 4] + entries[..., 1] * entries[..., 3])


def table_density(texel0, texel1, directions):
	"""evaluate_ltc_density (rcp_projected_solid_angle = 1 / pi) of the matrix get_ltc_coefficients builds from one texel's UNORM16 values, at
	shading-space unit directions [..., 3]."""
	d0 = np.asarray(texel0, dtype=np.float64) / 65535.0; d1 = np.asarray(texel1, dtype=np.float64) / 65535.0
	w = np.asarray(directions, dtype=np.float64)
	x = d0[0] * w[..., 0] + d0[3] * w[..., 2]
	y = d0[2] * w[..., 1]
	z = -d0[1] * w[..., 0] + d1[0] * w[..., 2]
	determinant = d0[2] * (d0[0] * d1[0] + d0[1] * d0[3])
	length_squared = x * x + y * y + z * z
	return np.maximum(z, 0.0) * determinant / (length_squared * length_squared) / np.pi


def target_lobe(theta, alpha, f0, directions):
	"""The specular BRDF of brdfs.glsl:58-87 (diffuse off) times cos(theta_i) for wo = (sin theta, 0, cos theta), zero below the horizon."""
	wi = np.asarray(directions, dtype=np.float64)
	wo = np.array([np.sin(theta), 0.0, np.cos(theta)])
	return np.where(wi[..., 2] > 0.0, specular_brdf(wo, wi, alpha, f0) * wi[..., 2], 0.0)


def specular_brdf(wo, wi, alpha, f0):
	with np.errstate(invalid="ignore", divide="ignore"):
		h = wi + wo
		h = h / np.sqrt((h * h).sum(axis=-1, keepdims=True))
		li = wi[..., 2]; lo = wo[..., 2]
		oh = (wo * h).sum(axis=-1); nh = h[..., 2]
		a2 = alpha * alpha
		ggx = (nh * a2 - nh) * nh + 1.0
		ggx = a2 / (ggx * ggx)
		masking = li * np.sqrt((-lo * a2 + lo) * lo + a2)
		shadowing = lo * np.sqrt((-li * a2 + li) * li + a2)
		smith = 0.5 / (masking + shadowing)
		flipped = 1.0 - np.clip(oh, 0.0, 1.0)
		fresnel = f0 + (1.0 - f0) * (flipped * flipped * flipped * flipped * flipped)
		return ggx * smith * fresnel / np.pi


def hemisphere_grid(theta_steps=1024, phi_steps=1024):
	"""Midpoint grid over the upper hemisphere: (directions [T, P, 3], solid angle weights [T, P])."""
	theta = (np.arange(theta_steps) + 0.5) * (0.5 * np.pi / theta_steps)
	phi = (np.arange(phi_steps) + 0.5) * (2.0 * np.pi / phi_steps)
	T, P = np.meshgrid(theta, phi, indexing="ij")
	directions = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], axis=-1)
	return directions, np.sin(T) * (0.5 * np.pi / theta_steps) * (2.0 * np.pi / phi_steps)


def l1_distance(fits, resolution, fresnel_count, layer, row, column, grid=None):
	"""Integral over the upper hemisphere of |target / albedo - LTC| for one cell of a table, the LTC evaluated as the shader does from the
	quantised texel and the lobe normalised by its integral over the same grid."""
	directions, weights = grid if grid is not None else hemisphere_grid()
	theta, alpha, f0 = cell(resolution, fresnel_count, layer, row, column)
	texel = np.asarray(fits)[layer, row, column]
	t0, t1 = quantise(texel)
	lobe = target_lobe(theta, alpha, f0, directions)
	albedo = float((lobe * weights).sum())
	return float((np.abs(lobe / albedo - table_density(t0, t1, directions)) * weights).sum())
