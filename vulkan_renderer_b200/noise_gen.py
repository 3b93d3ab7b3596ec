"""Generating the blue-noise and Ahmed-Wonka noise tables on the device (include/vkr_b200.h, vkr_generate_noise_table / vkr_write_noise_table;
DESIGN.md §5 "Generating the noise tables").

generate_noise_table() runs the generator through libvkr_b200.so (integer arithmetic on the device, bit-identical from run to run; there is no CPU
fallback) and returns the texels as the .blob file holds them; write_noise_table() writes ROOT/data/noise/<name>, which vkr_load_noise_table opens
relative to the working directory and Frame(noise_type=..., noise_root=ROOT) reads. These are this project's tables, not the files of the paper's
data download.

The numpy functions below restate both generators (vkr_noise_gen.cuh) and hold the checks of their properties: elementary-interval nets in 16-bit
integers and the radially averaged power spectrum of a dither array.
"""
import ctypes as C
import itertools
import os

import numpy as np

from . import api

LOADER_SEED = 3124705          # noise_table_t::random_seed as load_noise_table leaves it (src/noise_table.c:48)
FILE_PATTERNS = {api.NOISE_BLUE: "blue_noise_rgba_%02dx%02d_%02d.blob", api.NOISE_AHMED: "ahmed_2d_rgba_%02dx%02d_%02d.blob"}   # noise_table.c:80-91
NAMES = {"blue": api.NOISE_BLUE, "ahmed": api.NOISE_AHMED}
BLUE_SIGMA = 1.5               # vkr_noise_gen.cuh, kBlueSigma
BLUE_WEIGHT_LOG2_SCALE = 28    # kBlueWeightLog2Scale
_TAG_ORDER, _TAG_SCRAMBLE, _TAG_BLUE = 0x4F524452, 0x5343524D, 0x424C5545


def default_size(noise_type):
	"""(width, height, layers) the reference uses for a type (vkr_noise_gen_default_desc)."""
	desc = api.NoiseGenDesc()
	api.load_library().vkr_noise_gen_default_desc(int(noise_type), C.byref(desc))
	return desc.width, desc.height, desc.layers


def file_path(root, noise_type, width, height, layers):
	return os.path.join(root, "data", "noise", FILE_PATTERNS[noise_type] % (width, height, layers))


def generate_noise_table(noise_type, width=None, height=None, layers=None, seed=0, cuda_device=0):
	"""Generates a table on CUDA device cuda_device (default size: the reference's). Returns (texels [layers, height, width, 4] uint16,
	stats dict: device, kernel_ms, relaxation_limit_hits)."""
	lib = api.load_library()
	desc = api.NoiseGenDesc()
	lib.vkr_noise_gen_default_desc(int(noise_type), C.byref(desc))
	desc.width = width or desc.width; desc.height = height or desc.height; desc.layers = layers or desc.layers; desc.seed = seed
	texels = np.zeros((desc.layers, desc.height, desc.width, 4), dtype=np.uint16)
	stats = api.NoiseGenStats()
	device = api.Device()
	if lib.vkr_create_device(C.byref(device), cuda_device, None) != 0:
		raise RuntimeError("vkr_create_device failed for CUDA device %d" % cuda_device)
	try:
		if lib.vkr_generate_noise_table(C.byref(device), C.byref(desc), texels.ctypes.data, C.byref(stats)) != 0:
			raise RuntimeError("vkr_generate_noise_table failed (type %d, %d x %d x %d)" % (noise_type, desc.width, desc.height, desc.layers))
		name = device.name.decode(errors="replace")
	finally:
		lib.vkr_destroy_device(C.byref(device))
	return texels, dict(device=name, kernel_ms=float(stats.kernel_ms), relaxation_limit_hits=int(stats.relaxation_limit_hits))


def write_noise_table(root, noise_type, texels):
	"""Writes texels [layers, height, width, 4] uint16 as root/data/noise/<name> (directories created as needed). Returns the path."""
	texels = np.ascontiguousarray(texels, dtype=np.uint16)
	if texels.ndim != 4 or texels.shape[3] != 4:
		raise ValueError("texels must be [layers, height, width, 4], got %s" % (texels.shape,))
	layers, height, width, _ = texels.shape
	os.makedirs(root, exist_ok=True)
	if api.load_library().vkr_write_noise_table(os.fspath(root).encode(), int(noise_type), width, height, layers, texels.ctypes.data) != 0:
		raise RuntimeError("vkr_write_noise_table failed for %s" % root)
	return file_path(root, noise_type, width, height, layers)


def read_noise_table(root, noise_type, width, height, layers):
	"""root/data/noise/<name> as [layers, height, width, 4] uint16."""
	path = file_path(root, noise_type, width, height, layers)
	texels = np.fromfile(path, dtype="<u2")
	if texels.size != width * height * layers * 4:
		raise ValueError("%s holds %d values, not %d x %d x %d x 4" % (path, texels.size, width, height, layers))
	return texels.reshape(layers, height, width, 4)


# ---- the generators in numpy (vkr_noise_gen.cuh)
def hash32(x):
	x = np.asarray(x, dtype=np.uint32)
	with np.errstate(over="ignore"):
		x = x ^ (x >> np.uint32(16)); x = x * np.uint32(0x7FEB352D); x = x ^ (x >> np.uint32(15)); x = x * np.uint32(0x846CA68B); x = x ^ (x >> np.uint32(16))
	return x


def mix(h, v):
	return hash32(np.bitwise_xor(np.asarray(h, dtype=np.uint32), np.asarray(v, dtype=np.uint32)))


def order_seed(seed, s):
	return mix(mix(hash32(seed), _TAG_ORDER), s)


def scramble_seed(seed, s, dimension):
	return mix(mix(mix(hash32(seed), _TAG_SCRAMBLE), s), dimension)


def array_seed(seed, array):
	return mix(mix(hash32(seed), _TAG_BLUE), array)


_PERMUTATIONS = np.array(list(itertools.permutations(range(4))), dtype=np.uint32)   # lexicographic rank -> permutation of {0,1,2,3}


def hop_index(order, m, x, y):
	i = np.zeros_like(x)
	for k in range(m):
		shift = m - 1 - k
		node = np.uint32(k << 16) | ((y >> np.uint32(shift + 1)) << np.uint32(8)) | (x >> np.uint32(shift + 1))
		quadrant = (((y >> np.uint32(shift)) & np.uint32(1)) << np.uint32(1)) | ((x >> np.uint32(shift)) & np.uint32(1))
		i = (i << np.uint32(2)) | _PERMUTATIONS[mix(order, node) % np.uint32(24), quadrant]
	return i


def bitreverse16(v):
	v = np.asarray(v, dtype=np.uint32)
	v = ((v >> 1) & 0x5555) | ((v & 0x5555) << 1)
	v = ((v >> 2) & 0x3333) | ((v & 0x3333) << 2)
	v = ((v >> 4) & 0x0F0F) | ((v & 0x0F0F) << 4)
	return ((v >> 8) & 0x00FF) | ((v & 0x00FF) << 8)


def sobol1(i):
	i = np.asarray(i, dtype=np.uint32)
	result = np.zeros_like(i); c = 0x8000
	for k in range(16):
		result ^= np.where((i >> np.uint32(k)) & np.uint32(1), np.uint32(c), np.uint32(0))
		c ^= c >> 1
	return result


def owen16(scramble, v):
	v = np.asarray(v, dtype=np.uint32)
	result = v.copy()
	for b in range(16):
		result ^= (mix(scramble, ((v >> np.uint32(b + 1)) << np.uint32(4)) | np.uint32(b)) >> np.uint32(31)) << np.uint32(b)
	return result


def ahmed_layer(seed, size, layer):
	"""Layer `layer` of a size x size Ahmed-Wonka table: [size, size, 4] uint16."""
	m = size.bit_length() - 1
	y, x = np.meshgrid(np.arange(size, dtype=np.uint32), np.arange(size, dtype=np.uint32), indexing="ij")
	out = np.empty((size, size, 4), dtype=np.uint16)
	for pair in range(2):
		s = 2 * layer + pair
		i = hop_index(order_seed(seed, s), m, x, y)
		out[..., 2 * pair] = owen16(scramble_seed(seed, s, 0), bitreverse16(i))
		out[..., 2 * pair + 1] = owen16(scramble_seed(seed, s, 1), sobol1(i))
	return out


def ahmed_table(seed=0, size=256, layers=64):
	return np.stack([ahmed_layer(seed, size, layer) for layer in range(layers)])


def blue_weights(width, height):
	"""The toroidal Gaussian of the dither arrays, [dy, dx] uint32."""
	dx = np.arange(width); dy = np.arange(height)
	x = np.minimum(dx, width - dx).astype(np.float64); y = np.minimum(dy, height - dy).astype(np.float64)
	r2 = y[:, None] * y[:, None] + x[None, :] * x[None, :]
	return np.floor(np.ldexp(np.exp(-r2 / (2.0 * BLUE_SIGMA * BLUE_SIGMA)), BLUE_WEIGHT_LOG2_SCALE) + 0.5).astype(np.uint32)


def dither_array(width, height, seed, array, relaxation_limit=None):
	"""Dither array `array` (= 4 layer + channel) of a blue-noise table with this seed: (values [height, width] uint16, 1 if the relaxation hit
	its iteration limit else 0)."""
	n = width * height
	log2_width = width.bit_length() - 1
	weights = blue_weights(width, height).astype(np.int64)
	p = np.arange(n)
	px = p & (width - 1); py = p >> log2_width
	energy = np.zeros(n, dtype=np.int64)
	member = np.zeros(n, dtype=bool)
	big = np.iinfo(np.int64).max

	def update(q, add):
		w = weights[(py - (q >> log2_width)) & (height - 1), (px - (q & (width - 1))) & (width - 1)]
		energy[:] += w if add else -w
		member[q] = add

	def cluster():
		return int(np.argmax(np.where(member, energy, -1)))

	def void():
		return int(np.argmin(np.where(member, big, energy)))

	ones = n // 10
	a_seed = int(array_seed(seed, array))
	candidate = placed = 0
	while placed != ones:
		q = int(mix(a_seed, candidate)) & (n - 1); candidate += 1
		if not member[q]:
			update(q, True); placed += 1
	limit = n if relaxation_limit is None else relaxation_limit
	hit = 0
	if ones:
		iteration = 0
		while True:
			if iteration == limit:
				hit = 1; break
			c = cluster(); update(c, False)
			v = void()
			if v == c:
				update(c, True); break
			update(v, True); iteration += 1
	prototype = member.copy()
	rank = np.zeros(n, dtype=np.int64)
	for r in range(ones - 1, -1, -1):
		c = cluster(); rank[c] = r; update(c, False)
	assert not energy.any()
	for q in np.flatnonzero(prototype):
		update(int(q), True)
	for r in range(ones, n):
		v = void(); rank[v] = r; update(v, True)
	return ((2 * rank + 1) * (32768 // n)).astype(np.uint16).reshape(height, width), hit


# ---- properties
def net_holds(x, y, t):
	"""Whether the 2^t points (x, y) along the last axis, 16-bit integers, form a (0, t, 2)-net: for every a = 0 .. t, the elementary intervals of
	2^(16-a) x 2^(16-t+a) integers each hold one point. Broadcasts over the leading axes."""
	x = np.asarray(x, dtype=np.int64); y = np.asarray(y, dtype=np.int64)
	ok = np.ones(x.shape[:-1], dtype=bool)
	for a in range(t + 1):
		code = np.sort(((x >> (16 - a)) << (t - a)) | (y >> (16 - (t - a))), axis=-1)
		ok &= (np.diff(code, axis=-1) != 0).all(axis=-1)
	return ok


def blocks(channel, j):
	"""[..., H, W] -> [..., H / 2^j, W / 2^j, 4^j]: the aligned 2^j x 2^j blocks."""
	b = 1 << j
	*lead, h, w = channel.shape
	return channel.reshape(*lead, h // b, b, w // b, b).swapaxes(-3, -2).reshape(*lead, h // b, w // b, b * b)


def radial_power_spectrum(values, band_width=1.0 / 16.0):
	"""Radially averaged power spectrum of a 2D array over its variance (white noise: about 1 in every band). Band k holds the frequencies
	(k band_width, (k + 1) band_width] cycles per pixel; returns the mean of each band, DC left out."""
	a = np.asarray(values, dtype=np.float64)
	a = a - a.mean()
	power = np.abs(np.fft.fft2(a)) ** 2 / a.size / a.var()
	fy = np.fft.fftfreq(a.shape[0])[:, None]; fx = np.fft.fftfreq(a.shape[1])[None, :]
	r = np.sqrt(fx * fx + fy * fy)
	band = np.ceil(r / band_width - 1.0e-9).astype(np.int64) - 1
	keep = r > 0
	count = np.bincount(band[keep], minlength=1)
	total = np.bincount(band[keep], weights=power[keep], minlength=1)
	return total / np.maximum(count, 1)
