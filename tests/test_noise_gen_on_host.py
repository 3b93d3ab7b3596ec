"""The noise tables (vulkan_renderer_b200/csrc/vkr_noise_gen.cuh) compiled for the CPU (tests/noise_gen_on_host.cpp: the kernels' loops as plain
loops), held against the numpy restatement in vulkan_renderer_b200/noise_gen.py and against the properties their construction promises, plus the
refusals of vkr_generate_noise_table and the .blob round trip through the library's writer and its unchanged loader. The -m gpu tests hold the
kernels against this build bit for bit (tests/test_gpu_zzzzzzzzz_noise_tables.py).

Ahmed-Wonka: 1. host build = numpy over the whole default table.  2. every (layer, pair) point set is a (0,16,2)-net, every aligned 2^j x 2^j block
a (0,2j,2)-net.  3. every channel of every layer is a permutation of 0..65535.  4. no two point sets are equal.
Blue noise: 5. host build = numpy on dither arrays of several sizes.  6. every array holds each value (2r+1) 32768 / N once.  7. its lowest band
of the radially averaged power spectrum lies far below white noise's.
"""
import ctypes as C
import os

import numpy as np
import pytest

from vulkan_renderer_b200 import api, noise_gen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "tests", "build", "libnoise_gen_on_host.so")
AHMED_SIZE, BLUE_SIZE, LAYERS = 256, 64, 64      # the reference's defaults (vkr_noise_gen_default_desc)
# DESIGN.md §5: over the 256 arrays of the default 64 x 64 x 64 blue-noise table the lowest band (up to 1/16 cycles per pixel) of the power
# spectrum over the variance averages 5.9e-5 (largest array 1.03e-4); 64 arrays of white noise of the same size average 0.99 (smallest 0.58).
# The bound leaves a factor of 10 over the largest array.
BLUE_LOW_BAND_BOUND = 1.0e-3


def host_lib():
	if not os.path.exists(LIB_PATH):
		import __graft_entry__ as G
		G.build_device_on_host()
	lib = C.CDLL(LIB_PATH)
	lib.vkr_host_noise_blue_weights.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p]; lib.vkr_host_noise_blue_weights.restype = C.c_uint64
	lib.vkr_host_noise_ahmed.argtypes = [C.c_uint32] * 4 + [C.c_void_p]; lib.vkr_host_noise_ahmed.restype = None
	lib.vkr_host_noise_blue.argtypes = [C.c_uint32] * 5 + [C.c_void_p] * 2; lib.vkr_host_noise_blue.restype = None
	return lib


def host_ahmed(size=AHMED_SIZE, layers=LAYERS, seed=0):
	texels = np.zeros((layers, size, size, 4), dtype=np.uint16)
	host_lib().vkr_host_noise_ahmed(seed, size.bit_length() - 1, 0, layers, texels.ctypes.data)
	return texels


def host_blue(width=BLUE_SIZE, height=BLUE_SIZE, layers=LAYERS, seed=0, first_layer=0):
	"""layers [first_layer, first_layer + layers) of a blue-noise table -> (texels [layers, height, width, 4], limit hits per array)"""
	texels = np.zeros((layers, height, width, 4), dtype=np.uint16)
	hits = np.zeros(4 * layers, dtype=np.uint32)
	host_lib().vkr_host_noise_blue(seed, width, height, 4 * first_layer, 4 * (first_layer + layers), texels.ctypes.data, hits.ctypes.data)
	return texels, hits


@pytest.fixture(scope="module")
def ahmed():
	return host_ahmed()


@pytest.fixture(scope="module")
def point_sets(ahmed):
	"""[128, 256, 256, 2]: set s = 2 layer + pair, (x, y) per pixel"""
	return ahmed.reshape(LAYERS, AHMED_SIZE, AHMED_SIZE, 2, 2).transpose(0, 3, 1, 2, 4).reshape(2 * LAYERS, AHMED_SIZE, AHMED_SIZE, 2)


@pytest.fixture(scope="module")
def blue():
	return host_blue()


def test_ahmed_host_build_equals_numpy(ahmed):
	assert np.array_equal(ahmed, noise_gen.ahmed_table(0, AHMED_SIZE, LAYERS))


def test_ahmed_small_tables_equal_numpy():
	for size in (1, 2, 8, 64):
		assert np.array_equal(host_ahmed(size, 4, seed=11), noise_gen.ahmed_table(11, size, 4)), size


def test_ahmed_point_sets_are_nets(point_sets):
	assert noise_gen.net_holds(point_sets[..., 0].reshape(2 * LAYERS, -1), point_sets[..., 1].reshape(2 * LAYERS, -1), 16).all()


@pytest.mark.parametrize("j", [1, 2, 3, 4])
def test_every_aligned_block_is_a_net(point_sets, j):
	x = noise_gen.blocks(point_sets[..., 0], j); y = noise_gen.blocks(point_sets[..., 1], j)
	assert noise_gen.net_holds(x, y, 2 * j).all()


@pytest.mark.parametrize("j", [5, 6, 7])
def test_a_sample_of_larger_blocks_are_nets(point_sets, j):
	rng = np.random.default_rng(j)
	x = noise_gen.blocks(point_sets[..., 0], j); y = noise_gen.blocks(point_sets[..., 1], j)
	count = AHMED_SIZE >> j
	for _ in range(24):
		s, by, bx = int(rng.integers(2 * LAYERS)), int(rng.integers(count)), int(rng.integers(count))
		assert noise_gen.net_holds(x[s, by, bx], y[s, by, bx], 2 * j), (s, by, bx)


def test_unaligned_blocks_are_not_all_nets(point_sets):
	"""the net property is one of the aligned hierarchy: shifted by one pixel, 2 x 2 blocks stop being (0,2,2)-nets"""
	shifted = np.roll(point_sets, 1, axis=2)
	assert not noise_gen.net_holds(noise_gen.blocks(shifted[..., 0], 1), noise_gen.blocks(shifted[..., 1], 1), 2).all()


def test_every_channel_of_every_layer_is_a_permutation(ahmed):
	values = np.sort(ahmed.reshape(LAYERS, -1, 4), axis=1)
	assert (values == np.arange(65536, dtype=np.uint16)[None, :, None]).all()


def test_no_two_point_sets_are_equal(point_sets):
	rows = np.ascontiguousarray(point_sets.reshape(2 * LAYERS, -1)).view(np.dtype((np.void, 4 * AHMED_SIZE * AHMED_SIZE)))
	assert len(np.unique(rows)) == 2 * LAYERS


def test_blue_weights_equal_numpy():
	for width, height in ((16, 16), (32, 16), (64, 64), (128, 128)):
		weights = np.zeros(width * height, dtype=np.uint32)
		total = host_lib().vkr_host_noise_blue_weights(width, height, weights.ctypes.data)
		assert np.array_equal(weights.reshape(height, width), noise_gen.blue_weights(width, height)), (width, height)
		assert total == int(weights.astype(np.uint64).sum()) and total < 2 ** 32


@pytest.mark.parametrize("width,height,seed,first_layer", [(16, 16, 0, 0), (16, 16, 5, 3), (32, 16, 0, 1), (64, 64, 0, 0), (64, 64, 0, 63), (64, 64, 9, 2)])
def test_blue_host_build_equals_numpy(width, height, seed, first_layer):
	texels, hits = host_blue(width, height, 1, seed, first_layer)
	for channel in (0, 3) if width * height > 1024 else range(4):
		values, hit = noise_gen.dither_array(width, height, seed, 4 * first_layer + channel)
		assert np.array_equal(texels[0, :, :, channel], values), channel
		assert hits[channel] == hit


def test_every_dither_array_holds_every_value_once(blue):
	texels, hits = blue
	expected = (2 * np.arange(BLUE_SIZE * BLUE_SIZE) + 1) * (32768 // (BLUE_SIZE * BLUE_SIZE))
	values = np.sort(texels.reshape(LAYERS, -1, 4), axis=1)
	assert (values == expected[None, :, None]).all()
	print("relaxation limit hits: %d of %d arrays" % (int(hits.sum()), hits.size))


def test_dither_arrays_have_little_low_frequency_power(blue):
	texels, _ = blue
	arrays = texels.transpose(0, 3, 1, 2).reshape(-1, BLUE_SIZE, BLUE_SIZE)
	low = np.array([noise_gen.radial_power_spectrum(a)[0] for a in arrays])
	rng = np.random.default_rng(0)
	white = np.array([noise_gen.radial_power_spectrum(rng.integers(0, 65536, (BLUE_SIZE, BLUE_SIZE)))[0] for _ in range(64)])
	print("lowest band over variance: blue mean %.3e max %.3e; white mean %.3f min %.3f" % (low.mean(), low.max(), white.mean(), white.min()))
	assert white.min() > 0.3
	assert low.max() < BLUE_LOW_BAND_BOUND


def test_different_arrays_differ(blue):
	texels, _ = blue
	arrays = texels.transpose(0, 3, 1, 2).reshape(4 * LAYERS, -1)
	assert len(np.unique(arrays, axis=0)) == 4 * LAYERS


def _desc(noise_type, width, height, layers):
	desc = api.NoiseGenDesc(); desc.type = noise_type; desc.width = width; desc.height = height; desc.layers = layers; desc.seed = 0
	return desc


@pytest.mark.parametrize("noise_type,width,height,layers", [
	(api.NOISE_WHITE, 256, 256, 64), (7, 64, 64, 64),                              # no file of that type
	(api.NOISE_BLUE, 48, 64, 64), (api.NOISE_AHMED, 256, 256, 48), (api.NOISE_BLUE, 64, 64, 0),   # not powers of two
	(api.NOISE_AHMED, 256, 256, 16384),                                            # more layers than the loader reads
	(api.NOISE_AHMED, 256, 128, 64), (api.NOISE_AHMED, 512, 512, 1),               # not square, indices beyond 16 bits
	(api.NOISE_BLUE, 256, 128, 1),                                                 # dither array larger than shared memory holds
])
def test_generate_refuses_before_device_work(capfd, noise_type, width, height, layers):
	lib = api.load_library()
	device = api.Device()    # never created: a refusal must not reach the device
	out = np.zeros(16, dtype=np.uint16)
	assert lib.vkr_generate_noise_table(C.byref(device), C.byref(_desc(noise_type, width, height, layers)), out.ctypes.data, None) == 1
	assert "Failed to generate a noise table:" in capfd.readouterr().out


def test_generate_refuses_a_missing_device_or_descriptor(capfd):
	lib = api.load_library()
	out = np.zeros(16, dtype=np.uint16)
	assert lib.vkr_generate_noise_table(None, C.byref(_desc(api.NOISE_BLUE, 16, 16, 1)), out.ctypes.data, None) == 1
	assert lib.vkr_generate_noise_table(C.byref(api.Device()), None, out.ctypes.data, None) == 1
	assert capfd.readouterr().out.count("Failed to generate a noise table:") == 2


def test_written_tables_load_through_the_unchanged_loader(tmp_path, monkeypatch):
	"""vkr_write_noise_table -> vkr_load_noise_table (run where the files are) gives the same texels and random seed as the route Frame takes:
	read_noise_table and vkr_noise_table_from_image with the loader's seed"""
	lib = api.load_library()
	root = tmp_path / "tables"
	tables = {api.NOISE_AHMED: host_ahmed(seed=3), api.NOISE_BLUE: host_blue(32, 16, 2, seed=3)[0]}   # the default Ahmed size: 33.5 MB
	for noise_type, texels in tables.items():
		path = noise_gen.write_noise_table(str(root), noise_type, texels)
		assert os.path.getsize(path) == texels.nbytes
	monkeypatch.chdir(root)
	for noise_type, texels in tables.items():
		layers, height, width, _ = texels.shape
		loaded = api.NoiseTable()
		assert lib.vkr_load_noise_table(C.byref(loaded), None, width, height, layers, noise_type) == 0
		read = noise_gen.read_noise_table(str(root), noise_type, width, height, layers)
		uploaded = api.NoiseTable()
		assert lib.vkr_noise_table_from_image(C.byref(uploaded), None, width, height, layers, read.ctypes.data, noise_gen.LOADER_SEED) == 0
		for table in (loaded, uploaded):
			assert (table.width, table.height, table.layers, table.random_seed) == (width, height, layers, 3124705)
			assert np.array_equal(np.ctypeslib.as_array(table.h_noise, (texels.size,)), texels.ravel())
			lib.vkr_destroy_noise_table(C.byref(table), None)


def test_write_refuses_what_the_loader_cannot_read(tmp_path, capfd):
	lib = api.load_library()
	texels = np.zeros(64, dtype=np.uint16)
	assert lib.vkr_write_noise_table(str(tmp_path).encode(), api.NOISE_WHITE, 2, 2, 4, texels.ctypes.data) == 1
	assert lib.vkr_write_noise_table(str(tmp_path).encode(), api.NOISE_BLUE, 3, 2, 4, texels.ctypes.data) == 1
	assert lib.vkr_write_noise_table(str(tmp_path / "missing" / "root").encode(), api.NOISE_BLUE, 2, 2, 4, texels.ctypes.data) == 1
	assert "Failed" in capfd.readouterr().out and not (tmp_path / "data").exists()
