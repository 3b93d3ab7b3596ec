// tests/jpeg_on_host.cpp -- TEST INFRASTRUCTURE: the JPEG encoder (vulkan_renderer_b200/csrc/vkr_jpeg.cuh) compiled for the CPU. Loops stand in for
// the launches of vkr_jpeg.cu stage by stage: transform every block, count its bits, an exclusive scan of the counts, emit every block at its offset
// into zeroed words, count the 0xFF bytes per chunk, scan them and stuff. tests/test_jpeg_on_host.py holds this against stb_image_write's bytes; the
// -m gpu tests hold the kernels against this. Built by __graft_entry__.build() into tests/build/libjpeg_on_host.so. Nothing in the product links
// against it.
#include <cstdint>
#include <cstring>
#include <vector>

#include "vkr_jpeg.cuh"

using namespace vkr_jpeg;

// the file for rgb8 (width x height x 3) at quality; returns 1 without writing past capacity if it does not fit, *out_size = the file's size
extern "C" int vkr_host_encode_jpg(const uint8_t* rgb8, uint32_t width, uint32_t height, int quality, uint8_t* out_file, size_t capacity, size_t* out_size) {
	if (check_request("encode a JPEG on the host", rgb8, width, height, out_file, out_size)) return 1;
	Params p;
	make_params(quality, width, height, &p);
	const uint64_t n = p.block_count;
	std::vector<int16_t> coefficients(64 * n);
	for (uint64_t b = 0; b != n; ++b) transform_block(p, rgb8, b, coefficients.data() + 64 * b);
	std::vector<uint64_t> offsets(n + 1, 0);
	for (uint64_t b = 0; b != n; ++b) offsets[b + 1] = offsets[b] + block_bits(p, coefficients.data(), b);
	const uint64_t byte_count = (offsets[n] + 7) / 8;
	std::vector<uint32_t> words((byte_count + 3) / 4, 0);
	for (uint64_t b = 0; b != n; ++b) emit_block(p, coefficients.data(), offsets.data(), b, words.data());
	const uint64_t chunks = (byte_count + kChunkBytes - 1) / kChunkBytes;
	std::vector<uint64_t> ff_before(chunks + 1, 0);
	for (uint64_t c = 0; c != chunks; ++c) ff_before[c + 1] = ff_before[c] + chunk_ff_count(words.data(), byte_count, c);
	*out_size = kHeaderBytes + byte_count + ff_before[chunks] + kTrailerBytes;
	if (*out_size > capacity) return 1;
	write_header(quality, width, height, out_file);
	for (uint64_t c = 0; c != chunks; ++c) stuff_chunk(words.data(), byte_count, c, ff_before[c], out_file + kHeaderBytes);
	out_file[*out_size - 2] = 0xFF;
	out_file[*out_size - 1] = 0xD9;
	return 0;
}

// the quantised coefficients of every block in stream order (block_count * 64 int16, zigzag order); returns the block count
extern "C" uint64_t vkr_host_jpg_coefficients(const uint8_t* rgb8, uint32_t width, uint32_t height, int quality, int16_t* out) {
	Params p;
	make_params(quality, width, height, &p);
	if (out)
		for (uint64_t b = 0; b != p.block_count; ++b) transform_block(p, rgb8, b, out + 64 * b);
	return p.block_count;
}
