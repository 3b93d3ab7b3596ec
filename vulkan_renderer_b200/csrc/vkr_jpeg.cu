// vkr_jpeg.cu -- JPEG files of 8-bit RGB images encoded on the device (include/vkr_b200.h, vkr_encode_jpg, vkr_write_jpg, vkr_quantize_unorm8_device),
// byte-identical to stbi_write_jpg, the writer of the reference's *.jpg screenshots (src/main.c:1745-1751). The arithmetic and the bit layout live in
// vkr_jpeg.cuh, which tests/jpeg_on_host.cpp compiles for the CPU. All work runs on device->stream:
//   1. transform_kernel: one thread per 8x8 block in stream order -> 64 quantised coefficients (int16, zigzag order).
//   2. bits_kernel: each block's Huffman bit count, from its coefficients and its predecessor's DC.
//   3. exclusive scan of the counts (cub::DeviceScan) -> bit offsets; the total comes back to size the stream (one synchronisation).
//   4. emit_kernel: each block writes its bits at its offset into zeroed 32-bit words; the last block pads to a byte boundary with 1-bits.
//   5. ff_count_kernel, a scan of the counts, then stuff_kernel: 64-byte chunks of the stream, a 0x00 after each 0xFF (second synchronisation: the size).
//   6. the entropy-coded segment comes back into the caller's buffer between the header (written on the host) and EOI.
#include "../../include/vkr_b200.h"
#include "vkr_internal.h"
#include "vkr_jpeg.cuh"
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdio.h>
#include <vector>

using namespace vkr_jpeg;

namespace {

constexpr uint32_t kThreads = 128;

unsigned grid_for(uint64_t n) { return (unsigned) ((n + kThreads - 1) / kThreads); }

__global__ void __launch_bounds__(kThreads) jpeg_transform_kernel(const __grid_constant__ Params p, const uint8_t* __restrict__ rgb, int16_t* __restrict__ coefficients) {
	const uint64_t b = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (b < p.block_count) transform_block(p, rgb, b, coefficients + 64 * b);
}

// counts[block_count] stays 0 (memset), so the exclusive scan's last entry is the total
__global__ void __launch_bounds__(kThreads) jpeg_bits_kernel(const __grid_constant__ Params p, const int16_t* __restrict__ coefficients, uint64_t* __restrict__ counts) {
	const uint64_t b = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (b < p.block_count) counts[b] = block_bits(p, coefficients, b);
}

__global__ void __launch_bounds__(kThreads) jpeg_emit_kernel(const __grid_constant__ Params p, const int16_t* __restrict__ coefficients, const uint64_t* __restrict__ offsets,
	uint32_t* words)
{
	const uint64_t b = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (b < p.block_count) emit_block(p, coefficients, offsets, b, words);
}

__global__ void __launch_bounds__(kThreads) jpeg_ff_count_kernel(const uint32_t* __restrict__ words, uint64_t byte_count, uint64_t chunks, uint64_t* __restrict__ counts) {
	const uint64_t c = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (c < chunks) counts[c] = chunk_ff_count(words, byte_count, c);
}

__global__ void __launch_bounds__(kThreads) jpeg_stuff_kernel(const uint32_t* __restrict__ words, uint64_t byte_count, uint64_t chunks, const uint64_t* __restrict__ ff_before,
	uint8_t* __restrict__ out)
{
	const uint64_t c = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (c < chunks) stuff_chunk(words, byte_count, c, ff_before[c], out);
}

__global__ void __launch_bounds__(kThreads) jpeg_quantize_kernel(const float4* __restrict__ frame, uint64_t pixel_count, uint8_t* __restrict__ rgb) {
	const uint64_t i = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (i >= pixel_count) return;
	const float4 v = frame[i];
	rgb[3 * i + 0] = unorm8(v.x);
	rgb[3 * i + 1] = unorm8(v.y);
	rgb[3 * i + 2] = unorm8(v.z);
}

#define VKR_JPEG_TRY(call) do { if ((call) != cudaSuccess) { rc = 1; goto done; } } while (0)

// exclusive scan of count + 1 entries (the last one 0) in place of a separate total
int scan(uint64_t* in, uint64_t* out, uint64_t count, cudaStream_t stream) {
	size_t bytes = 0;
	void* temp = nullptr;
	int rc = 0;
	VKR_JPEG_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int64_t) count + 1, stream));
	VKR_JPEG_TRY(cudaMallocAsync(&temp, bytes, stream));
	VKR_JPEG_TRY(cub::DeviceScan::ExclusiveSum(temp, bytes, in, out, (int64_t) count + 1, stream));
done:
	if (temp) cudaFreeAsync(temp, stream);
	return rc;
}

// The file for d_rgb8 into out (capacity bytes) or, with grow, into *grow resized to fit. *out_size: the file's size whenever it could be computed.
int encode(const vkr_device_t* device, const uint8_t* d_rgb8, uint32_t width, uint32_t height, int quality, uint8_t* out, size_t capacity, size_t* out_size,
	std::vector<uint8_t>* grow)
{
	Params p;
	make_params(quality, width, height, &p);
	const uint64_t n = p.block_count;
	cudaStream_t stream = (cudaStream_t) device->stream;
	int16_t* coefficients = nullptr;
	uint64_t *counts = nullptr, *offsets = nullptr, *ff_counts = nullptr, *ff_before = nullptr;
	uint32_t* words = nullptr;
	uint8_t* stuffed = nullptr;
	uint64_t total_bits = 0, byte_count = 0, chunks = 0, ff_total = 0;
	size_t size = 0;
	int rc = 0;
	VKR_JPEG_TRY(cudaSetDevice(device->cuda_device));
	VKR_JPEG_TRY(cudaMallocAsync((void**) &coefficients, sizeof(int16_t) * 64 * n, stream));
	VKR_JPEG_TRY(cudaMallocAsync((void**) &counts, sizeof(uint64_t) * (n + 1), stream));
	VKR_JPEG_TRY(cudaMallocAsync((void**) &offsets, sizeof(uint64_t) * (n + 1), stream));
	VKR_JPEG_TRY(cudaMemsetAsync(counts + n, 0, sizeof(uint64_t), stream));
	jpeg_transform_kernel<<<grid_for(n), kThreads, 0, stream>>>(p, d_rgb8, coefficients);
	VKR_JPEG_TRY(cudaGetLastError());
	jpeg_bits_kernel<<<grid_for(n), kThreads, 0, stream>>>(p, coefficients, counts);
	VKR_JPEG_TRY(cudaGetLastError());
	if (scan(counts, offsets, n, stream)) { rc = 1; goto done; }
	VKR_JPEG_TRY(cudaMemcpyAsync(&total_bits, offsets + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
	VKR_JPEG_TRY(cudaStreamSynchronize(stream));
	byte_count = (total_bits + 7) / 8;
	chunks = (byte_count + kChunkBytes - 1) / kChunkBytes;
	VKR_JPEG_TRY(cudaMallocAsync((void**) &words, sizeof(uint32_t) * ((byte_count + 3) / 4), stream));
	VKR_JPEG_TRY(cudaMallocAsync((void**) &ff_counts, sizeof(uint64_t) * (chunks + 1), stream));
	VKR_JPEG_TRY(cudaMallocAsync((void**) &ff_before, sizeof(uint64_t) * (chunks + 1), stream));
	VKR_JPEG_TRY(cudaMemsetAsync(words, 0, sizeof(uint32_t) * ((byte_count + 3) / 4), stream));
	VKR_JPEG_TRY(cudaMemsetAsync(ff_counts + chunks, 0, sizeof(uint64_t), stream));
	jpeg_emit_kernel<<<grid_for(n), kThreads, 0, stream>>>(p, coefficients, offsets, words);
	VKR_JPEG_TRY(cudaGetLastError());
	jpeg_ff_count_kernel<<<grid_for(chunks), kThreads, 0, stream>>>(words, byte_count, chunks, ff_counts);
	VKR_JPEG_TRY(cudaGetLastError());
	if (scan(ff_counts, ff_before, chunks, stream)) { rc = 1; goto done; }
	VKR_JPEG_TRY(cudaMemcpyAsync(&ff_total, ff_before + chunks, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
	VKR_JPEG_TRY(cudaStreamSynchronize(stream));
	size = kHeaderBytes + byte_count + ff_total + kTrailerBytes;
	*out_size = size;
	if (grow) { grow->resize(size); out = grow->data(); capacity = size; }
	if (size > capacity) {
		printf("Failed to encode a %u x %u JPEG: the file takes %zu bytes, the buffer holds %zu.\n", width, height, size, capacity);
		rc = 2;
		goto done;
	}
	VKR_JPEG_TRY(cudaMallocAsync((void**) &stuffed, byte_count + ff_total, stream));
	jpeg_stuff_kernel<<<grid_for(chunks), kThreads, 0, stream>>>(words, byte_count, chunks, ff_before, stuffed);
	VKR_JPEG_TRY(cudaGetLastError());
	VKR_JPEG_TRY(cudaMemcpyAsync(out + kHeaderBytes, stuffed, byte_count + ff_total, cudaMemcpyDeviceToHost, stream));
	VKR_JPEG_TRY(cudaStreamSynchronize(stream));
	write_header(quality, width, height, out);
	out[size - 2] = 0xFF;
	out[size - 1] = 0xD9;
done:
	if (rc == 1) printf("Failed to encode a %u x %u JPEG on CUDA device %d: %s\n", width, height, device->cuda_device, cudaGetErrorString(cudaGetLastError()));
	for (void* ptr : { (void*) coefficients, (void*) counts, (void*) offsets, (void*) words, (void*) ff_counts, (void*) ff_before, (void*) stuffed })
		if (ptr) cudaFreeAsync(ptr, stream);
	if (cudaStreamSynchronize(stream) != cudaSuccess) rc = 1;   // nothing is left pending on the caller's buffer
	return rc ? 1 : 0;
}

int write_file(const char* path, const std::vector<uint8_t>& file, FILE* f) {
	bool ok = fwrite(file.data(), 1, file.size(), f) == file.size();
	ok = (fclose(f) == 0) && ok;
	if (!ok) { printf("Failed to write the *.jpg file at %s.\n", path); remove(path); return 1; }
	return 0;
}

} // namespace

namespace vkr {

int jpeg_quantize(const vkr_device_t* device, const float* d_rgba32f, uint32_t width, uint32_t height, uint8_t* d_rgb8) {
	const uint64_t pixel_count = (uint64_t) width * height;
	cudaStream_t stream = (cudaStream_t) device->stream;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess) return 1;
	if (pixel_count) jpeg_quantize_kernel<<<grid_for(pixel_count), kThreads, 0, stream>>>((const float4*) d_rgba32f, pixel_count, d_rgb8);
	if (cudaGetLastError() != cudaSuccess) { printf("Failed to quantise a frame on CUDA device %d.\n", device->cuda_device); return 1; }
	return 0;
}

int jpeg_write_device_image(const vkr_device_t* device, const char* path, const uint8_t* d_rgb8, uint32_t width, uint32_t height, int quality) {
	FILE* f = fopen(path, "wb");
	if (!f) { printf("Failed to store a screenshot to the *.jpg file at %s. Please check path and permissions.\n", path); return 1; }
	std::vector<uint8_t> file;
	size_t size = 0;
	if (encode(device, d_rgb8, width, height, quality, nullptr, 0, &size, &file)) { fclose(f); remove(path); return 1; }
	return write_file(path, file, f);
}

} // namespace vkr

extern "C" int vkr_quantize_unorm8_device(const vkr_device_t* device, const void* d_rgba32f, uint32_t width, uint32_t height, void* d_rgb8) {
	if (!device || !d_rgba32f || !d_rgb8) { printf("Failed to quantise a frame: no device, no frame or no output.\n"); return 1; }
	return vkr::jpeg_quantize(device, (const float*) d_rgba32f, width, height, (uint8_t*) d_rgb8);
}

extern "C" int vkr_encode_jpg(const vkr_device_t* device, const uint8_t* d_rgb8, uint32_t width, uint32_t height, int quality, uint8_t* out_file, size_t capacity, size_t* out_size) {
	if (check_request("encode a JPEG", d_rgb8, width, height, out_file, out_size)) return 1;
	if (!device) { printf("Failed to encode a JPEG: no device.\n"); return 1; }
	return encode(device, d_rgb8, width, height, quality, out_file, capacity, out_size, nullptr);
}

extern "C" int vkr_write_jpg(const vkr_device_t* device, const char* path, uint32_t width, uint32_t height, const uint8_t* rgb8, int quality) {
	size_t unused = 0;
	if (check_request("write a JPEG", rgb8, width, height, path, &unused)) return 1;
	if (!device) { printf("Failed to write a JPEG: no device.\n"); return 1; }
	FILE* f = fopen(path, "wb");
	if (!f) { printf("Failed to store an image to the *.jpg file at %s. Please check path and permissions.\n", path); return 1; }
	void* d_rgb8 = nullptr;
	std::vector<uint8_t> file;
	size_t size = 0;
	const int failed = vkr::upload(&d_rgb8, rgb8, 3 * (size_t) width * height, device) || encode(device, (const uint8_t*) d_rgb8, width, height, quality, nullptr, 0, &size, &file);
	if (d_rgb8) cudaFree(d_rgb8);
	if (failed) { fclose(f); remove(path); return 1; }
	return write_file(path, file, f);
}
