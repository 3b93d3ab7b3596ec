// vkr_raster.cu -- the rasterised visibility buffer (include/vkr_b200.h, vkr_rasterizer_t, vkr_rasterize_visibility): subpass 0 of the reference
// (src/main.c:1421-1427) with the rules of vkr_raster.cuh. All work runs on device->stream:
//   1. the depth-test keys (depth bits << 32 | primitive, 8 B per pixel) are cleared to all ones;
//   2. raster_setup_kernel, one thread per triangle: vertex stage, trivial reject, clipping, snapping, culling; a polygon whose pixel bounding box
//      has at most kSmallPixels pixels is rasterised right there (atomicMin on the keys), a larger one records how many 32x32 chunks its box has;
//   3. an inclusive scan of the chunk counts (cub::DeviceScan) numbers the chunks of all large polygons;
//   4. raster_large_kernel: as many persistent CTAs as fit on the device at once, each taking a contiguous range of chunks; thread 0 finds a
//      chunk's primitive (binary search) and sets it up when the range enters a new one, the CTA's threads test the chunk's pixels;
//   5. raster_resolve_kernel: keys -> primitive indices (0xFFFFFFFF where nothing was drawn) and, if asked for, depth (1.0 there).
// atomicMin on keys whose high word is a non-negative float makes the result independent of the order in which threads run. Compile with -fmad=false.
#include "../../include/vkr_b200.h"
#include "vkr_raster.cuh"
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

using namespace vkr;

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 32;             // side of a chunk of a large polygon's bounding box, in pixels
constexpr int kSmallPixels = 64;       // polygons with at most this many pixels in their box are rasterised by the setup thread

struct raster_params {
	const uint2* quantized_positions;
	const unsigned char* constants;
	uint32_t triangle_count;
	int width, height;
	unsigned long long* keys;
	unsigned long long* chunks;            // per triangle: chunks of its box if it is large, else 0
	const unsigned long long* chunk_ends;  // inclusive scan of chunks
};

__device__ __forceinline__ void depth_test(unsigned long long* keys, size_t pixel, unsigned long long key) {
	if (key != kRasterClearKey) atomicMin(keys + pixel, key);
}

__global__ void __launch_bounds__(kThreads) raster_setup_kernel(const __grid_constant__ raster_params p) {
	const uint32_t prim = blockIdx.x * kThreads + threadIdx.x;
	if (prim >= p.triangle_count) return;
	raster_polygon poly;
	raster_polygon_of(p.quantized_positions, p.constants, prim, p.width, p.height, poly);
	raster_triangle tris[kRasterMaxFan];
	int box[4];
	const int fans = raster_fans_of(poly, p.width, p.height, tris, box);
	unsigned long long chunks = 0;
	if (fans) {
		const int bw = box[2] - box[0] + 1, bh = box[3] - box[1] + 1;
		if ((long long) bw * bh <= kSmallPixels) {
			for (int y = box[1]; y <= box[3]; ++y)
				for (int x = box[0]; x <= box[2]; ++x) depth_test(p.keys, (size_t) y * p.width + x, raster_polygon_fragment(tris, fans, x, y, prim));
		}
		else chunks = (unsigned long long) ((bw + kChunk - 1) / kChunk) * ((bh + kChunk - 1) / kChunk);
	}
	p.chunks[prim] = chunks;
}

// CTA b takes the contiguous chunk range [b total / grid, (b + 1) total / grid), so consecutive chunks mostly belong to the same triangle and
// thread 0 sets a triangle up once per CTA rather than once per chunk
__global__ void __launch_bounds__(kThreads) raster_large_kernel(const __grid_constant__ raster_params p) {
	__shared__ raster_triangle tris[kRasterMaxFan];
	__shared__ int fans, box[4];
	__shared__ uint32_t prim;
	__shared__ unsigned long long prim_first, prim_end;   // chunks of the set-up triangle: [prim_first, prim_end)
	const unsigned long long total = p.chunk_ends[p.triangle_count - 1];
	const unsigned long long begin = total * blockIdx.x / gridDim.x, end = total * (blockIdx.x + 1) / gridDim.x;
	if (threadIdx.x == 0) { prim_first = 0; prim_end = 0; }
	__syncthreads();
	for (unsigned long long c = begin; c < end; ++c) {
		if (threadIdx.x == 0 && c >= prim_end) {
			uint32_t lo = 0, hi = p.triangle_count - 1;   // the first triangle whose chunks end after c
			while (lo < hi) {
				const uint32_t mid = lo + (hi - lo) / 2;
				if (p.chunk_ends[mid] > c) hi = mid; else lo = mid + 1;
			}
			raster_polygon poly;
			raster_polygon_of(p.quantized_positions, p.constants, lo, p.width, p.height, poly);
			fans = raster_fans_of(poly, p.width, p.height, tris, box);
			prim = lo;
			prim_end = p.chunk_ends[lo];
			prim_first = prim_end - p.chunks[lo];
		}
		__syncthreads();
		const unsigned long long chunk = c - prim_first;
		const int chunks_x = (box[2] - box[0] + kChunk) / kChunk;
		const int cx = box[0] + (int) (chunk % chunks_x) * kChunk, cy = box[1] + (int) (chunk / chunks_x) * kChunk;
		for (int j = threadIdx.x; j < kChunk * kChunk; j += kThreads) {
			const int x = cx + j % kChunk, y = cy + j / kChunk;
			if (x <= box[2] && y <= box[3]) depth_test(p.keys, (size_t) y * p.width + x, raster_polygon_fragment(tris, fans, x, y, prim));
		}
		__syncthreads();
	}
}

__global__ void __launch_bounds__(kThreads) raster_resolve_kernel(const unsigned long long* __restrict__ keys, size_t pixels, uint32_t* __restrict__ visibility, float* __restrict__ depth) {
	const size_t i = (size_t) blockIdx.x * kThreads + threadIdx.x;
	if (i >= pixels) return;
	const unsigned long long key = keys[i];
	const bool drawn = key != kRasterClearKey;
	visibility[i] = drawn ? (uint32_t) key : 0xFFFFFFFFu;
	if (depth) depth[i] = drawn ? __uint_as_float((uint32_t) (key >> 32)) : 1.0f;
}

unsigned blocks_for(size_t n) { return (unsigned) ((n + kThreads - 1) / kThreads); }

// scratch layout: chunk counts and their scan, 8 B per triangle each, then cub's temporary storage
size_t scan_temp_bytes(uint64_t capacity) {
	size_t bytes = 0;
	if (cub::DeviceScan::InclusiveSum(nullptr, bytes, (const unsigned long long*) nullptr, (unsigned long long*) nullptr, (int64_t) capacity) != cudaSuccess) return 0;
	return bytes;
}

} // namespace

#define VKR_RASTER_OK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { printf("%s: %s\n", what, cudaGetErrorString(e_)); return 1; } } while (0)

extern "C" void vkr_destroy_rasterizer(vkr_rasterizer_t* r, const vkr_device_t* device) {
	if (!r) return;
	if (device && device->stream && (r->d_keys || r->d_scratch)) { cudaSetDevice(device->cuda_device); cudaStreamSynchronize((cudaStream_t) device->stream); }
	if (r->d_keys) cudaFree(r->d_keys);
	if (r->d_scratch) cudaFree(r->d_scratch);
	if (r->d_constants) cudaFree(r->d_constants);
	memset(r, 0, sizeof(*r));
}

extern "C" int vkr_create_rasterizer(vkr_rasterizer_t* r, const vkr_device_t* device, uint32_t width, uint32_t height, uint64_t triangle_capacity) {
	if (!r) { printf("Failed to create a rasterizer: the rasterizer is NULL.\n"); return 1; }
	memset(r, 0, sizeof(*r));
	if (!device) { printf("Failed to create a rasterizer: the device is NULL.\n"); return 1; }
	if (!width || !height || width > kRasterMaxDimension || height > kRasterMaxDimension) {
		printf("Failed to create a rasterizer: the resolution %ux%u is not within 1..%u per side.\n", width, height, kRasterMaxDimension);
		return 1;
	}
	if (!triangle_capacity || triangle_capacity >= 0xFFFFFFFFull) {
		printf("Failed to create a rasterizer: the triangle capacity %llu is not within 1..%u.\n", (unsigned long long) triangle_capacity, 0xFFFFFFFEu);
		return 1;
	}
	const size_t key_bytes = sizeof(unsigned long long) * (size_t) width * height;
	const size_t temp_bytes = scan_temp_bytes(triangle_capacity);
	const size_t scratch_bytes = 2 * sizeof(unsigned long long) * (size_t) triangle_capacity + temp_bytes;
	int sm_count = 0, ctas_per_sm = 0;
	if (!temp_bytes || cudaSetDevice(device->cuda_device) != cudaSuccess || cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device->cuda_device) != cudaSuccess
		|| cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, raster_large_kernel, kThreads, 0) != cudaSuccess
		|| cudaMalloc(&r->d_keys, key_bytes) != cudaSuccess || cudaMalloc(&r->d_scratch, scratch_bytes) != cudaSuccess || cudaMalloc(&r->d_constants, 256) != cudaSuccess)
	{
		printf("Failed to create a rasterizer of resolution %ux%u for %llu triangles: could not allocate %llu bytes on CUDA device %d.\n", width, height,
			(unsigned long long) triangle_capacity, (unsigned long long) (key_bytes + scratch_bytes + 256), device->cuda_device);
		vkr_destroy_rasterizer(r, nullptr);
		return 1;
	}
	r->width = width; r->height = height; r->triangle_capacity = triangle_capacity;
	r->scratch_bytes = scratch_bytes; r->scan_temp_bytes = temp_bytes; r->large_ctas = (uint32_t) (sm_count * (ctas_per_sm > 0 ? ctas_per_sm : 1));
	return 0;
}

extern "C" int vkr_rasterize_visibility(vkr_rasterizer_t* r, const vkr_device_t* device, const vkr_scene_t* scene, const void* constants, void* d_visibility, void* d_depth) {
	if (!r || !device || !scene || !constants || !d_visibility) { printf("Failed to rasterize the visibility buffer: the rasterizer, device, scene, constants or visibility buffer is NULL.\n"); return 1; }
	if (!r->d_keys || !r->width || !r->height) { printf("Failed to rasterize the visibility buffer: the rasterizer has not been created.\n"); return 1; }
	if (scene->triangle_count > r->triangle_capacity) {
		printf("Failed to rasterize the visibility buffer: the scene has %llu triangles, the rasterizer was created for %llu.\n", (unsigned long long) scene->triangle_count,
			(unsigned long long) r->triangle_capacity);
		return 1;
	}
	if (scene->triangle_count && !scene->d_quantized_positions) { printf("Failed to rasterize the visibility buffer: the scene has no positions on the device.\n"); return 1; }
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_RASTER_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	const size_t pixels = (size_t) r->width * r->height;
	const uint32_t n = (uint32_t) scene->triangle_count;
	unsigned long long* chunks = (unsigned long long*) r->d_scratch;
	unsigned long long* chunk_ends = chunks + r->triangle_capacity;
	void* temp = chunk_ends + r->triangle_capacity;
	raster_params p;
	p.quantized_positions = (const uint2*) scene->d_quantized_positions; p.constants = (const unsigned char*) r->d_constants;
	p.triangle_count = n; p.width = (int) r->width; p.height = (int) r->height;
	p.keys = (unsigned long long*) r->d_keys; p.chunks = chunks; p.chunk_ends = chunk_ends;
	VKR_RASTER_OK(cudaMemcpyAsync(r->d_constants, constants, 256, cudaMemcpyHostToDevice, stream), "Failed to upload the constants of the rasterizer");
	VKR_RASTER_OK(cudaMemsetAsync(r->d_keys, 0xFF, sizeof(unsigned long long) * pixels, stream), "Failed to clear the depth-test keys");
	if (n) {
		raster_setup_kernel<<<blocks_for(n), kThreads, 0, stream>>>(p);
		VKR_RASTER_OK(cudaGetLastError(), "Failed to launch the triangle setup of the rasterizer");
		size_t temp_bytes = r->scan_temp_bytes;
		VKR_RASTER_OK(cub::DeviceScan::InclusiveSum(temp, temp_bytes, chunks, chunk_ends, (int64_t) n, stream), "Failed to scan the chunks of the large triangles");
		raster_large_kernel<<<r->large_ctas, kThreads, 0, stream>>>(p);
		VKR_RASTER_OK(cudaGetLastError(), "Failed to launch the large-triangle kernel of the rasterizer");
	}
	raster_resolve_kernel<<<blocks_for(pixels), kThreads, 0, stream>>>(p.keys, pixels, (uint32_t*) d_visibility, (float*) d_depth);
	VKR_RASTER_OK(cudaGetLastError(), "Failed to launch the resolve of the rasterizer");
	return 0;
}
