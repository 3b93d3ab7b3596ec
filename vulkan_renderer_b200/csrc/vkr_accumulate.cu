// vkr_accumulate.cu -- averaging frames on the device and measuring a frame's error against a reference (include/vkr_b200.h, vkr_accumulator_t,
// vkr_compare_frames). No counterpart in the reference, which renders one frame at a time; these kernels turn its experiment list into a
// measurement of noise and bias. The arithmetic and the order of every addition live in vkr_accumulate.cuh, which the CPU tests compile too.
// Separate launches after the frame; the shading kernels are untouched.
#include "../../include/vkr_b200.h"
#include "vkr_accumulate.cuh"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#define VKR_CUDA_OK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { printf("%s: %s\n", what, cudaGetErrorString(e_)); return 1; } } while (0)

using namespace vkr_acc;

namespace {

constexpr int kThreads = 256;
// block partials [kReduceBlocks][kSlots], then the total [kSlots]
constexpr size_t kPartialBytes = sizeof(double) * kSlots * (kReduceBlocks + 1);

__global__ void __launch_bounds__(kThreads) accumulate_kernel(const float4* __restrict__ frame, double* __restrict__ state, uint64_t pixels, uint64_t n) {
	const uint64_t i = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (i >= pixels) return;
	const float4 x = frame[i];
	accumulate_pixel(state, pixels, i, x.x, x.y, x.z, n);
}

__global__ void __launch_bounds__(kThreads) resolve_kernel(const double* __restrict__ state, uint64_t pixels, uint64_t n, float* mean_rgba, float* variance_rgba) {
	const uint64_t i = (uint64_t) blockIdx.x * kThreads + threadIdx.x;
	if (i < pixels) resolve_pixel(state, pixels, i, n, mean_rgba, variance_rgba);
}

// one block per partition: per-thread sums, then the halving tree of vkr_accumulate.cuh; block partial -> partials[blockIdx.x]
__device__ void block_tree(double (*terms)[kSlots], double* partials) {
	const int t = threadIdx.x;
	__syncthreads();
	for (int s = kReduceThreads / 2; s > 0; s >>= 1) {
		if (t < s) combine_terms(terms[t], terms[t + s]);
		__syncthreads();
	}
	if (t < kSlots) partials[(size_t) blockIdx.x * kSlots + t] = terms[0][t];
}

__global__ void __launch_bounds__(kReduceThreads) error_partials_kernel(const float* __restrict__ frame, const float* __restrict__ reference, uint64_t pixels, double* partials) {
	__shared__ double terms[kReduceThreads][kSlots];
	thread_error_terms(terms[threadIdx.x], frame, reference, pixels, blockIdx.x, threadIdx.x);
	block_tree(terms, partials);
}

__global__ void __launch_bounds__(kReduceThreads) variance_partials_kernel(const double* __restrict__ state, uint64_t pixels, uint64_t n, double* partials) {
	__shared__ double terms[kReduceThreads][kSlots];
	thread_variance_terms(terms[threadIdx.x], state, pixels, n, blockIdx.x, threadIdx.x);
	block_tree(terms, partials);
}

__global__ void __launch_bounds__(kReduceThreads) estimate_partials_kernel(const double* __restrict__ state, const uint32_t* __restrict__ tile_frames, uint32_t width,
	uint64_t pixels, double* partials)
{
	__shared__ double terms[kReduceThreads][kSlots];
	thread_estimate_terms(terms[threadIdx.x], state, tile_frames, width, pixels, blockIdx.x, threadIdx.x);
	block_tree(terms, partials);
}

// one block: slot k of the total = the block partials in index order
__global__ void total_kernel(double* partials) {
	const int k = threadIdx.x;
	if (k < kSlots) partials[(size_t) kReduceBlocks * kSlots + k] = total_slot(partials, k);
}

// ---- adaptive accumulation: one CTA per 16x8 tile, thread k on pixel k of the tile (vkr_accumulate.cuh). A warp covers two 16-pixel rows, so each
// plane is read and written in 128-byte runs; the grid is the tile count, independent of the SM count.
static_assert(kTileWidth == VKR_TILE_WIDTH && kTileHeight == VKR_TILE_ROW_HEIGHT, "the adaptive accumulator's tiles are the shading pass's tiles");

__global__ void __launch_bounds__(kTilePixels) adaptive_accumulate_kernel(const float4* __restrict__ frame, double* __restrict__ state, uint32_t* tile_frames,
	const uint8_t* __restrict__ active, uint32_t width, uint32_t height)
{
	const uint32_t tile = blockIdx.x;
	if (!active[tile]) return;
	const uint32_t n = tile_frames[tile];
	uint64_t i;
	if (tile_pixel(width, height, tile, threadIdx.x, &i)) {
		const float4 x = frame[i];
		accumulate_pixel(state, (uint64_t) width * height, i, x.x, x.y, x.z, (uint64_t) n + 1);
	}
	__syncthreads();   // every thread has read n
	if (threadIdx.x == 0) tile_frames[tile] = n + 1;
}

__global__ void __launch_bounds__(kTilePixels) adaptive_tile_test_kernel(const double* __restrict__ state, const uint32_t* __restrict__ tile_frames, uint8_t* active,
	uint32_t width, uint32_t height, double target, uint32_t min_frames, uint32_t max_frames)
{
	const uint32_t tile = blockIdx.x;
	if (!active[tile]) return;
	const uint32_t n = tile_frames[tile];
	bool converged = false;
	if (tile_needs_test(n, min_frames, max_frames)) {   // the same for the whole CTA
		uint64_t i;
		const bool pass = !tile_pixel(width, height, tile, threadIdx.x, &i) || pixel_converged(state, (uint64_t) width * height, i, n, target);
		converged = __syncthreads_and(pass) != 0;
	}
	if (threadIdx.x == 0) active[tile] = tile_stays_active(n, converged, min_frames, max_frames) ? 1 : 0;
}

__global__ void __launch_bounds__(kTilePixels) adaptive_resolve_kernel(const double* __restrict__ state, const uint32_t* __restrict__ tile_frames, uint32_t width, uint32_t height,
	float* mean_rgba, float* variance_rgba)
{
	uint64_t i;
	if (tile_pixel(width, height, blockIdx.x, threadIdx.x, &i)) resolve_pixel(state, (uint64_t) width * height, i, tile_frames[blockIdx.x], mean_rgba, variance_rgba);
}

unsigned grid_of(uint64_t pixels) { return (unsigned) ((pixels + kThreads - 1) / kThreads); }

// enqueues a reduction whose block kernel has been launched already, then the final sum, and copies the total to host memory
int finish_reduction(double* d_partials, double* h_total, cudaStream_t stream) {
	total_kernel<<<1, 32, 0, stream>>>(d_partials);
	VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the reduction");
	VKR_CUDA_OK(cudaMemcpyAsync(h_total, d_partials + (size_t) kReduceBlocks * kSlots, sizeof(double) * kSlots, cudaMemcpyDeviceToHost, stream), "Failed to copy the reduction to the host");
	VKR_CUDA_OK(cudaStreamSynchronize(stream), "Failed to wait for the reduction");
	return 0;
}

} // namespace

extern "C" void vkr_destroy_accumulator(vkr_accumulator_t* acc, const vkr_device_t* device) {
	if (device && device->stream && (acc->d_state || acc->d_partials)) { cudaSetDevice(device->cuda_device); cudaStreamSynchronize((cudaStream_t) device->stream); }
	if (acc->d_state) cudaFree(acc->d_state);
	if (acc->d_partials) cudaFree(acc->d_partials);
	if (acc->h_partials) cudaFreeHost(acc->h_partials);
	memset(acc, 0, sizeof(*acc));
}

extern "C" int vkr_create_accumulator(vkr_accumulator_t* acc, const vkr_device_t* device, uint32_t width, uint32_t height) {
	memset(acc, 0, sizeof(*acc));
	if (!width || !height) { printf("Failed to create an accumulator: the resolution is %ux%u.\n", width, height); return 1; }
	const size_t state_bytes = sizeof(double) * kStatePlanes * (size_t) width * height;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess || cudaMalloc(&acc->d_state, state_bytes) != cudaSuccess || cudaMalloc(&acc->d_partials, kPartialBytes) != cudaSuccess
		|| cudaHostAlloc(&acc->h_partials, sizeof(double) * kSlots, cudaHostAllocDefault) != cudaSuccess)
	{
		printf("Failed to create an accumulator of resolution %ux%u: could not allocate %llu bytes on CUDA device %d.\n", width, height, (unsigned long long) (state_bytes + kPartialBytes), device->cuda_device);
		vkr_destroy_accumulator(acc, nullptr);
		return 1;
	}
	acc->width = width; acc->height = height;
	return 0;
}

extern "C" int vkr_accumulator_reset(vkr_accumulator_t* acc, const vkr_device_t* device) {
	(void) device;   // the first frame after a reset overwrites the state, no clearing needed
	if (!acc->d_state) { printf("The accumulator has not been created.\n"); return 1; }
	acc->frame_count = 0;
	return 0;
}

extern "C" int vkr_accumulate_frame(vkr_accumulator_t* acc, const vkr_device_t* device, const void* d_frame_rgba32f) {
	if (!acc->d_state || !d_frame_rgba32f || ((uintptr_t) d_frame_rgba32f & 15)) { printf("Failed to accumulate a frame: no accumulator, or the frame is NULL or not 16-byte aligned.\n"); return 1; }
	const uint64_t pixels = (uint64_t) acc->width * acc->height;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	accumulate_kernel<<<grid_of(pixels), kThreads, 0, (cudaStream_t) device->stream>>>((const float4*) d_frame_rgba32f, (double*) acc->d_state, pixels, acc->frame_count + 1);
	VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the accumulation");
	++acc->frame_count;
	return 0;
}

extern "C" int vkr_accumulator_resolve(const vkr_accumulator_t* acc, const vkr_device_t* device, void* d_mean_rgba32f, void* d_variance_rgba32f) {
	if (!acc->d_state || acc->frame_count == 0) { printf("Failed to resolve the accumulator: no frame has been accumulated.\n"); return 1; }
	if (d_variance_rgba32f && acc->frame_count < 2) { printf("Failed to resolve the accumulator: a variance needs at least 2 frames, there is %llu.\n", (unsigned long long) acc->frame_count); return 1; }
	if (!d_mean_rgba32f && !d_variance_rgba32f) return 0;
	const uint64_t pixels = (uint64_t) acc->width * acc->height;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	resolve_kernel<<<grid_of(pixels), kThreads, 0, (cudaStream_t) device->stream>>>((const double*) acc->d_state, pixels, acc->frame_count, (float*) d_mean_rgba32f, (float*) d_variance_rgba32f);
	VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the resolve of the accumulator");
	return 0;
}

extern "C" int vkr_accumulator_mean_variance(const vkr_accumulator_t* acc, const vkr_device_t* device, double out_mean_variance[3]) {
	if (!acc->d_state || acc->frame_count < 2) { printf("Failed to compute the mean variance: it needs at least 2 accumulated frames, there are %llu.\n", (unsigned long long) acc->frame_count); return 1; }
	const uint64_t pixels = (uint64_t) acc->width * acc->height;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	variance_partials_kernel<<<kReduceBlocks, kReduceThreads, 0, stream>>>((const double*) acc->d_state, pixels, acc->frame_count, (double*) acc->d_partials);
	if (finish_reduction((double*) acc->d_partials, (double*) acc->h_partials, stream)) return 1;
	finish_mean_variance((const double*) acc->h_partials, out_mean_variance);
	return 0;
}

extern "C" int vkr_compare_frames(const vkr_device_t* device, uint32_t width, uint32_t height, const void* d_frame_rgba32f, const void* d_reference_rgba32f, vkr_frame_error_t* out) {
	if (!width || !height || !d_frame_rgba32f || !d_reference_rgba32f || !out) { printf("Failed to compare frames: %ux%u pixels, frame %p, reference %p.\n", width, height, d_frame_rgba32f, d_reference_rgba32f); return 1; }
	const uint64_t pixels = (uint64_t) width * height;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	double* d_partials = nullptr;
	double total[kSlots];
	VKR_CUDA_OK(cudaMallocAsync((void**) &d_partials, kPartialBytes, stream), "Failed to allocate the reduction scratch");
	error_partials_kernel<<<kReduceBlocks, kReduceThreads, 0, stream>>>((const float*) d_frame_rgba32f, (const float*) d_reference_rgba32f, pixels, d_partials);
	const int rc = finish_reduction(d_partials, total, stream);
	cudaFreeAsync(d_partials, stream);
	if (rc) return 1;
	finish_error(total, out->mse, out->rel_mse, out->mae, &out->max_abs_error, &out->pixel_count, &out->nonfinite_pixels);
	return 0;
}

// ---- adaptive accumulator
extern "C" void vkr_destroy_adaptive_accumulator(vkr_adaptive_accumulator_t* acc, const vkr_device_t* device) {
	if (device && device->stream && acc->d_state) { cudaSetDevice(device->cuda_device); cudaStreamSynchronize((cudaStream_t) device->stream); }
	if (acc->d_state) cudaFree(acc->d_state);
	if (acc->d_tile_frames) cudaFree(acc->d_tile_frames);
	if (acc->d_tile_active) cudaFree(acc->d_tile_active);
	if (acc->d_partials) cudaFree(acc->d_partials);
	if (acc->h_partials) cudaFreeHost(acc->h_partials);
	memset(acc, 0, sizeof(*acc));
}

extern "C" int vkr_adaptive_accumulator_reset(vkr_adaptive_accumulator_t* acc, const vkr_device_t* device) {
	if (!acc->d_state) { printf("The adaptive accumulator has not been created.\n"); return 1; }
	const size_t tiles = (size_t) acc->tiles_x * acc->tiles_y;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	VKR_CUDA_OK(cudaMemsetAsync(acc->d_tile_frames, 0, sizeof(uint32_t) * tiles, stream), "Failed to clear the tile frame counts");
	VKR_CUDA_OK(cudaMemsetAsync(acc->d_tile_active, 1, tiles, stream), "Failed to activate the tiles");
	acc->frame_count = 0;
	acc->active_tile_count = (uint32_t) tiles;
	return 0;
}

extern "C" int vkr_create_adaptive_accumulator(vkr_adaptive_accumulator_t* acc, const vkr_device_t* device, uint32_t width, uint32_t height) {
	memset(acc, 0, sizeof(*acc));
	if (!width || !height) { printf("Failed to create an adaptive accumulator: the resolution is %ux%u.\n", width, height); return 1; }
	const size_t state_bytes = sizeof(double) * kStatePlanes * (size_t) width * height, tiles = (size_t) tiles_across(width) * tiles_down(height);
	if (cudaSetDevice(device->cuda_device) != cudaSuccess || cudaMalloc(&acc->d_state, state_bytes) != cudaSuccess || cudaMalloc(&acc->d_tile_frames, sizeof(uint32_t) * tiles) != cudaSuccess
		|| cudaMalloc(&acc->d_tile_active, tiles) != cudaSuccess || cudaMalloc(&acc->d_partials, kPartialBytes) != cudaSuccess
		|| cudaHostAlloc(&acc->h_partials, sizeof(double) * kSlots, cudaHostAllocDefault) != cudaSuccess)
	{
		printf("Failed to create an adaptive accumulator of resolution %ux%u: could not allocate %llu bytes on CUDA device %d.\n", width, height,
			(unsigned long long) (state_bytes + 5 * tiles + kPartialBytes), device->cuda_device);
		vkr_destroy_adaptive_accumulator(acc, nullptr);
		return 1;
	}
	acc->width = width; acc->height = height; acc->tiles_x = tiles_across(width); acc->tiles_y = tiles_down(height);
	if (vkr_adaptive_accumulator_reset(acc, device)) { vkr_destroy_adaptive_accumulator(acc, device); return 1; }
	return 0;
}

extern "C" int vkr_adaptive_accumulate_frame(vkr_adaptive_accumulator_t* acc, const vkr_device_t* device, const void* d_frame_rgba32f) {
	if (!acc->d_state || !d_frame_rgba32f || ((uintptr_t) d_frame_rgba32f & 15)) { printf("Failed to accumulate a frame: no adaptive accumulator, or the frame is NULL or not 16-byte aligned.\n"); return 1; }
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	adaptive_accumulate_kernel<<<acc->tiles_x * acc->tiles_y, kTilePixels, 0, (cudaStream_t) device->stream>>>((const float4*) d_frame_rgba32f, (double*) acc->d_state,
		(uint32_t*) acc->d_tile_frames, (const uint8_t*) acc->d_tile_active, acc->width, acc->height);
	VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the adaptive accumulation");
	++acc->frame_count;
	return 0;
}

extern "C" int vkr_adaptive_update_tiles(vkr_adaptive_accumulator_t* acc, const vkr_device_t* device, double target_rel_mse, uint32_t min_frames, uint32_t max_frames,
	uint8_t* out_active, uint32_t* out_active_count)
{
	if (!acc->d_state) { printf("The adaptive accumulator has not been created.\n"); return 1; }
	if (!(target_rel_mse >= 0.0) || !finite_value(target_rel_mse)) { printf("Failed to update the tiles: the target relMSE %g is negative or not finite.\n", target_rel_mse); return 1; }
	if (min_frames < 2 || max_frames < min_frames) { printf("Failed to update the tiles: min_frames = %u must be at least 2 and max_frames = %u at least min_frames.\n", min_frames, max_frames); return 1; }
	const uint32_t tiles = acc->tiles_x * acc->tiles_y;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	adaptive_tile_test_kernel<<<tiles, kTilePixels, 0, stream>>>((const double*) acc->d_state, (const uint32_t*) acc->d_tile_frames, (uint8_t*) acc->d_tile_active,
		acc->width, acc->height, target_rel_mse, min_frames, max_frames);
	VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the tile test");
	uint8_t* flags = out_active;
	if (!flags && !(flags = (uint8_t*) malloc(tiles))) { printf("Failed to allocate %u tile flags.\n", tiles); return 1; }
	cudaError_t err = cudaMemcpyAsync(flags, acc->d_tile_active, tiles, cudaMemcpyDeviceToHost, stream);
	if (err == cudaSuccess) err = cudaStreamSynchronize(stream);
	uint32_t active = 0;
	for (uint32_t t = 0; t != tiles; ++t) active += flags[t] != 0;
	if (flags != out_active) free(flags);
	VKR_CUDA_OK(err, "Failed to read back the tile flags");
	acc->active_tile_count = active;
	if (out_active_count) *out_active_count = active;
	return 0;
}

extern "C" int vkr_adaptive_tile_frames(const vkr_adaptive_accumulator_t* acc, const vkr_device_t* device, uint32_t* out_tile_frames) {
	if (!acc->d_state || !out_tile_frames) { printf("Failed to read the tile frame counts: no adaptive accumulator or no output.\n"); return 1; }
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	VKR_CUDA_OK(cudaMemcpyAsync(out_tile_frames, acc->d_tile_frames, sizeof(uint32_t) * acc->tiles_x * acc->tiles_y, cudaMemcpyDeviceToHost, stream), "Failed to copy the tile frame counts");
	VKR_CUDA_OK(cudaStreamSynchronize(stream), "Failed to wait for the tile frame counts");
	return 0;
}

// every tile has at least min(frame_count, 2) frames: a tile stops only with n_t >= min_frames >= 2, and an active one has taken every frame
extern "C" int vkr_adaptive_resolve(const vkr_adaptive_accumulator_t* acc, const vkr_device_t* device, void* d_mean_rgba32f, void* d_variance_rgba32f) {
	if (!acc->d_state || acc->frame_count == 0) { printf("Failed to resolve the adaptive accumulator: no frame has been accumulated.\n"); return 1; }
	if (d_variance_rgba32f && acc->frame_count < 2) { printf("Failed to resolve the adaptive accumulator: a variance needs at least 2 frames, there is %llu.\n", (unsigned long long) acc->frame_count); return 1; }
	if (!d_mean_rgba32f && !d_variance_rgba32f) return 0;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	adaptive_resolve_kernel<<<acc->tiles_x * acc->tiles_y, kTilePixels, 0, (cudaStream_t) device->stream>>>((const double*) acc->d_state, (const uint32_t*) acc->d_tile_frames,
		acc->width, acc->height, (float*) d_mean_rgba32f, (float*) d_variance_rgba32f);
	VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the resolve of the adaptive accumulator");
	return 0;
}

extern "C" int vkr_adaptive_estimated_rel_mse(const vkr_adaptive_accumulator_t* acc, const vkr_device_t* device, double out_rel_mse[3]) {
	if (!acc->d_state || acc->frame_count < 2) { printf("Failed to estimate the relMSE: it needs at least 2 accumulated frames, there are %llu.\n", (unsigned long long) acc->frame_count); return 1; }
	const uint64_t pixels = (uint64_t) acc->width * acc->height;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	estimate_partials_kernel<<<kReduceBlocks, kReduceThreads, 0, stream>>>((const double*) acc->d_state, (const uint32_t*) acc->d_tile_frames, acc->width, pixels, (double*) acc->d_partials);
	if (finish_reduction((double*) acc->d_partials, (double*) acc->h_partials, stream)) return 1;
	finish_mean_variance((const double*) acc->h_partials, out_rel_mse);   // slot c over the pixel count
	return 0;
}
