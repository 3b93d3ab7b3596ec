// vkr_accumulate.cu -- averaging frames on the device and measuring a frame's error against a reference (include/vkr_b200.h, vkr_accumulator_t,
// vkr_compare_frames). No counterpart in the reference, which renders one frame at a time; these kernels turn its experiment list into a
// measurement of noise and bias. The arithmetic and the order of every addition live in vkr_accumulate.cuh, which the CPU tests compile too.
// Separate launches after the frame; the shading kernels are untouched.
#include "../../include/vkr_b200.h"
#include "vkr_accumulate.cuh"
#include <cuda_runtime.h>
#include <cstdio>
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

// one block: slot k of the total = the block partials in index order
__global__ void total_kernel(double* partials) {
	const int k = threadIdx.x;
	if (k < kSlots) partials[(size_t) kReduceBlocks * kSlots + k] = total_slot(partials, k);
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
