// vkr_ltc_fit.cu -- fitting the specular BRDF's LTC table on the device and writing it as fit<i>.dat files (include/vkr_b200.h, vkr_fit_ltc_table,
// vkr_write_ltc_fits). The reference reads these files from its data download (src/ltc_table.c:23-116) and has no fitter; the files written here
// load through the unchanged vkr_load_ltc_table. The arithmetic, the summation order and the minimiser live in vkr_ltc_fit.cuh, which the CPU
// tests compile too. One CTA per chain (Fresnel layer, inclination row); its threads share every objective evaluation's samples and all of them
// run the simplex logic on the same values.
#include "../../include/vkr_b200.h"
#include "vkr_ltc_fit.cuh"
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <string>
#include <vector>

#define VKR_CUDA_OK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { printf("%s: %s\n", what, cudaGetErrorString(e_)); return 1; } } while (0)

using namespace vkr_ltc;

namespace {

// the halving tree of vkr_ltc_fit.cuh in shared memory; every thread leaves with the totals
struct DeviceReducer {
	double (*partial)[kThreads];   // [kSlots][kThreads]
	__device__ void tree(int slots) {
		const int t = threadIdx.x;
		__syncthreads();
		for (int s = kThreads / 2; s > 0; s >>= 1) {
			if (t < s) for (int k = 0; k != slots; ++k) partial[k][t] = partial[k][t] + partial[k][t + s];
			__syncthreads();
		}
	}
	__device__ void moments(double* out, const Cell& cell, const Quadrature& q) {
		double terms[kSlots];
		thread_moment_terms(terms, cell, q, threadIdx.x);
		for (int k = 0; k != kSlots; ++k) partial[k][threadIdx.x] = terms[k];
		tree(kSlots);
		for (int k = 0; k != kSlots; ++k) out[k] = partial[k][0];
		__syncthreads();
	}
	__device__ double objective(const double* x, const Cell& cell, const Quadrature& q, double rcp_albedo) {
		partial[0][threadIdx.x] = thread_objective_term(x, cell, q, rcp_albedo, threadIdx.x);
		tree(1);
		const double total = partial[0][0];
		__syncthreads();
		return total;
	}
};

// block c fits chain c; tables: make_tables
__global__ void __launch_bounds__(kThreads, 1) fit_kernel(uint32_t resolution, uint32_t fresnel_count, uint32_t n, uint32_t iteration_limit, const double* __restrict__ tables,
	float* fits, double* errors, uint32_t* evaluations, uint32_t* limit_hits)
{
	__shared__ double partial[kSlots][kThreads];
	DeviceReducer reducer = { partial };
	const uint32_t chain = blockIdx.x;
	const Quadrature q = quadrature_of(tables, n);
	const double* cos_theta = cos_theta_of(tables, n);
	const bool leader = threadIdx.x == 0;   // every thread computes the same values; thread 0 stores them
	fit_chain(reducer, chain, resolution, fresnel_count, cos_theta, cos_theta + resolution, q, iteration_limit,
		leader ? fits + (uint64_t) chain * resolution * 5 : nullptr, leader ? errors + (uint64_t) chain * resolution : nullptr,
		leader ? evaluations + (uint64_t) chain * resolution : nullptr, leader ? limit_hits + chain : nullptr);
}

int check_desc(const vkr_ltc_fit_desc_t* desc) {
	if (!desc || desc->resolution < 2 || desc->resolution > VKR_LTC_FIT_MAX_RESOLUTION || desc->fresnel_count < 2 || desc->fresnel_count > VKR_LTC_FIT_MAX_FRESNEL_COUNT
		|| desc->quadrature_size < 2 || desc->quadrature_size > VKR_LTC_FIT_MAX_QUADRATURE_SIZE || desc->iteration_limit < 1 || desc->iteration_limit > VKR_LTC_FIT_MAX_ITERATION_LIMIT)
	{
		if (desc) printf("Failed to fit a linearly transformed cosine table: resolution %u (2..%u), Fresnel count %u (2..%u), quadrature size %u (2..%u), iteration limit %u (1..%u).\n",
			desc->resolution, VKR_LTC_FIT_MAX_RESOLUTION, desc->fresnel_count, VKR_LTC_FIT_MAX_FRESNEL_COUNT, desc->quadrature_size, VKR_LTC_FIT_MAX_QUADRATURE_SIZE,
			desc->iteration_limit, VKR_LTC_FIT_MAX_ITERATION_LIMIT);
		else printf("Failed to fit a linearly transformed cosine table: no descriptor.\n");
		return 1;
	}
	return 0;
}

} // namespace

extern "C" void vkr_ltc_fit_default_desc(vkr_ltc_fit_desc_t* desc) {
	desc->resolution = 64; desc->fresnel_count = 51; desc->quadrature_size = 32; desc->iteration_limit = 400;
}

extern "C" int vkr_fit_ltc_table(const vkr_device_t* device, const vkr_ltc_fit_desc_t* desc, float* out_fits, vkr_ltc_fit_stats_t* stats) {
	if (check_desc(desc)) return 1;
	if (!device || !out_fits) { printf("Failed to fit a linearly transformed cosine table: no device or no output array.\n"); return 1; }
	const uint32_t resolution = desc->resolution, n = desc->quadrature_size;
	const uint64_t chains = (uint64_t) desc->fresnel_count * resolution, cells = chains * resolution;
	std::vector<double> tables(table_size(n, resolution));
	make_tables(tables.data(), n, resolution);
	std::vector<double> errors(cells);
	std::vector<uint32_t> evaluations(cells), limit_hits(chains);
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	const size_t table_bytes = sizeof(double) * tables.size(), fit_bytes = sizeof(float) * 5 * cells, error_bytes = sizeof(double) * cells;
	const size_t evaluation_bytes = sizeof(uint32_t) * cells, hit_bytes = sizeof(uint32_t) * chains;
	char* block = nullptr;
	const size_t bytes = table_bytes + error_bytes + fit_bytes + evaluation_bytes + hit_bytes;
	if (cudaMalloc((void**) &block, bytes) != cudaSuccess) { printf("Failed to fit a linearly transformed cosine table: could not allocate %llu bytes on CUDA device %d.\n", (unsigned long long) bytes, device->cuda_device); return 1; }
	double* d_tables = (double*) block; double* d_errors = (double*) (block + table_bytes); float* d_fits = (float*) (block + table_bytes + error_bytes);
	uint32_t* d_evaluations = (uint32_t*) (block + table_bytes + error_bytes + fit_bytes); uint32_t* d_hits = d_evaluations + cells;
	cudaEvent_t begin = nullptr, end = nullptr;
	int rc = 0;
	float ms = 0.0f;
	if (cudaEventCreate(&begin) != cudaSuccess || cudaEventCreate(&end) != cudaSuccess
		|| cudaMemcpyAsync(d_tables, tables.data(), table_bytes, cudaMemcpyHostToDevice, stream) != cudaSuccess || cudaEventRecord(begin, stream) != cudaSuccess) rc = 1;
	if (!rc) {
		fit_kernel<<<(unsigned) chains, kThreads, 0, stream>>>(resolution, desc->fresnel_count, n, desc->iteration_limit, d_tables, d_fits, d_errors, d_evaluations, d_hits);
		if (cudaGetLastError() != cudaSuccess || cudaEventRecord(end, stream) != cudaSuccess
			|| cudaMemcpyAsync(out_fits, d_fits, fit_bytes, cudaMemcpyDeviceToHost, stream) != cudaSuccess
			|| cudaMemcpyAsync(errors.data(), d_errors, error_bytes, cudaMemcpyDeviceToHost, stream) != cudaSuccess
			|| cudaMemcpyAsync(evaluations.data(), d_evaluations, evaluation_bytes, cudaMemcpyDeviceToHost, stream) != cudaSuccess
			|| cudaMemcpyAsync(limit_hits.data(), d_hits, hit_bytes, cudaMemcpyDeviceToHost, stream) != cudaSuccess
			|| cudaStreamSynchronize(stream) != cudaSuccess || cudaEventElapsedTime(&ms, begin, end) != cudaSuccess) rc = 1;
	}
	if (rc) printf("Failed to fit a linearly transformed cosine table on CUDA device %d: %s\n", device->cuda_device, cudaGetErrorString(cudaGetLastError()));
	if (begin) cudaEventDestroy(begin);
	if (end) cudaEventDestroy(end);
	cudaFree(block);
	if (rc) return 1;
	if (stats) {
		stats->cell_count = cells; stats->objective_evaluations = 0; stats->iteration_limit_hits = 0; stats->fit_ms = ms;
		double sum = 0.0;
		for (uint64_t i = 0; i != cells; ++i) { stats->objective_evaluations += evaluations[i]; sum += errors[i]; }
		for (uint64_t c = 0; c != chains; ++c) stats->iteration_limit_hits += limit_hits[c];
		if (stats->cell_errors) std::copy(errors.begin(), errors.end(), stats->cell_errors);
		std::sort(errors.begin(), errors.end());
		stats->max_error = errors.back(); stats->median_error = errors[cells / 2]; stats->mean_error = sum / (double) cells;
	}
	return 0;
}

// fit<i>.dat as src/ltc_table.c:46-84 reads it: uint64 resolution, then resolution^2 texels of 5 float32, texel row * resolution + column
extern "C" int vkr_write_ltc_fits(const char* directory, uint32_t resolution, uint32_t fresnel_count, const float* fits) {
	if (!directory || !fits || resolution < 1 || resolution > VKR_LTC_FIT_MAX_RESOLUTION || fresnel_count < 1 || fresnel_count > VKR_LTC_FIT_MAX_FRESNEL_COUNT) {
		printf("Failed to write linearly transformed cosine tables: directory %s, resolution %u, Fresnel count %u.\n", directory ? directory : "(null)", resolution, fresnel_count);
		return 1;
	}
	const uint64_t texels = (uint64_t) resolution * resolution;
	for (uint32_t i = 0; i != fresnel_count; ++i) {
		const std::string path = std::string(directory) + "/fit" + std::to_string(i) + ".dat";
		FILE* file = fopen(path.c_str(), "wb");
		if (!file) { printf("Failed to open %s for writing.\n", path.c_str()); return 1; }
		const uint64_t header = resolution;
		bool ok = fwrite(&header, 8, 1, file) == 1 && fwrite(fits + 5 * texels * i, 4, 5 * texels, file) == 5 * texels;
		ok = (fclose(file) == 0) && ok;
		if (!ok) { printf("Failed to write %s.\n", path.c_str()); return 1; }
	}
	return 0;
}
