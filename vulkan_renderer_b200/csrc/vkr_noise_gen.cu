// vkr_noise_gen.cu -- generating the blue-noise and Ahmed-Wonka noise tables on the device and writing them as the .blob files that
// vkr_load_noise_table reads (include/vkr_b200.h, vkr_generate_noise_table, vkr_write_noise_table). The reference reads these files from its data
// download (src/noise_table.c:76-107) and has no generator. The arithmetic lives in vkr_noise_gen.cuh, which the CPU tests compile too.
//   - Ahmed-Wonka: one thread per texel, both pairs.
//   - blue noise: one CTA per dither array; energies, weights and the set stay in shared memory, and each insertion or removal is one pass over the
//     pixels that updates the energies and finds the next cluster or void with one CTA-wide maximum.
#include "../../include/vkr_b200.h"
#include "vkr_noise_gen.cuh"
#include <cuda_runtime.h>
#include <errno.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>
#include <string>
#include <vector>

using namespace vkr_noise;

static_assert((1u << kAhmedMaxLog2) == VKR_NOISE_GEN_MAX_AHMED_SIZE && kBlueMaxPixels == VKR_NOISE_GEN_MAX_BLUE_PIXELS, "include/vkr_b200.h states the limits");

namespace {

constexpr uint32_t kAhmedThreads = 256;
constexpr uint32_t kBlueThreads = 1024;
constexpr uint32_t kBlueWarps = kBlueThreads / 32;

__global__ void __launch_bounds__(kAhmedThreads) ahmed_kernel(uint32_t seed, uint32_t m, uint32_t layers, uint2* __restrict__ texels) {
	const uint32_t size = 1u << m;
	const uint64_t t = (uint64_t) blockIdx.x * kAhmedThreads + threadIdx.x;
	if (t >= (uint64_t) size * size * layers) return;
	const uint32_t x = (uint32_t) t & (size - 1), y = (uint32_t) (t >> m) & (size - 1), layer = (uint32_t) (t >> (2 * m));
	uint16_t v[4];
	ahmed_texel(seed, m, layer, x, y, v);
	texels[t] = make_uint2(v[0] | ((uint32_t) v[1] << 16), v[2] | ((uint32_t) v[3] << 16));
}

// the Cta of dither_array: thread t owns pixels t, t + kBlueThreads, ...; only the owner touches a pixel's energy and membership
struct DeviceCta {
	uint32_t n, width, height, log2_width;
	const uint32_t* weights;                  // shared
	uint32_t* energy;                         // shared
	uint8_t* member;                          // shared
	uint8_t* kept;                            // shared
	uint64_t (*warp_best)[kBlueWarps];        // shared [2][kBlueWarps]: one buffer per parity, so one barrier per step suffices
	uint16_t* out;                            // global: texel channel of pixel p at out[4 p]
	uint32_t parity;

	__device__ void sync() { __syncthreads(); }
	__device__ void clear() {
		for (uint32_t p = threadIdx.x; p < n; p += kBlueThreads) { energy[p] = 0; member[p] = 0; }
		__syncthreads();
	}
	__device__ bool in_set(uint32_t p) const { return member[p] != 0; }
	__device__ void keep_prototype() {
		for (uint32_t p = threadIdx.x; p < n; p += kBlueThreads) kept[p] = member[p];
		__syncthreads();
	}
	__device__ bool prototype(uint32_t p) const { return kept[p] != 0; }
	__device__ void emit(uint32_t p, uint32_t rank) { if (threadIdx.x == 0) out[4 * (uint64_t) p] = dither_value(rank, n); }
	__device__ uint64_t step(uint32_t q, bool add, uint32_t mode) {
		uint64_t best = 0;
		for (uint32_t p = threadIdx.x; p < n; p += kBlueThreads) {
			uint32_t e = energy[p];
			bool in = member[p] != 0;
			if (q != kNoPixel) {
				const uint32_t w = toroidal_weight(weights, log2_width, width, height, p, q);
				e = add ? e + w : e - w;
				energy[p] = e;
				if (p == q) { in = add; member[p] = add; }
			}
			const uint64_t k = select_key(p, e, in, mode);
			best = k > best ? k : best;
		}
		for (int offset = 16; offset; offset >>= 1) {
			const uint64_t other = __shfl_xor_sync(0xFFFFFFFFu, best, offset);
			best = other > best ? other : best;
		}
		if ((threadIdx.x & 31) == 0) warp_best[parity][threadIdx.x >> 5] = best;
		__syncthreads();
		best = 0;
		for (uint32_t w = 0; w != kBlueWarps; ++w) best = warp_best[parity][w] > best ? warp_best[parity][w] : best;
		parity ^= 1;
		return best;
	}
};

size_t blue_shared_bytes(uint32_t n) { return 2 * sizeof(uint64_t) * kBlueWarps + (size_t) n * (2 * sizeof(uint32_t) + 2); }

// block a makes dither array a = 4 layer + channel
__global__ void __launch_bounds__(kBlueThreads, 1) blue_kernel(uint32_t seed, uint32_t width, uint32_t height, uint32_t log2_width, const uint32_t* __restrict__ weights,
	uint16_t* texels, uint32_t* limit_hits)
{
	extern __shared__ uint64_t shared[];
	const uint32_t n = width * height, array = blockIdx.x;
	DeviceCta cta;
	cta.n = n; cta.width = width; cta.height = height; cta.log2_width = log2_width; cta.parity = 0;
	cta.warp_best = (uint64_t (*)[kBlueWarps]) shared;
	uint32_t* w = (uint32_t*) (shared + 2 * kBlueWarps);
	cta.energy = w + n;
	cta.member = (uint8_t*) (cta.energy + n);
	cta.kept = cta.member + n;
	for (uint32_t i = threadIdx.x; i < n; i += kBlueThreads) w[i] = weights[i];
	cta.weights = w;
	cta.out = texels + (uint64_t) (array >> 2) * n * 4 + (array & 3);
	const uint32_t hit = dither_array(cta, n, array_seed(seed, array), n);   // clear() synchronises before the weights are read
	if (threadIdx.x == 0) limit_hits[array] = hit;
}

bool power_of_two(uint32_t v) { return v && !(v & (v - 1)); }
uint32_t log2_of(uint32_t v) { uint32_t r = 0; while ((1u << r) < v) ++r; return r; }

// the loader's rules (vkr_load_noise_table) for a file-backed type
int check_layout(const char* what, vkr_noise_type_t type, uint32_t width, uint32_t height, uint32_t layers) {
	if (type != vkr_noise_type_blue && type != vkr_noise_type_ahmed) { printf("Failed to %s a noise table: type %d has no file (blue = 1, ahmed = 2).\n", what, (int) type); return 1; }
	if (width > 9999 || height > 9999 || layers > 9999 || !power_of_two(width) || !power_of_two(height) || !power_of_two(layers)) {
		printf("Failed to %s a noise table: %u x %u x %u is not a power-of-two size the loader accepts.\n", what, width, height, layers);
		return 1;
	}
	return 0;
}

int check_desc(const vkr_noise_gen_desc_t* desc) {
	if (!desc) { printf("Failed to generate a noise table: no descriptor.\n"); return 1; }
	if (check_layout("generate", desc->type, desc->width, desc->height, desc->layers)) return 1;
	if (desc->type == vkr_noise_type_ahmed && (desc->width != desc->height || desc->width > (1u << kAhmedMaxLog2))) {
		printf("Failed to generate a noise table: Ahmed tables are square and at most %u x %u, not %u x %u.\n", 1u << kAhmedMaxLog2, 1u << kAhmedMaxLog2, desc->width, desc->height);
		return 1;
	}
	if (desc->type == vkr_noise_type_blue && desc->width * desc->height > kBlueMaxPixels) {
		printf("Failed to generate a noise table: dither arrays hold at most %u pixels, not %u x %u.\n", kBlueMaxPixels, desc->width, desc->height);
		return 1;
	}
	return 0;
}

#define VKR_NOISE_TRY(call) do { if ((call) != cudaSuccess) { rc = 1; goto done; } } while (0)

} // namespace

extern "C" void vkr_noise_gen_default_desc(vkr_noise_type_t type, vkr_noise_gen_desc_t* desc) {
	// get_default_noise_resolution (src/noise_table.c:22-40)
	desc->type = type;
	desc->width = desc->height = (type == vkr_noise_type_blue) ? 64 : 256;
	desc->layers = 64;
	desc->seed = 0;
}

extern "C" int vkr_generate_noise_table(const vkr_device_t* device, const vkr_noise_gen_desc_t* desc, uint16_t* texels_rgba16, vkr_noise_gen_stats_t* stats) {
	if (check_desc(desc)) return 1;
	if (!device || !texels_rgba16) { printf("Failed to generate a noise table: no device or no output array.\n"); return 1; }
	const uint32_t width = desc->width, height = desc->height, layers = desc->layers, n = width * height;
	const size_t texel_bytes = sizeof(uint16_t) * 4 * (size_t) n * layers;
	const bool blue = desc->type == vkr_noise_type_blue;
	const uint32_t arrays = 4 * layers;
	std::vector<uint32_t> weights, hits;
	if (blue) { weights.resize(n); hits.resize(arrays); make_blue_weights(width, height, weights.data()); }
	const size_t weight_bytes = sizeof(uint32_t) * weights.size(), hit_bytes = sizeof(uint32_t) * hits.size();
	cudaStream_t stream = (cudaStream_t) device->stream;
	char* block = nullptr;
	cudaEvent_t begin = nullptr, end = nullptr;
	float ms = 0.0f;
	int rc = 0;
	VKR_NOISE_TRY(cudaSetDevice(device->cuda_device));
	VKR_NOISE_TRY(cudaMalloc((void**) &block, texel_bytes + weight_bytes + hit_bytes));
	VKR_NOISE_TRY(cudaEventCreate(&begin));
	VKR_NOISE_TRY(cudaEventCreate(&end));
	if (blue) {
		uint32_t* d_weights = (uint32_t*) (block + texel_bytes);
		uint32_t* d_hits = d_weights + n;
		const size_t shared = blue_shared_bytes(n);
		VKR_NOISE_TRY(cudaFuncSetAttribute(blue_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) shared));
		VKR_NOISE_TRY(cudaMemcpyAsync(d_weights, weights.data(), weight_bytes, cudaMemcpyHostToDevice, stream));
		VKR_NOISE_TRY(cudaEventRecord(begin, stream));
		blue_kernel<<<arrays, kBlueThreads, shared, stream>>>(desc->seed, width, height, log2_of(width), d_weights, (uint16_t*) block, d_hits);
		VKR_NOISE_TRY(cudaGetLastError());
		VKR_NOISE_TRY(cudaEventRecord(end, stream));
		VKR_NOISE_TRY(cudaMemcpyAsync(hits.data(), d_hits, hit_bytes, cudaMemcpyDeviceToHost, stream));
	}
	else {
		const uint64_t texels = (uint64_t) n * layers;
		VKR_NOISE_TRY(cudaEventRecord(begin, stream));
		ahmed_kernel<<<(unsigned) ((texels + kAhmedThreads - 1) / kAhmedThreads), kAhmedThreads, 0, stream>>>(desc->seed, log2_of(width), layers, (uint2*) block);
		VKR_NOISE_TRY(cudaGetLastError());
		VKR_NOISE_TRY(cudaEventRecord(end, stream));
	}
	VKR_NOISE_TRY(cudaMemcpyAsync(texels_rgba16, block, texel_bytes, cudaMemcpyDeviceToHost, stream));
	VKR_NOISE_TRY(cudaStreamSynchronize(stream));
	VKR_NOISE_TRY(cudaEventElapsedTime(&ms, begin, end));
done:
	if (rc) printf("Failed to generate a noise table on CUDA device %d: %s\n", device->cuda_device, cudaGetErrorString(cudaGetLastError()));
	if (begin) cudaEventDestroy(begin);
	if (end) cudaEventDestroy(end);
	cudaFree(block);
	if (rc) return 1;
	if (stats) {
		stats->kernel_ms = ms;
		stats->relaxation_limit_hits = 0;
		for (uint32_t h : hits) stats->relaxation_limit_hits += h;
	}
	return 0;
}

// root/data/noise/<name> with the name vkr_load_noise_table opens: raw uint16 RGBA texels, [layer][y][x][4]
extern "C" int vkr_write_noise_table(const char* root, vkr_noise_type_t type, uint32_t width, uint32_t height, uint32_t layers, const uint16_t* texels_rgba16) {
	if (!root || !texels_rgba16) { printf("Failed to write a noise table: no root directory or no texels.\n"); return 1; }
	if (check_layout("write", type, width, height, layers)) return 1;
	std::string directory = root;
	for (const char* part : { "", "/data", "/data/noise" }) {   // the parent of root must exist
		const std::string path = directory + part;
		if (mkdir(path.c_str(), 0777) != 0 && errno != EEXIST) { printf("Failed to create the directory %s: %s\n", path.c_str(), strerror(errno)); return 1; }
	}
	char name[96];
	snprintf(name, sizeof(name), type == vkr_noise_type_blue ? "/data/noise/blue_noise_rgba_%02dx%02d_%02d.blob" : "/data/noise/ahmed_2d_rgba_%02dx%02d_%02d.blob",
		(int) width, (int) height, (int) layers);
	const std::string path = directory + name;
	FILE* file = fopen(path.c_str(), "wb");
	if (!file) { printf("Failed to open %s for writing.\n", path.c_str()); return 1; }
	const size_t count = (size_t) width * height * layers * 4;
	bool ok = fwrite(texels_rgba16, sizeof(uint16_t), count, file) == count;
	ok = (fclose(file) == 0) && ok;
	if (!ok) { printf("Failed to write %s.\n", path.c_str()); return 1; }
	return 0;
}
