// tests/noise_gen_on_host.cpp -- TEST INFRASTRUCTURE: the noise tables (vulkan_renderer_b200/csrc/vkr_noise_gen.cuh) compiled for the CPU. Loops stand
// in for the launches: texel by texel for the Ahmed-Wonka table, and for a dither array one pass over its pixels per insertion or removal in place of
// the CTA's threads. Only integer operations, maxima and exact sums are involved, so the result does not depend on the order. tests/test_noise_gen_on_host.py
// holds this against the numpy restatement in vulkan_renderer_b200/noise_gen.py; the -m gpu tests hold the kernels against this bit for bit. Built by
// __graft_entry__.build() into tests/build/libnoise_gen_on_host.so. Nothing in the product links against it.
#include <cstdint>
#include <vector>

#include "vkr_noise_gen.cuh"

using namespace vkr_noise;

namespace {

struct HostCta {
	uint32_t n, width, height, log2_width;
	const uint32_t* weights;
	std::vector<uint32_t> energy;
	std::vector<uint8_t> member, kept;
	uint16_t* out;   // texel channel of pixel p at out[4 p]

	void sync() {}
	void clear() { energy.assign(n, 0); member.assign(n, 0); }
	bool in_set(uint32_t p) const { return member[p] != 0; }
	void keep_prototype() { kept = member; }
	bool prototype(uint32_t p) const { return kept[p] != 0; }
	void emit(uint32_t p, uint32_t rank) { out[4 * (uint64_t) p] = dither_value(rank, n); }
	uint64_t step(uint32_t q, bool add, uint32_t mode) {
		uint64_t best = 0;
		for (uint32_t p = 0; p != n; ++p) {
			if (q != kNoPixel) {
				const uint32_t w = toroidal_weight(weights, log2_width, width, height, p, q);
				energy[p] = add ? energy[p] + w : energy[p] - w;
				if (p == q) member[p] = add;
			}
			const uint64_t k = select_key(p, energy[p], member[p] != 0, mode);
			best = k > best ? k : best;
		}
		return best;
	}
};

uint32_t log2_of(uint32_t v) { uint32_t r = 0; while ((1u << r) < v) ++r; return r; }

} // namespace

extern "C" uint64_t vkr_host_noise_blue_weights(uint32_t width, uint32_t height, uint32_t* weights) { return make_blue_weights(width, height, weights); }

// layers [layer_begin, layer_end) of a 2^m x 2^m Ahmed-Wonka table; texels: (layer_end - layer_begin) * 4^m * 4 uint16
extern "C" void vkr_host_noise_ahmed(uint32_t seed, uint32_t m, uint32_t layer_begin, uint32_t layer_end, uint16_t* texels) {
	const uint32_t size = 1u << m;
	#pragma omp parallel for schedule(static)
	for (int64_t layer = layer_begin; layer < (int64_t) layer_end; ++layer)
		for (uint32_t y = 0; y != size; ++y)
			for (uint32_t x = 0; x != size; ++x)
				ahmed_texel(seed, m, (uint32_t) layer, x, y, texels + 4 * (((uint64_t) (layer - layer_begin) * size + y) * size + x));
}

// dither arrays [array_begin, array_end) of a width x height x layers blue-noise table, as the kernel makes them: array a = 4 layer + channel goes to
// channel a mod 4 of layer a / 4 - array_begin / 4 of texels; limit_hits: one entry per array. array_begin is a multiple of 4.
extern "C" void vkr_host_noise_blue(uint32_t seed, uint32_t width, uint32_t height, uint32_t array_begin, uint32_t array_end, uint16_t* texels, uint32_t* limit_hits) {
	const uint32_t n = width * height;
	std::vector<uint32_t> weights(n);
	make_blue_weights(width, height, weights.data());
	#pragma omp parallel for schedule(dynamic, 1)
	for (int64_t a = array_begin; a < (int64_t) array_end; ++a) {
		HostCta cta;
		cta.n = n; cta.width = width; cta.height = height; cta.log2_width = log2_of(width); cta.weights = weights.data();
		cta.out = texels + (uint64_t) ((a - array_begin) >> 2) * n * 4 + (a & 3);
		limit_hits[a - array_begin] = dither_array(cta, n, array_seed(seed, (uint32_t) a), n);
	}
}
