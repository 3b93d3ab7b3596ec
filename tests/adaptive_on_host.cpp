// tests/adaptive_on_host.cpp -- TEST INFRASTRUCTURE: the adaptive accumulator's arithmetic (vulkan_renderer_b200/csrc/vkr_accumulate.cuh) compiled for
// the CPU. The loops stand in for the launches: tile by tile, pixel k = 0 .. 127 of each tile, for the masked accumulate, the tile test and the resolve
// (one CTA per tile on the device), and block by block, thread by thread, then the halving tree and final sum for the estimated relMSE, so every
// float64 operation happens in the order the kernels perform it. -ffp-contract=off stands in for nvcc's -fmad=false. tests/test_adaptive_on_host.py
// holds this against numpy float64; the -m gpu tests hold the kernels against this bit for bit. Built by __graft_entry__.build() into
// tests/build/libadaptive_on_host.so. Nothing in the product links against it.
#include <cstdint>

#include "vkr_accumulate.cuh"

using namespace vkr_acc;

static uint32_t tile_count(uint32_t width, uint32_t height) { return tiles_across(width) * tiles_down(height); }

// one frame (width * height float4) into the state of the active tiles; n_t += 1 for each of them
extern "C" void vkr_host_adaptive_accumulate(uint32_t width, uint32_t height, const float* frame, double* state, uint32_t* tile_frames, const uint8_t* active) {
	const uint64_t pixels = (uint64_t) width * height;
	for (uint32_t t = 0; t != tile_count(width, height); ++t) {
		if (!active[t]) continue;
		const uint32_t n = tile_frames[t];
		for (int k = 0; k != kTilePixels; ++k) {
			uint64_t i;
			if (tile_pixel(width, height, t, k, &i)) accumulate_pixel(state, pixels, i, frame[4 * i], frame[4 * i + 1], frame[4 * i + 2], (uint64_t) n + 1);
		}
		tile_frames[t] = n + 1;
	}
}

// the tile test: active is updated in place
extern "C" void vkr_host_adaptive_update(uint32_t width, uint32_t height, const double* state, const uint32_t* tile_frames, uint8_t* active, double target,
	uint32_t min_frames, uint32_t max_frames)
{
	const uint64_t pixels = (uint64_t) width * height;
	for (uint32_t t = 0; t != tile_count(width, height); ++t) {
		if (!active[t]) continue;
		const uint32_t n = tile_frames[t];
		bool converged = false;
		if (tile_needs_test(n, min_frames, max_frames)) {
			converged = true;
			for (int k = 0; k != kTilePixels; ++k) {
				uint64_t i;
				if (tile_pixel(width, height, t, k, &i)) converged = converged && pixel_converged(state, pixels, i, n, target);
			}
		}
		active[t] = tile_stays_active(n, converged, min_frames, max_frames) ? 1 : 0;
	}
}

// mean_rgba / variance_rgba may be NULL, like vkr_adaptive_resolve
extern "C" void vkr_host_adaptive_resolve(uint32_t width, uint32_t height, const double* state, const uint32_t* tile_frames, float* mean_rgba, float* variance_rgba) {
	const uint64_t pixels = (uint64_t) width * height;
	for (uint32_t t = 0; t != tile_count(width, height); ++t)
		for (int k = 0; k != kTilePixels; ++k) {
			uint64_t i;
			if (tile_pixel(width, height, t, k, &i)) resolve_pixel(state, pixels, i, tile_frames[t], mean_rgba, variance_rgba);
		}
}

extern "C" void vkr_host_adaptive_estimate(uint32_t width, uint32_t height, const double* state, const uint32_t* tile_frames, double out[3]) {
	const uint64_t pixels = (uint64_t) width * height;
	double total[kSlots];
	reduce_on_host(total, [&](double* t, int b, int k) { thread_estimate_terms(t, state, tile_frames, width, pixels, b, k); });
	finish_mean_variance(total, out);
}
