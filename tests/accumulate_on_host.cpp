// tests/accumulate_on_host.cpp -- TEST INFRASTRUCTURE: the accumulator's arithmetic (vulkan_renderer_b200/csrc/vkr_accumulate.cuh) compiled for the
// CPU. The loops stand in for the launches: pixel by pixel for the accumulate and resolve kernels, and block by block, thread by thread, then the
// same halving tree and final sum for the reductions, so every float64 operation happens in the order the kernels perform it. -ffp-contract=off
// stands in for nvcc's -fmad=false. tests/test_accumulate_on_host.py holds this against numpy float64; the -m gpu tests hold the kernels against this
// bit for bit. Built by __graft_entry__.build() into tests/build/libaccumulate_on_host.so. Nothing in the product links against it.
#include <cstdint>

#include "vkr_accumulate.cuh"

using namespace vkr_acc;

// frames: frame_count frames of pixels float4 each, back to back -> state (kStatePlanes planes of pixels doubles)
extern "C" void vkr_host_accumulate(uint64_t pixels, uint64_t frame_count, const float* frames, double* state) {
	for (uint64_t f = 0; f != frame_count; ++f) {
		const float* x = frames + 4 * pixels * f;
		for (uint64_t i = 0; i != pixels; ++i) accumulate_pixel(state, pixels, i, x[4 * i], x[4 * i + 1], x[4 * i + 2], f + 1);
	}
}

// mean_rgba / variance_rgba may be NULL, like vkr_accumulator_resolve
extern "C" void vkr_host_resolve(uint64_t pixels, uint64_t frame_count, const double* state, float* mean_rgba, float* variance_rgba) {
	for (uint64_t i = 0; i != pixels; ++i) resolve_pixel(state, pixels, i, frame_count, mean_rgba, variance_rgba);
}

extern "C" void vkr_host_mean_variance(uint64_t pixels, uint64_t frame_count, const double* state, double out[3]) {
	double total[kSlots];
	reduce_on_host(total, [&](double* t, int b, int k) { thread_variance_terms(t, state, pixels, frame_count, b, k); });
	finish_mean_variance(total, out);
}

struct frame_error { double mse[3], rel_mse[3], mae[3], max_abs_error; uint64_t pixel_count, nonfinite_pixels; };   // vkr_frame_error_t's layout

extern "C" void vkr_host_compare(uint64_t pixels, const float* frame, const float* reference, frame_error* out) {
	double total[kSlots];
	reduce_on_host(total, [&](double* t, int b, int k) { thread_error_terms(t, frame, reference, pixels, b, k); });
	finish_error(total, out->mse, out->rel_mse, out->mae, &out->max_abs_error, &out->pixel_count, &out->nonfinite_pixels);
}
