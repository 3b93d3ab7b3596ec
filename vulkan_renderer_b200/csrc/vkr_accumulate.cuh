// vkr_accumulate.cuh -- averaging frames and measuring their error (include/vkr_b200.h, vkr_accumulator_t / vkr_compare_frames).
//
// Everything the kernels of vkr_accumulate.cu compute is written here as per-pixel and per-thread functions, and every addition has a fixed
// order, so that a host build (tests/accumulate_on_host.cpp, plain g++ with -ffp-contract=off) performs the same float64 operations in the same
// order and gets the same bits. nvcc compiles the library with -fmad=false, so no product or quotient is fused into an addition on either side.
//
// Accumulation (one thread per pixel, frames in the order they are added): per channel a running mean and sum of squared deviations by
// Welford's rule, frame n = 1, 2, ...:  d = x - mean; mean += d / n; m2 += d * (x - mean). The first frame is stored as it is (mean = x,
// m2 = 0), and a frame with d = 0 leaves the channel as it is: that is what the rule gives, except that -0 stays -0, so copies of one frame
// average to that frame bit for bit. State: kStatePlanes planes of width * height doubles,
// {mean r, g, b, m2 r, g, b}, so that every access of a warp is one coalesced run.
//
// Reductions (frame error, mean variance): kReduceBlocks blocks, block b over the contiguous pixel range [b * chunk, (b + 1) * chunk) with
// chunk = ceil(pixels / kReduceBlocks) -- never sized from the device. Thread t of a block sums the pixels b * chunk + t, + kReduceThreads, ...
// in that order, the threads of a block combine in a fixed halving tree (partial[t] += partial[t + s] for t < s, s = kReduceThreads / 2, ..., 1), and one block then
// sums the kReduceBlocks partials in index order. The result is the same on every device and on the host.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define VKR_ACC_FN __host__ __device__ inline
#else
#define VKR_ACC_FN inline
#endif

namespace vkr_acc {

constexpr int kStatePlanes = 6;       // mean r, g, b, m2 r, g, b
constexpr int kReduceBlocks = 1024;
constexpr int kReduceThreads = 256;
// slots of a partial: sums of (x-r)^2 [0..2], of (x-r)^2 / (r^2 + eps) [3..5], of |x-r| [6..8] (the mean variance uses [0..2] for the sum of
// m2 / (n-1)); the largest |x-r| [9]; pixels with six finite inputs [10]; pixels with a non-finite input [11]. Counts are exact in double.
constexpr int kSlots = 12;
constexpr int kSlotMax = 9, kSlotCount = 10, kSlotNonfinite = 11;
constexpr double kRelMseEpsilon = 0.01;   // relMSE = (x-r)^2 / (r^2 + 0.01), part of the definition

VKR_ACC_FN bool finite_value(double v) { return v - v == 0.0; }   // false for +-inf and NaN

// ---- accumulation: one frame's pixel i into the state (n = number of this frame, 1 for the first)
VKR_ACC_FN void welford_update(double x, double n, double& mean, double& m2) {
	if (n == 1.0) { mean = x; m2 = 0.0; return; }
	const double d = x - mean;
	if (d == 0.0) return;   // the rule would change nothing but the sign of a zero mean (-0 + +0 = +0)
	mean = mean + d / n;
	m2 = m2 + d * (x - mean);
}

VKR_ACC_FN void accumulate_pixel(double* state, uint64_t plane, uint64_t i, float r, float g, float b, uint64_t n) {
	const double nd = (double) n;
	const float x[3] = { r, g, b };
	for (int c = 0; c != 3; ++c) {
		double mean = 0.0, m2 = 0.0;
		if (n != 1) { mean = state[c * plane + i]; m2 = state[(3 + c) * plane + i]; }
		welford_update((double) x[c], nd, mean, m2);
		state[c * plane + i] = mean; state[(3 + c) * plane + i] = m2;
	}
}

// ---- resolve: mean rounded to float (alpha 1), per-frame sample variance m2 / (n - 1) rounded to float (alpha 0; needs n >= 2)
VKR_ACC_FN void resolve_pixel(const double* state, uint64_t plane, uint64_t i, uint64_t n, float* mean_rgba, float* variance_rgba) {
	if (mean_rgba) {
		for (int c = 0; c != 3; ++c) mean_rgba[4 * i + c] = (float) state[c * plane + i];
		mean_rgba[4 * i + 3] = 1.0f;
	}
	if (variance_rgba) {
		const double dof = (double) (n - 1);
		for (int c = 0; c != 3; ++c) variance_rgba[4 * i + c] = (float) (state[(3 + c) * plane + i] / dof);
		variance_rgba[4 * i + 3] = 0.0f;
	}
}

// ---- per-pixel terms of the reductions
VKR_ACC_FN void zero_terms(double* t) { for (int k = 0; k != kSlots; ++k) t[k] = 0.0; }

// frame x against reference r at pixel i (float4 each; alpha ignored): all six RGB inputs finite, or the pixel only counts as non-finite
VKR_ACC_FN void add_error_terms(double* t, const float* frame, const float* reference, uint64_t i) {
	double x[3], r[3];
	bool finite = true;
	for (int c = 0; c != 3; ++c) {
		x[c] = (double) frame[4 * i + c]; r[c] = (double) reference[4 * i + c];
		finite = finite && finite_value(x[c]) && finite_value(r[c]);
	}
	if (!finite) { t[kSlotNonfinite] = t[kSlotNonfinite] + 1.0; return; }
	for (int c = 0; c != 3; ++c) {
		const double d = x[c] - r[c];
		const double d2 = d * d;
		const double a = d < 0.0 ? -d : d;
		t[c] = t[c] + d2;
		t[3 + c] = t[3 + c] + d2 / (r[c] * r[c] + kRelMseEpsilon);
		t[6 + c] = t[6 + c] + a;
		if (a > t[kSlotMax]) t[kSlotMax] = a;
	}
	t[kSlotCount] = t[kSlotCount] + 1.0;
}

// the per-frame sample variance of pixel i, m2 / (n - 1), per channel
VKR_ACC_FN void add_variance_terms(double* t, const double* state, uint64_t plane, uint64_t i, double dof) {
	for (int c = 0; c != 3; ++c) t[c] = t[c] + state[(3 + c) * plane + i] / dof;
	t[kSlotCount] = t[kSlotCount] + 1.0;
}

// a += b, slot by slot (the largest |x-r| by maximum)
VKR_ACC_FN void combine_terms(double* a, const double* b) {
	for (int k = 0; k != kSlots; ++k) {
		if (k == kSlotMax) { if (b[k] > a[k]) a[k] = b[k]; }
		else a[k] = a[k] + b[k];
	}
}

// ---- the fixed partition
VKR_ACC_FN uint64_t partition_chunk(uint64_t pixels) { return (pixels + kReduceBlocks - 1) / kReduceBlocks; }
VKR_ACC_FN uint64_t partition_begin(uint64_t pixels, int block) { const uint64_t b = partition_chunk(pixels) * (uint64_t) block; return b < pixels ? b : pixels; }
VKR_ACC_FN uint64_t partition_end(uint64_t pixels, int block) { return partition_begin(pixels, block + 1); }

// what thread t of block b sums: pixels begin + t, begin + t + kReduceThreads, ... < end, in that order
VKR_ACC_FN void thread_error_terms(double* t, const float* frame, const float* reference, uint64_t pixels, int block, int thread) {
	zero_terms(t);
	const uint64_t end = partition_end(pixels, block);
	for (uint64_t i = partition_begin(pixels, block) + (uint64_t) thread; i < end; i += kReduceThreads) add_error_terms(t, frame, reference, i);
}

VKR_ACC_FN void thread_variance_terms(double* t, const double* state, uint64_t pixels, uint64_t n, int block, int thread) {
	zero_terms(t);
	const double dof = (double) (n - 1);
	const uint64_t end = partition_end(pixels, block);
	for (uint64_t i = partition_begin(pixels, block) + (uint64_t) thread; i < end; i += kReduceThreads) add_variance_terms(t, state, pixels, i, dof);
}

// slot k of the total: the kReduceBlocks block partials ([block][kSlots]) in index order
VKR_ACC_FN double total_slot(const double* partials, int k) {
	double s = partials[k];
	for (int b = 1; b != kReduceBlocks; ++b) {
		const double v = partials[(uint64_t) b * kSlots + k];
		if (k == kSlotMax) { if (v > s) s = v; }
		else s = s + v;
	}
	return s;
}

// ---- the metrics from the total (vkr_frame_error_t); means over no pixel are NaN
VKR_ACC_FN void finish_error(const double* total, double* mse, double* rel_mse, double* mae, double* max_abs_error, uint64_t* pixel_count, uint64_t* nonfinite_pixels) {
	const double n = total[kSlotCount];
	for (int c = 0; c != 3; ++c) { mse[c] = total[c] / n; rel_mse[c] = total[3 + c] / n; mae[c] = total[6 + c] / n; }
	*max_abs_error = total[kSlotMax];
	*pixel_count = (uint64_t) n; *nonfinite_pixels = (uint64_t) total[kSlotNonfinite];
}

VKR_ACC_FN void finish_mean_variance(const double* total, double* mean_variance) {
	for (int c = 0; c != 3; ++c) mean_variance[c] = total[c] / total[kSlotCount];
}

// ---- adaptive accumulation (vkr_adaptive_accumulator_t): the same state planes, plus per 16x8 screen tile (the unit a CTA of the shading pass shades)
// a frame count n_t and an active flag. Tile t = ty * tiles_x + tx holds the pixels x = 16 tx + k % 16, y = 8 ty + k / 16, k = 0 .. 127, that lie in
// the frame (edge tiles are clipped). The kernels run one CTA of kTilePixels threads per tile, thread k on pixel k.
//   Masked accumulate: every pixel of an active tile takes the frame by accumulate_pixel with n = n_t + 1, then n_t += 1; inactive tiles are not touched.
//   Tile test (target, min_frames, max_frames), per active tile with n = n_t: n >= max_frames -> inactive; else if n >= min_frames and every pixel
//   passes pixel_converged -> inactive. pixel_converged per channel c = 0, 1, 2 in that order: v = m2 / ((double) n * (double) (n - 1)),
//   bound = target * (mean * mean + kRelMseEpsilon), pass iff mean and m2 are finite and v <= bound. The conjunction over the pixels is exact,
//   so its order does not matter. A tile never becomes active again.
//   Estimated error: per channel the mean over all pixels of v / (mean * mean + kRelMseEpsilon), v with the pixel's own tile's n_t, summed with the
//   fixed partition, tree and final sum above (slots [0..2] and kSlotCount).
constexpr int kTileWidth = 16, kTileHeight = 8, kTilePixels = kTileWidth * kTileHeight;   // VKR_TILE_WIDTH x VKR_TILE_ROW_HEIGHT

VKR_ACC_FN uint32_t tiles_across(uint32_t width) { return (width + kTileWidth - 1) / kTileWidth; }
VKR_ACC_FN uint32_t tiles_down(uint32_t height) { return (height + kTileHeight - 1) / kTileHeight; }

// pixel k of tile `tile` -> its index i; false if that pixel lies outside the frame
VKR_ACC_FN bool tile_pixel(uint32_t width, uint32_t height, uint32_t tile, int k, uint64_t* i) {
	const uint32_t tx = tile % tiles_across(width), ty = tile / tiles_across(width);
	const uint32_t x = tx * kTileWidth + (uint32_t) k % kTileWidth, y = ty * kTileHeight + (uint32_t) k / kTileWidth;
	if (x >= width || y >= height) return false;
	*i = (uint64_t) y * width + x;
	return true;
}

VKR_ACC_FN uint32_t pixel_tile(uint32_t width, uint64_t i) {
	return (uint32_t) (i / width) / kTileHeight * tiles_across(width) + (uint32_t) (i % width) / kTileWidth;
}

// the estimated variance of the mean of n frames (n >= 2)
VKR_ACC_FN double variance_of_mean(double m2, uint32_t n) { return m2 / ((double) n * (double) (n - 1)); }

VKR_ACC_FN bool pixel_converged(const double* state, uint64_t plane, uint64_t i, uint32_t n, double target) {
	bool pass = true;
	for (int c = 0; c != 3; ++c) {
		const double mean = state[c * plane + i], m2 = state[(3 + c) * plane + i];
		const double v = variance_of_mean(m2, n);
		const double bound = target * (mean * mean + kRelMseEpsilon);
		pass = pass && finite_value(mean) && finite_value(m2) && v <= bound;
	}
	return pass;
}

// whether the pixels of an active tile with n frames have to be tested at all (they are read only then, and only then is n >= 2)
VKR_ACC_FN bool tile_needs_test(uint32_t n, uint32_t min_frames, uint32_t max_frames) { return n >= min_frames && n < max_frames; }

// the tile test's outcome for an active tile; converged: every pixel passed pixel_converged (looked at only if tile_needs_test)
VKR_ACC_FN bool tile_stays_active(uint32_t n, bool converged, uint32_t min_frames, uint32_t max_frames) {
	if (n >= max_frames) return false;
	return !(tile_needs_test(n, min_frames, max_frames) && converged);
}

VKR_ACC_FN void add_estimate_terms(double* t, const double* state, uint64_t plane, uint64_t i, uint32_t n) {
	for (int c = 0; c != 3; ++c) {
		const double mean = state[c * plane + i];
		t[c] = t[c] + variance_of_mean(state[(3 + c) * plane + i], n) / (mean * mean + kRelMseEpsilon);
	}
	t[kSlotCount] = t[kSlotCount] + 1.0;
}

VKR_ACC_FN void thread_estimate_terms(double* t, const double* state, const uint32_t* tile_frames, uint32_t width, uint64_t pixels, int block, int thread) {
	zero_terms(t);
	const uint64_t end = partition_end(pixels, block);
	for (uint64_t i = partition_begin(pixels, block) + (uint64_t) thread; i < end; i += kReduceThreads) add_estimate_terms(t, state, pixels, i, tile_frames[pixel_tile(width, i)]);
}

// ---- the reductions as one CPU thread runs them: the same blocks, threads, tree and final sum as the kernels (host builds only)
#ifndef __CUDACC__
template <class ThreadTerms> inline void reduce_on_host(double* total, ThreadTerms thread_terms) {
	static double partials[kReduceBlocks * kSlots];
	static double block[kReduceThreads][kSlots];
	for (int b = 0; b != kReduceBlocks; ++b) {
		for (int t = 0; t != kReduceThreads; ++t) thread_terms(block[t], b, t);
		for (int s = kReduceThreads / 2; s > 0; s >>= 1)
			for (int t = 0; t < s; ++t) combine_terms(block[t], block[t + s]);
		for (int k = 0; k != kSlots; ++k) partials[b * kSlots + k] = block[0][k];
	}
	for (int k = 0; k != kSlots; ++k) total[k] = total_slot(partials, k);
}
#endif

} // namespace vkr_acc
