// vkr_noise_gen.cuh -- generating the file-backed noise tables of vkr_noise_type_t (include/vkr_b200.h, vkr_generate_noise_table; DESIGN.md §5).
//
// Everything the kernels of vkr_noise_gen.cu compute is written here in 32-bit integer operations, so that a host build (tests/noise_gen_on_host.cpp)
// gets the same bits whatever the thread count or the order in which a CTA's threads finish. The only floating-point input is the dither arrays'
// weight table, which the host computes once (make_blue_weights) and hands to both builds.
//
// Layout (the loader's, src/noise_table.c:54-105): uint16 RGBA texels [layer][y][x][4]; the shader reads u / 65535.
//
// Hash: hash32 is Wellons' "lowbias32" integer finaliser (a bijection of uint32); mix(h, v) = hash32(h ^ v) chains inputs into a hash.
//
// Ahmed-Wonka table (vkr_noise_type_ahmed), after Ahmed and Wonka 2020: texel RG holds pair 0, BA pair 1, and point set s = 2 layer + pair is one
// scrambled (0,2)-sequence handed out in a hierarchical order of the pixels of a W = H = 2^m table (m <= 8):
//   - index i_s(x, y) has m base-4 digits, coarsest level k = 0 first; digit k = perm[quadrant] with quadrant = 2 ybit + xbit of the pixel inside its
//     level-k node (node size 2^(m-k), node coordinates (x, y) >> (m-k)) and perm the permutation of {0,1,2,3} of lexicographic rank
//     mix(order_seed(s), k << 16 | node_y << 8 | node_x) mod 24. Every aligned 2^j x 2^j block holds 4^j consecutive indices.
//   - point i of the 2D Sobol sequence at 16 bits: dimension 0 = bitreverse16(i); dimension 1 = XOR of c_k over the set bits k of i, c_0 = 0x8000,
//     c_k = c_(k-1) ^ (c_(k-1) >> 1).
//   - nested-uniform (Owen) scramble per coordinate: bit b is flipped by the top bit of mix(scramble_seed(s, dimension), (v >> (b + 1)) << 4 | b),
//     v the unscrambled coordinate.
//   Every aligned block of 4^j consecutive indices of a (0,2)-sequence is a (0, 2j, 2)-net, and an Owen scramble keeps that; so every aligned
//   2^j x 2^j block of a point set is a (0, 2j, 2)-net in 16-bit integers, and at 256 x 256 each channel of a layer is a permutation of 0..65535.
//
// Blue-noise dither arrays (vkr_noise_type_blue): every channel of every layer is its own array a = 4 layer + channel of N = W H pixels, made by
// void-and-cluster (Ulichney 1993) with exact integer energies:
//   - weights w(dx, dy) = floor(2^28 exp(-(dx'^2 + dy'^2) / (2 * 1.5^2)) + 1/2), dx' = min(dx, W - dx), dy' likewise (toroidal Gaussian, sigma 1.5);
//     the energy of a pixel is the sum of w over the offsets to the pixels of the current set. The sum over the whole torus stays below 2^32.
//   - tightest cluster: the pixel of the set with the largest energy; largest void: the pixel outside it with the smallest; ties go to the lowest
//     linear index y W + x. A CTA finds either with one maximum over the key (energy or ~energy) << 32 | ~index (select_key).
//   - initial pattern: floor(N / 10) pixels, candidate c = mix(array_seed(a), c) mod N for c = 0, 1, ..., skipping pixels already set.
//   - relaxation: remove the tightest cluster, insert the largest void; stop when the void is the pixel just removed (it goes back), or after N
//     iterations (an iteration limit hit, reported).
//   - phase 1: from the relaxed pattern, remove tightest clusters, ranks ones - 1 down to 0. Phase 2: from the relaxed pattern, insert largest voids,
//     ranks ones .. N/2 - 1. Phase 3: with the roles of set and complement reversed, insert the tightest cluster of the complement, ranks up to N - 1.
//     The complement's energy is S - E with S the same torus sum at every pixel, exactly, so its tightest cluster is the largest void of E with the
//     same tie rule: phase 3 is phase 2 carried on to N.
//   - value u = (2 r + 1) * 32768 / N of rank r, so each array holds every such value once.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define VKR_NOISE_FN __host__ __device__ inline
#define VKR_NOISE_HOST_FN __host__ inline
#else
#define VKR_NOISE_FN inline
#define VKR_NOISE_HOST_FN inline
#endif
#include <math.h>

namespace vkr_noise {

constexpr uint32_t kAhmedMaxLog2 = 8;              // indices fit 16 bits
constexpr uint32_t kBlueMaxPixels = 16384;         // energies and weights of one array in shared memory
constexpr uint32_t kBlueWeightLog2Scale = 28;
constexpr double kBlueSigma = 1.5;
constexpr uint32_t kNoPixel = 0xFFFFFFFFu;
enum : uint32_t { kSelectNone = 0, kSelectCluster = 1, kSelectVoid = 2 };
// domain tags of the seeds
constexpr uint32_t kTagOrder = 0x4F524452u, kTagScramble = 0x5343524Du, kTagBlue = 0x424C5545u;

VKR_NOISE_FN uint32_t hash32(uint32_t x) {
	x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
	return x;
}
VKR_NOISE_FN uint32_t mix(uint32_t h, uint32_t v) { return hash32(h ^ v); }

VKR_NOISE_FN uint32_t order_seed(uint32_t seed, uint32_t set) { return mix(mix(hash32(seed), kTagOrder), set); }
VKR_NOISE_FN uint32_t scramble_seed(uint32_t seed, uint32_t set, uint32_t dimension) { return mix(mix(mix(hash32(seed), kTagScramble), set), dimension); }
VKR_NOISE_FN uint32_t array_seed(uint32_t seed, uint32_t array) { return mix(mix(hash32(seed), kTagBlue), array); }

// ---- Ahmed-Wonka table

// entry q of the permutation of {0,1,2,3} of lexicographic rank perm < 24 (factorial number system, digits 6, 2, 1)
VKR_NOISE_FN uint32_t permute4(uint32_t perm, uint32_t q) {
	uint32_t remaining = 0x3210u;   // nibble j: the j-th smallest element not yet used
	const uint32_t digits[3] = { perm / 6, (perm / 2) % 3, perm % 2 };
	for (uint32_t k = 0; ; ++k) {
		const uint32_t d = k < 3 ? digits[k] : 0;
		const uint32_t element = (remaining >> (4 * d)) & 0xFu;
		if (k == q) return element;
		remaining = (remaining & ((1u << (4 * d)) - 1u)) | ((remaining >> (4 * d + 4)) << (4 * d));
	}
}

VKR_NOISE_FN uint32_t hop_index(uint32_t order, uint32_t m, uint32_t x, uint32_t y) {
	uint32_t i = 0;
	for (uint32_t k = 0; k != m; ++k) {
		const uint32_t shift = m - 1 - k;
		const uint32_t node = (k << 16) | ((y >> (shift + 1)) << 8) | (x >> (shift + 1));
		const uint32_t quadrant = (((y >> shift) & 1u) << 1) | ((x >> shift) & 1u);
		i = (i << 2) | permute4(mix(order, node) % 24u, quadrant);
	}
	return i;
}

VKR_NOISE_FN uint32_t bitreverse16(uint32_t v) {
	v = ((v >> 1) & 0x5555u) | ((v & 0x5555u) << 1);
	v = ((v >> 2) & 0x3333u) | ((v & 0x3333u) << 2);
	v = ((v >> 4) & 0x0F0Fu) | ((v & 0x0F0Fu) << 4);
	return ((v >> 8) & 0x00FFu) | ((v & 0x00FFu) << 8);
}

VKR_NOISE_FN uint32_t sobol1(uint32_t i) {
	uint32_t result = 0;
	for (uint32_t c = 0x8000u; i; i >>= 1, c ^= c >> 1)
		if (i & 1u) result ^= c;
	return result;
}

VKR_NOISE_FN uint32_t owen16(uint32_t scramble, uint32_t v) {
	uint32_t result = v;
	for (uint32_t b = 0; b != 16; ++b) result ^= (mix(scramble, ((v >> (b + 1)) << 4) | b) >> 31) << b;
	return result;
}

// the four channels of texel (x, y) of a layer of a 2^m x 2^m table
VKR_NOISE_FN void ahmed_texel(uint32_t seed, uint32_t m, uint32_t layer, uint32_t x, uint32_t y, uint16_t out[4]) {
	for (uint32_t pair = 0; pair != 2; ++pair) {
		const uint32_t s = 2 * layer + pair;
		const uint32_t i = hop_index(order_seed(seed, s), m, x, y);
		out[2 * pair] = (uint16_t) owen16(scramble_seed(seed, s, 0), bitreverse16(i));
		out[2 * pair + 1] = (uint16_t) owen16(scramble_seed(seed, s, 1), sobol1(i));
	}
}

// ---- blue-noise dither arrays

// W * H weights, [dy][dx]. Returns their sum, the energy of every pixel when the set is the whole torus (< 2^32 for every supported size).
VKR_NOISE_HOST_FN uint64_t make_blue_weights(uint32_t width, uint32_t height, uint32_t* weights) {
	uint64_t sum = 0;
	for (uint32_t dy = 0; dy != height; ++dy)
		for (uint32_t dx = 0; dx != width; ++dx) {
			const double x = (double) (dx < width - dx ? dx : width - dx), y = (double) (dy < height - dy ? dy : height - dy);
			const double w = floor(ldexp(exp(-(x * x + y * y) / (2.0 * kBlueSigma * kBlueSigma)), (int) kBlueWeightLog2Scale) + 0.5);
			weights[dy * width + dx] = (uint32_t) w;
			sum += (uint32_t) w;
		}
	return sum;
}

VKR_NOISE_FN uint32_t toroidal_weight(const uint32_t* weights, uint32_t log2_width, uint32_t width, uint32_t height, uint32_t p, uint32_t q) {
	const uint32_t dx = ((p & (width - 1)) - (q & (width - 1))) & (width - 1);
	const uint32_t dy = ((p >> log2_width) - (q >> log2_width)) & (height - 1);
	return weights[dy * width + dx];
}

// 0: not a candidate. The largest key is the tightest cluster (mode kSelectCluster) or the largest void (kSelectVoid), lowest index on ties.
VKR_NOISE_FN uint64_t select_key(uint32_t p, uint32_t energy, bool in_set, uint32_t mode) {
	if (mode == kSelectCluster && in_set) return ((uint64_t) energy << 32) | (uint32_t) ~p;
	if (mode == kSelectVoid && !in_set) return ((uint64_t) (uint32_t) ~energy << 32) | (uint32_t) ~p;
	return 0;
}
VKR_NOISE_FN uint32_t pixel_of(uint64_t key) { return ~(uint32_t) key; }
VKR_NOISE_FN uint16_t dither_value(uint32_t rank, uint32_t n) { return (uint16_t) ((2 * rank + 1) * (32768u / n)); }

// One dither array of n pixels. Cta provides, with every thread of a CTA calling in step:
//   clear()                      energies 0, set empty
//   in_set(p)                    whether p is in the set
//   step(q, add, mode)           inserts (add) or removes pixel q (kNoPixel: neither), updates every energy by +-w(p - q), and returns the largest
//                                select_key over all pixels afterwards
//   keep_prototype(), prototype(p)   a copy of the set
//   emit(p, rank)                stores the value of rank at p
//   sync()
// Returns 1 if the relaxation stopped at the iteration limit, else 0.
template <class Cta>
VKR_NOISE_FN uint32_t dither_array(Cta& cta, uint32_t n, uint32_t seed, uint32_t relaxation_limit) {
	const uint32_t ones = n / 10;
	cta.clear();
	uint64_t key = 0;
	for (uint32_t candidate = 0, placed = 0; placed != ones; ++candidate) {
		const uint32_t p = mix(seed, candidate) & (n - 1);
		const bool taken = cta.in_set(p);
		cta.sync();   // every thread has read the set before step() changes it
		if (taken) continue;
		key = cta.step(p, true, kSelectCluster);
		++placed;
	}
	uint32_t limit_hit = 0;
	if (ones) {
		for (uint32_t iteration = 0; ; ++iteration) {
			if (iteration == relaxation_limit) { limit_hit = 1; break; }
			const uint32_t cluster = pixel_of(key);
			key = cta.step(cluster, false, kSelectVoid);
			const uint32_t gap = pixel_of(key);
			if (gap == cluster) { cta.step(cluster, true, kSelectNone); break; }
			key = cta.step(gap, true, kSelectCluster);
		}
	}
	cta.keep_prototype();
	// phase 1
	key = cta.step(kNoPixel, false, kSelectCluster);
	for (uint32_t rank = ones; rank-- != 0;) {
		const uint32_t cluster = pixel_of(key);
		cta.emit(cluster, rank);
		key = cta.step(cluster, false, kSelectCluster);
	}
	// the set is empty and every energy 0 again; back to the relaxed pattern
	for (uint32_t p = 0; p != n; ++p)
		if (cta.prototype(p)) cta.step(p, true, kSelectNone);
	// phases 2 and 3
	key = cta.step(kNoPixel, true, kSelectVoid);
	for (uint32_t rank = ones; rank != n; ++rank) {
		const uint32_t gap = pixel_of(key);
		cta.emit(gap, rank);
		key = cta.step(gap, true, kSelectVoid);
	}
	return limit_hit;
}

} // namespace vkr_noise
