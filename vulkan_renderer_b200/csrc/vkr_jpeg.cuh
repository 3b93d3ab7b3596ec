// vkr_jpeg.cuh -- baseline sequential JPEG (ITU-T T.81) of an 8-bit RGB image, three components, Huffman coded with the tables of Annex K
// (include/vkr_b200.h, vkr_encode_jpg; DESIGN.md §5 "JPEG screenshots").
//
// The file is the one stbi_write_jpg (stb_image_write v1.14, which the reference's screenshots use) writes for the same pixels and quality, byte
// for byte. The format leaves the encoder free in its colour conversion, DCT, rounding and headers, so each of these is pinned to stb's choice:
//   - quality q: 0 means 90; q <= 90 (tested before the clamp) selects 4:2:0 (16x16 MCUs: Y0 Y1 Y2 Y3 Cb Cr), above it 4:4:4 (8x8 MCUs: Y Cb Cr).
//     q is clamped to 1..100 and scaled the IJG way, s = q < 50 ? 5000 / q : 200 - 2 q; each entry of the Annex K tables (K.1, K.2) becomes
//     clamp((T s + 50) / 100, 1, 255) in integers.
//   - pixels outside the image repeat the last row / column.
//   - RGB -> YCbCr in float: Y = 0.299 R + 0.587 G + 0.114 B - 128, Cb = -0.16874 R - 0.33126 G + 0.5 B, Cr = 0.5 R - 0.41869 G - 0.08131 B, summed
//     left to right. In 4:2:0, a chroma sample is (a + b + c + d) * 0.25 over the 2x2 pixels, left to right, top row first.
//   - DCT: the float AAN flow graph (Arai, Agui and Nakajima 1988; Pennebaker and Mitchell, fig. 4-8), rows first, then columns. Its outputs are
//     the DCT coefficients times 8 a(u) a(v), a(0) = 1, a(k) = sqrt(2) cos(k pi / 16); quantisation multiplies by 1 / (Q * A[u] * A[v]) with
//     A[k] = a(k) * sqrt(8) rounded to float, the product evaluated left to right, once on the host (make_params).
//   - rounding: (int) (v < 0 ? v - 0.5 : v + 0.5), i.e. half away from zero.
// Every product and sum is rounded on its own (nvcc -fmad=false, host builds -ffp-contract=off), so the host build of this header and the kernels
// agree bit for bit.
//
// Entropy coding: DC differences against the previous block of the same component in stream order (0 before the first), AC run/size symbols with
// a ZRL (0xF0) per 16 zeros and an EOB unless coefficient 63 is non-zero. After the last block the stream is padded with 1-bits to a byte
// boundary, and every 0xFF byte of it is followed by a stuffed 0x00 (T.81 F.1.2.3, B.1.1.5).
//
// Data-parallel shape (vkr_jpeg.cu; tests/jpeg_on_host.cpp runs the same stages as loops): block b of the stream is coded from its own 64
// coefficients and its predecessor's DC alone (walk_block), so every block's bit count is known independently, an exclusive scan gives each its bit
// offset, and each block writes its bits into a zeroed array of 32-bit words (bit 31 first). Only a block's first and last word can be shared with
// a neighbour; those are OR-ed in, so the result does not depend on the order of the writes.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#ifdef __CUDACC__
#define VKR_JPEG_FN __host__ __device__ inline
#else
#define VKR_JPEG_FN inline
#endif

namespace vkr_jpeg {

constexpr uint32_t kMaxSide = 65535;      // SOF0 holds 16-bit sizes
constexpr size_t kHeaderBytes = 607;      // SOI .. SOS as write_header lays them out
constexpr size_t kTrailerBytes = 2;       // EOI

// zigzag position of the coefficient at natural (row-major) index i (T.81 figure A.6)
constexpr uint8_t kZigzag[64] = {
	 0,  1,  5,  6, 14, 15, 27, 28,  2,  4,  7, 13, 16, 26, 29, 42,  3,  8, 12, 17, 25, 30, 41, 43,  9, 11, 18, 24, 31, 40, 44, 53,
	10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63 };

// T.81 tables K.1 (luminance) and K.2 (chrominance), natural order
constexpr uint8_t kLumaQuant[64] = {
	16, 11, 10, 16,  24,  40,  51,  61,   12, 12, 14, 19,  26,  58,  60,  55,   14, 13, 16, 24,  40,  57,  69,  56,   14, 17, 22, 29,  51,  87,  80,  62,
	18, 22, 37, 56,  68, 109, 103,  77,   24, 35, 55, 64,  81, 104, 113,  92,   49, 64, 78, 87, 103, 121, 120, 101,   72, 92, 95, 98, 112, 100, 103,  99 };
constexpr uint8_t kChromaQuant[64] = {
	17, 18, 24, 47, 99, 99, 99, 99,   18, 21, 26, 66, 99, 99, 99, 99,   24, 26, 56, 99, 99, 99, 99, 99,   47, 66, 99, 99, 99, 99, 99, 99,
	99, 99, 99, 99, 99, 99, 99, 99,   99, 99, 99, 99, 99, 99, 99, 99,   99, 99, 99, 99, 99, 99, 99, 99,   99, 99, 99, 99, 99, 99, 99, 99 };

// T.81 tables K.3 - K.6 as DHT stores them: code counts per length 1..16, then the symbols
constexpr uint8_t kDcLumaBits[16] = { 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0 };
constexpr uint8_t kDcChromaBits[16] = { 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0 };
constexpr uint8_t kDcSymbols[12] = { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11 };
constexpr uint8_t kAcLumaBits[16] = { 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d };
constexpr uint8_t kAcLumaSymbols[162] = {
	0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08,
	0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
	0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
	0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
	0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
	0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
	0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa };
constexpr uint8_t kAcChromaBits[16] = { 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77 };
constexpr uint8_t kAcChromaSymbols[162] = {
	0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91,
	0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
	0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
	0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
	0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
	0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
	0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa };

// a(k) = sqrt(2) cos(k pi / 16), a(0) = 1, and sqrt(8): the AAN output scale
constexpr float kAanScale[8] = { 1.0f, 1.387039845f, 1.306562965f, 1.175875602f, 1.0f, 0.785694958f, 0.541196100f, 0.275899379f };
constexpr float kSqrt8 = 2.828427125f;

// Everything the kernels need besides the pixels; passed by value (2.8 KB, under the 4 KB of kernel parameters). The tables are copied in
// here because device code cannot read the host's constexpr arrays.
// A Huffman code is (length << 16) | code, code right-aligned; class 0 = luminance, 1 = chrominance.
struct Params {
	float reciprocal[2][64];      // natural order
	uint32_t dc_code[2][16];      // by magnitude category 0..11
	uint32_t ac_code[2][256];     // by run/size symbol
	uint8_t zigzag[64];           // kZigzag
	uint32_t width, height;
	uint32_t subsample;           // 1: 4:2:0
	uint32_t mcus_x;
	uint64_t block_count;
};

// T.81 Annex C: code lengths in symbol order, codes counting up within each length
inline void make_codes(const uint8_t bits[16], const uint8_t* symbols, uint32_t* table) {
	uint32_t code = 0, k = 0;
	for (uint32_t length = 1; length <= 16; ++length) {
		for (uint32_t i = 0; i != bits[length - 1]; ++i, ++k, ++code)
			table[symbols[k]] = (length << 16) | code;
		code <<= 1;
	}
}

// the scaled quantisation tables in zigzag order, as DQT stores them; returns 1 for 4:2:0
inline uint32_t make_quant_tables(int quality, uint8_t luma[64], uint8_t chroma[64]) {
	if (quality == 0) quality = 90;
	const uint32_t subsample = quality <= 90 ? 1 : 0;
	quality = quality < 1 ? 1 : (quality > 100 ? 100 : quality);
	const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
	for (int i = 0; i != 64; ++i) {
		const int l = (kLumaQuant[i] * scale + 50) / 100, c = (kChromaQuant[i] * scale + 50) / 100;
		luma[kZigzag[i]] = (uint8_t) (l < 1 ? 1 : (l > 255 ? 255 : l));
		chroma[kZigzag[i]] = (uint8_t) (c < 1 ? 1 : (c > 255 ? 255 : c));
	}
	return subsample;
}

inline void make_params(int quality, uint32_t width, uint32_t height, Params* p) {
	uint8_t quant[2][64];
	p->subsample = make_quant_tables(quality, quant[0], quant[1]);
	float scale[8];
	for (int k = 0; k != 8; ++k) scale[k] = kAanScale[k] * kSqrt8;
	for (int c = 0; c != 2; ++c)
		for (int i = 0; i != 64; ++i) {
			const float q = (float) quant[c][kZigzag[i]];
			const float denominator = q * scale[i >> 3];
			p->reciprocal[c][i] = 1.0f / (denominator * scale[i & 7]);
		}
	for (int c = 0; c != 2; ++c)
		for (int i = 0; i != 256; ++i) p->ac_code[c][i] = 0;
	make_codes(kDcLumaBits, kDcSymbols, p->dc_code[0]);
	make_codes(kDcChromaBits, kDcSymbols, p->dc_code[1]);
	make_codes(kAcLumaBits, kAcLumaSymbols, p->ac_code[0]);
	make_codes(kAcChromaBits, kAcChromaSymbols, p->ac_code[1]);
	for (int i = 0; i != 64; ++i) p->zigzag[i] = kZigzag[i];
	const uint32_t mcu = p->subsample ? 16 : 8;
	p->width = width; p->height = height;
	p->mcus_x = (width + mcu - 1) / mcu;
	p->block_count = (uint64_t) p->mcus_x * ((height + mcu - 1) / mcu) * (p->subsample ? 6 : 3);
}

// SOI, APP0 (JFIF 1.1, 1:1, no thumbnail), DQT (both tables), SOF0, DHT (all four tables), SOS: kHeaderBytes bytes
inline void write_header(int quality, uint32_t width, uint32_t height, uint8_t* out) {
	uint8_t* o = out;
	auto put = [&](uint32_t b) { *o++ = (uint8_t) b; };
	auto put16 = [&](uint32_t v) { put(v >> 8); put(v & 0xFF); };
	auto table = [&](uint32_t id, const uint8_t bits[16], const uint8_t* symbols, uint32_t symbol_count) {
		put(id);
		for (int i = 0; i != 16; ++i) put(bits[i]);
		for (uint32_t i = 0; i != symbol_count; ++i) put(symbols[i]);
	};
	put16(0xFFD8);
	put16(0xFFE0); put16(16); put('J'); put('F'); put('I'); put('F'); put(0); put(1); put(1); put(0); put16(1); put16(1); put(0); put(0);
	uint8_t quant[2][64];
	const uint32_t subsample = make_quant_tables(quality, quant[0], quant[1]);
	put16(0xFFDB); put16(2 + 2 * 65);
	for (int c = 0; c != 2; ++c) { put(c); for (int i = 0; i != 64; ++i) put(quant[c][i]); }
	put16(0xFFC0); put16(17); put(8); put16(height); put16(width); put(3);
	put(1); put(subsample ? 0x22 : 0x11); put(0);
	put(2); put(0x11); put(1);
	put(3); put(0x11); put(1);
	put16(0xFFC4); put16(2 + 2 * (17 + 12) + 2 * (17 + 162));
	table(0x00, kDcLumaBits, kDcSymbols, 12);
	table(0x10, kAcLumaBits, kAcLumaSymbols, 162);
	table(0x01, kDcChromaBits, kDcSymbols, 12);
	table(0x11, kAcChromaBits, kAcChromaSymbols, 162);
	put16(0xFFDA); put16(12); put(3); put(1); put(0x00); put(2); put(0x11); put(3); put(0x11); put(0); put(63); put(0);
}

// ---- per block ------------------------------------------------------------------------------------------------------------------------------

// block b of the stream: component class (0 luminance, 1 chrominance), its MCU, its place in the MCU
struct BlockPlace { uint32_t mcu_x, mcu_y, k, chroma; };
VKR_JPEG_FN BlockPlace place_of(const Params& p, uint64_t b) {
	const uint32_t per_mcu = p.subsample ? 6 : 3;
	const uint64_t mcu = b / per_mcu;
	BlockPlace q;
	q.k = (uint32_t) (b - mcu * per_mcu);
	q.mcu_x = (uint32_t) (mcu % p.mcus_x);
	q.mcu_y = (uint32_t) (mcu / p.mcus_x);
	q.chroma = q.k >= per_mcu - 2;
	return q;
}

// the previous block of the same component in stream order, or -1
VKR_JPEG_FN int64_t predecessor(const Params& p, uint64_t b) {
	const uint32_t per_mcu = p.subsample ? 6 : 3;
	const uint32_t k = (uint32_t) (b % per_mcu);
	if (p.subsample && k >= 1 && k <= 3) return (int64_t) b - 1;     // Y1..Y3 follow Y0..Y2 in the same MCU
	if (b < per_mcu) return -1;
	if (p.subsample && k == 0) return (int64_t) b - 3;               // Y3 of the previous MCU
	return (int64_t) b - per_mcu;
}

VKR_JPEG_FN float luma(float r, float g, float b) { return 0.29900f * r + 0.58700f * g + 0.11400f * b - 128.0f; }
VKR_JPEG_FN float chroma_b(float r, float g, float b) { return -0.16874f * r - 0.33126f * g + 0.50000f * b; }
VKR_JPEG_FN float chroma_r(float r, float g, float b) { return 0.50000f * r - 0.41869f * g - 0.08131f * b; }

// the AAN flow graph on 8 samples s[0], s[stride], ...; outputs scaled by 8 a(k) (columns) or 8 a(k) a(row) after both passes
VKR_JPEG_FN void aan_dct8(float* s, int stride) {
	const float x0 = s[0], x1 = s[stride], x2 = s[2 * stride], x3 = s[3 * stride];
	const float x4 = s[4 * stride], x5 = s[5 * stride], x6 = s[6 * stride], x7 = s[7 * stride];
	const float a0 = x0 + x7, a7 = x0 - x7, a1 = x1 + x6, a6 = x1 - x6;
	const float a2 = x2 + x5, a5 = x2 - x5, a3 = x3 + x4, a4 = x3 - x4;
	// even half
	const float b0 = a0 + a3, b3 = a0 - a3, b1 = a1 + a2, b2 = a1 - a2;
	const float rotated = (b2 + b3) * 0.707106781f;
	s[0] = b0 + b1;
	s[4 * stride] = b0 - b1;
	s[2 * stride] = b3 + rotated;
	s[6 * stride] = b3 - rotated;
	// odd half: the rotation by pi/8 with the shared product, then the butterflies
	const float c4 = a4 + a5, c5 = a5 + a6, c6 = a6 + a7;
	const float shared = (c4 - c6) * 0.382683433f;
	const float r4 = c4 * 0.541196100f + shared;
	const float r6 = c6 * 1.306562965f + shared;
	const float r5 = c5 * 0.707106781f;
	const float d7 = a7 + r5, d5 = a7 - r5;
	s[5 * stride] = d5 + r4;
	s[3 * stride] = d5 - r4;
	s[1 * stride] = d7 + r6;
	s[7 * stride] = d7 - r6;
}

VKR_JPEG_FN uint32_t clamp_index(uint32_t v, uint32_t size) { return v < size ? v : size - 1; }

// block b's quantised coefficients in zigzag order
VKR_JPEG_FN void transform_block(const Params& p, const uint8_t* rgb, uint64_t b, int16_t out[64]) {
	const BlockPlace q = place_of(p, b);
	const uint32_t w = p.width, h = p.height;
	float s[64];
	if (!q.chroma) {
		const uint32_t x0 = q.mcu_x * (p.subsample ? 16 : 8) + (q.k & 1) * 8, y0 = q.mcu_y * (p.subsample ? 16 : 8) + (q.k >> 1) * 8;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
		for (int i = 0; i < 64; ++i) {
			const uint8_t* px = rgb + 3 * ((size_t) clamp_index(y0 + (i >> 3), h) * w + clamp_index(x0 + (i & 7), w));
			s[i] = luma((float) px[0], (float) px[1], (float) px[2]);
		}
	}
	else {
		const bool red = q.k == (p.subsample ? 5u : 2u);
		if (p.subsample) {
			const uint32_t x0 = q.mcu_x * 16, y0 = q.mcu_y * 16;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
			for (int i = 0; i < 64; ++i) {
				float c[4];
				for (int j = 0; j != 4; ++j) {
					const uint8_t* px = rgb + 3 * ((size_t) clamp_index(y0 + 2 * (i >> 3) + (j >> 1), h) * w + clamp_index(x0 + 2 * (i & 7) + (j & 1), w));
					c[j] = red ? chroma_r((float) px[0], (float) px[1], (float) px[2]) : chroma_b((float) px[0], (float) px[1], (float) px[2]);
				}
				s[i] = (c[0] + c[1] + c[2] + c[3]) * 0.25f;
			}
		}
		else {
			const uint32_t x0 = q.mcu_x * 8, y0 = q.mcu_y * 8;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
			for (int i = 0; i < 64; ++i) {
				const uint8_t* px = rgb + 3 * ((size_t) clamp_index(y0 + (i >> 3), h) * w + clamp_index(x0 + (i & 7), w));
				s[i] = red ? chroma_r((float) px[0], (float) px[1], (float) px[2]) : chroma_b((float) px[0], (float) px[1], (float) px[2]);
			}
		}
	}
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
	for (int row = 0; row < 8; ++row) aan_dct8(s + 8 * row, 1);
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
	for (int col = 0; col < 8; ++col) aan_dct8(s + col, 8);
	const float* reciprocal = p.reciprocal[q.chroma];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
	for (int i = 0; i < 64; ++i) {
		const float v = s[i] * reciprocal[i];
		out[p.zigzag[i]] = (int16_t) (int) (v < 0.0f ? v - 0.5f : v + 0.5f);
	}
}

// magnitude category (T.81 F.1.2.1) and the appended bits: v for v > 0, v - 1 in the low bits for v < 0
VKR_JPEG_FN uint32_t category(int v) {
	uint32_t m = (uint32_t) (v < 0 ? -v : v), n = 0;
	while (m) { ++n; m >>= 1; }
	return n;
}
VKR_JPEG_FN uint32_t extra_bits(int v, uint32_t n) { return (uint32_t) (v < 0 ? v - 1 : v) & ((1u << n) - 1u); }

// the codes of block b in order: sink.put(bits, length), length <= 16
template <class Sink>
VKR_JPEG_FN void walk_block(const Params& p, const int16_t* coefficients, int previous_dc, uint32_t chroma, Sink& sink) {
	const int diff = coefficients[0] - previous_dc;
	const uint32_t n = category(diff);
	const uint32_t dc = p.dc_code[chroma][n];
	sink.put(dc & 0xFFFF, dc >> 16);
	if (n) sink.put(extra_bits(diff, n), n);
	const uint32_t* ac = p.ac_code[chroma];
	uint32_t run = 0;
	for (int i = 1; i < 64; ++i) {
		const int v = coefficients[i];
		if (v == 0) { ++run; continue; }
		for (; run >= 16; run -= 16) sink.put(ac[0xF0] & 0xFFFF, ac[0xF0] >> 16);
		const uint32_t size = category(v);
		const uint32_t code = ac[(run << 4) | size];
		sink.put(code & 0xFFFF, code >> 16);
		sink.put(extra_bits(v, size), size);
		run = 0;
	}
	if (run) sink.put(ac[0x00] & 0xFFFF, ac[0x00] >> 16);   // EOB unless coefficient 63 was the last non-zero one
}

struct BitCounter {
	uint32_t bits = 0;
	VKR_JPEG_FN void put(uint32_t, uint32_t length) { bits += length; }
};

VKR_JPEG_FN int previous_dc(const Params& p, const int16_t* coefficients, uint64_t b) {
	const int64_t prev = predecessor(p, b);
	return prev < 0 ? 0 : coefficients[64 * (uint64_t) prev];
}

VKR_JPEG_FN uint32_t block_bits(const Params& p, const int16_t* coefficients, uint64_t b) {
	BitCounter counter;
	walk_block(p, coefficients + 64 * b, previous_dc(p, coefficients, b), place_of(p, b).chroma, counter);
	return counter.bits;
}

VKR_JPEG_FN void or_word(uint32_t* word, uint32_t v) {
#ifdef __CUDA_ARCH__
	atomicOr(word, v);
#else
	*word |= v;
#endif
}

// writes a block's bits from bit offset `position` on into a zeroed word array; the first and the last word are OR-ed, the others stored
struct WordWriter {
	uint32_t* words;
	uint64_t word_index;
	uint32_t word, used;        // pending word, bits of it filled (from bit 31 down)
	bool first;
	VKR_JPEG_FN WordWriter(uint32_t* w, uint64_t position) : words(w), word_index(position >> 5), word(0), used((uint32_t) (position & 31)), first(true) {}
	VKR_JPEG_FN void flush_full() {
		if (first) or_word(words + word_index, word);
		else words[word_index] = word;
		first = false;
		++word_index;
		word = 0;
	}
	VKR_JPEG_FN void put(uint32_t bits, uint32_t length) {
		if (!length) return;
		const uint32_t free = 32 - used;
		if (length < free) { word |= bits << (free - length); used += length; return; }
		const uint32_t rest = length - free;
		word |= bits >> rest;
		flush_full();
		used = rest;
		if (rest) word = bits << (32 - rest);
	}
	VKR_JPEG_FN void finish() { if (used) or_word(words + word_index, word); }
};

// block b's bits at its offset; the last block also pads the stream with 1-bits to a byte boundary
VKR_JPEG_FN void emit_block(const Params& p, const int16_t* coefficients, const uint64_t* offsets, uint64_t b, uint32_t* words) {
	WordWriter writer(words, offsets[b]);
	walk_block(p, coefficients + 64 * b, previous_dc(p, coefficients, b), place_of(p, b).chroma, writer);
	if (b + 1 == p.block_count) {
		const uint32_t pad = (uint32_t) ((8 - (offsets[b + 1] & 7)) & 7);
		writer.put((1u << pad) - 1u, pad);
	}
	writer.finish();
}

// byte i of the padded stream
VKR_JPEG_FN uint8_t stream_byte(const uint32_t* words, uint64_t i) { return (uint8_t) (words[i >> 2] >> (24 - 8 * (i & 3))); }

// stuffing, chunk by chunk: the 0xFF bytes of chunk c, then the chunk copied to out + c * kChunkBytes + (0xFF bytes before it), a 0x00 after each 0xFF
constexpr uint32_t kChunkBytes = 64;
VKR_JPEG_FN uint32_t chunk_ff_count(const uint32_t* words, uint64_t byte_count, uint64_t c) {
	uint32_t n = 0;
	const uint64_t end = (c + 1) * kChunkBytes < byte_count ? (c + 1) * kChunkBytes : byte_count;
	for (uint64_t i = c * kChunkBytes; i < end; ++i) n += stream_byte(words, i) == 0xFF;
	return n;
}
VKR_JPEG_FN void stuff_chunk(const uint32_t* words, uint64_t byte_count, uint64_t c, uint64_t ff_before, uint8_t* out) {
	uint8_t* o = out + c * kChunkBytes + ff_before;
	const uint64_t end = (c + 1) * kChunkBytes < byte_count ? (c + 1) * kChunkBytes : byte_count;
	for (uint64_t i = c * kChunkBytes; i < end; ++i) {
		const uint8_t v = stream_byte(words, i);
		*o++ = v;
		if (v == 0xFF) *o++ = 0;
	}
}

// what an 8-bit UNORM render target stores for a float channel (vkr_quantize_unorm8): round(clamp(x, 0, 1) * 255), NaN -> 0
VKR_JPEG_FN uint8_t unorm8(float x) {
	x = (x > 0.0f) ? ((x < 1.0f) ? x : 1.0f) : 0.0f;
	return (uint8_t) (x * 255.0f + 0.5f);
}

// the refusals both builds share; what names the caller in the message
inline int check_request(const char* what, const void* pixels, uint32_t width, uint32_t height, const void* out, const size_t* out_size) {
	if (!pixels || !out || !out_size) { printf("Failed to %s: no pixels, no output buffer or no size.\n", what); return 1; }
	if (!width || !height || width > kMaxSide || height > kMaxSide) { printf("Failed to %s: a JPEG holds 1 .. %u pixels per side, not %u x %u.\n", what, kMaxSide, width, height); return 1; }
	return 0;
}

} // namespace vkr_jpeg
