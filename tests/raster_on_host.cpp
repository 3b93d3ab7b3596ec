// tests/raster_on_host.cpp -- TEST INFRASTRUCTURE: the rasteriser's per-triangle and per-pixel functions (csrc/vkr_raster.cuh) compiled for the CPU,
// next to the brute-force oracle (tests/raster_oracle.h). The kernels' atomicMin becomes a plain min, their chunking a loop over each polygon's box.
// Built by __graft_entry__.build() into tests/build/libraster_on_host.so; tests/test_raster_on_host.py and the GPU tests call it. Nothing in the
// product links against it.
#include <cmath>
#include <cstdint>
#include <cstring>

#define VKR_DEVICE_CODE_ON_HOST 1
#define VKR_DEV inline
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }

// the CUDA vector types the headers use, laid out as on the device
struct float4 { float x, y, z, w; };
struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
struct ushort4 { uint16_t x, y, z, w; };
typedef int cudaError_t;
typedef void* cudaStream_t;
static inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
template <class T> static inline T __ldg(const T* p) { return *p; }
// declared so that the trace header parses; the functions used here never call them
unsigned __ballot_sync(unsigned, int); int __any_sync(unsigned, int); int __all_sync(unsigned, int); void __syncwarp(unsigned); int __popc(unsigned); int __ffs(unsigned);
void __nanosleep(unsigned); unsigned __activemask(); int __shfl_sync(unsigned, int, int); size_t __cvta_generic_to_shared(const void*);
static inline int __clz(int x) { return x ? __builtin_clz((unsigned) x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long) x) : 64; }

#include <algorithm>
using std::min; using std::max;
#include "vkr_raster.cuh"
#include "raster_oracle.h"
#include <vector>

using namespace vkr;

// The kernels' work for every triangle in turn: keys[pixel] = min over fragments (depth-test keys), fragments per pixel and per triangle
static void rasterize(uint32_t width, uint32_t height, const void* constants, const uint32_t* quantized_positions, uint64_t triangle_count,
	std::vector<unsigned long long>& keys, uint32_t* pixel_fragments, uint32_t* triangle_fragments)
{
	keys.assign((size_t) width * height, kRasterClearKey);
	const uint2* q = reinterpret_cast<const uint2*>(quantized_positions);
	for (uint64_t prim = 0; prim != triangle_count; ++prim) {
		raster_polygon poly;
		raster_polygon_of(q, (const unsigned char*) constants, (uint32_t) prim, (int) width, (int) height, poly);
		raster_triangle tris[kRasterMaxFan];
		int box[4];
		const int fans = raster_fans_of(poly, (int) width, (int) height, tris, box);
		uint32_t count = 0;
		for (int y = box[1]; y <= box[3]; ++y) for (int x = box[0]; x <= box[2]; ++x) {
			const unsigned long long key = raster_polygon_fragment(tris, fans, x, y, (uint32_t) prim);
			if (key == kRasterClearKey) continue;
			const size_t pixel = (size_t) y * width + x;
			keys[pixel] = std::min(keys[pixel], key);
			if (pixel_fragments) ++pixel_fragments[pixel];
			++count;
		}
		if (triangle_fragments) triangle_fragments[prim] = count;
	}
}

// what vkr_rasterize_visibility writes; depth may be null
extern "C" void vkr_raster_on_host_visibility(uint32_t width, uint32_t height, const void* constants, const uint32_t* quantized_positions, uint64_t triangle_count,
	uint32_t* out_visibility, float* out_depth)
{
	std::vector<unsigned long long> keys;
	rasterize(width, height, constants, quantized_positions, triangle_count, keys, nullptr, nullptr);
	for (size_t i = 0; i != keys.size(); ++i) {
		const bool drawn = keys[i] != kRasterClearKey;
		out_visibility[i] = drawn ? (uint32_t) keys[i] : 0xFFFFFFFFu;
		if (out_depth) out_depth[i] = drawn ? __uint_as_float((uint32_t) (keys[i] >> 32)) : 1.0f;
	}
}

// the depth test off: fragments per pixel (uint32 per pixel, zeroed by the caller) and per triangle
extern "C" void vkr_raster_on_host_fragments(uint32_t width, uint32_t height, const void* constants, const uint32_t* quantized_positions, uint64_t triangle_count,
	uint32_t* out_pixel_fragments, uint32_t* out_triangle_fragments)
{
	std::vector<unsigned long long> keys;
	rasterize(width, height, constants, quantized_positions, triangle_count, keys, out_pixel_fragments, out_triangle_fragments);
}

// the oracle: visibility and depth; out_fragments (may be null) = fragments per pixel with the depth test off
extern "C" void vkr_raster_oracle_visibility(uint32_t width, uint32_t height, const void* constants, const uint32_t* quantized_positions, uint64_t triangle_count,
	uint32_t* out_visibility, float* out_depth, uint32_t* out_fragments)
{
	ro_rasterize(width, height, (const unsigned char*) constants, quantized_positions, triangle_count, out_visibility, out_depth, out_fragments);
}
