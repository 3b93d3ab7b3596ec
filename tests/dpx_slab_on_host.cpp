// tests/dpx_slab_on_host.cpp -- TEST INFRASTRUCTURE: the slab test of the trace warps (vkr_trace.cuh: make_clamped_slabs() + ray_box_pair<true>, signed
// integer min / max on the float bits) compiled for the CPU next to the fmaxf form it replaced, for tests/test_dpx_slab_test.py.
// The host build of vkr_trace.cuh runs plain C++ in place of __vimax3_s32 / __vimin3_s32 with the same integer semantics.
// Built by __graft_entry__.build() into tests/build/libdpx_slab_on_host.so. Nothing in the product links against it.
#include <cmath>
#include <cstdint>
#include <cstring>

#define VKR_DEVICE_CODE_ON_HOST 1
#define VKR_DEV inline
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
struct float4 { float x, y, z, w; };
template <class T> static inline T __ldg(const T* p) { return *p; }

#include "vkr_trace.cuh"

using namespace vkr;

// One interleaved pair per ray (rays = {ox, oy, oz, dx, dy, dz, tmin, tmax}, pairs16 as interleave_node_pair() writes them), three ways:
//   0: the fmaxf pair test on the unclamped set-up (make_slabs<false>, what the trace warps ran before; NaN slab distances for zero components)
//   1: the integer pair test on the clamped set-up (make_clamped_slabs + ray_box_pair<true>, what the trace warps run now)
//   2: the fmaxf pair test on the clamped set-up
// hits[6 * i + 2 * k + c] = child c hit by way k, t_near[6 * i + 2 * k + c] its entry distance.
extern "C" void vkr_dpx_pair_tests(uint32_t n, const float* rays, const float* pairs16, uint8_t* hits, float* t_near) {
	for (uint32_t i = 0; i != n; ++i) {
		const float* r = rays + 8 * (size_t) i;
		const float* w = pairs16 + 16 * (size_t) i;
		const f3 o = make3(r[0], r[1], r[2]), d = make3(r[3], r[4], r[5]);
		const float a[8] = { w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7] }, b[4] = { w[8], w[9], w[10], w[11] };
		const ray_slabs plain = make_slabs<false>(o, d), clamped = make_clamped_slabs(o, d);
		bool h[6]; float t[6];
		ray_box_pair<false>(a, b, plain, r[6], r[7], &h[0], &h[1], &t[0], &t[1]);
		ray_box_pair<true>(a, b, clamped, r[6], r[7], &h[2], &h[3], &t[2], &t[3]);
		ray_box_pair<false>(a, b, clamped, r[6], r[7], &h[4], &h[5], &t[4], &t[5]);
		for (int k = 0; k != 6; ++k) { hits[6 * (size_t) i + k] = h[k] ? 1 : 0; t_near[6 * (size_t) i + k] = t[k]; }
	}
}

// The per-thread any-hit query over the interleaved pairs of a tree (node pairs in the plain layout, interleaved here) in both forms:
// occluded_interleaved<false> (fmaxf, guarded set-up) and occluded_interleaved<true> (the trace warps' form). Answers and pairs visited per ray.
extern "C" void vkr_dpx_trace_interleaved(const float* nodes, uint64_t pair_count, const float* tris, uint32_t ray_count, const float* rays, uint8_t* out_fmax,
	uint8_t* out_dpx, uint32_t* visits_fmax, uint32_t* visits_dpx)
{
	float* pairs16 = new float[16 * pair_count];
	for (uint64_t i = 0; i != pair_count; ++i) interleave_node_pair(reinterpret_cast<const float4*>(nodes) + 4 * i, pairs16 + 16 * i);
	const float4* t4 = reinterpret_cast<const float4*>(tris);
	int stack[kMaxStackDepth + 2];
	for (uint32_t i = 0; i != ray_count; ++i) {
		const float* r = rays + 8 * (size_t) i;
		const f3 o = make3(r[0], r[1], r[2]), d = make3(r[3], r[4], r[5]);
		int v0 = 0, v1 = 0;
		out_fmax[i] = occluded_interleaved<false>(pairs16, t4, o, d, r[6], r[7], stack, 1, &v0) ? 1 : 0;
		out_dpx[i] = occluded_interleaved<true>(pairs16, t4, o, d, r[6], r[7], stack, 1, &v1) ? 1 : 0;
		visits_fmax[i] = (uint32_t) v0; visits_dpx[i] = (uint32_t) v1;
	}
	delete[] pairs16;
}
