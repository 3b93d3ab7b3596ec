/* oracle/vkr_math.h -- TEST INFRASTRUCTURE (CPU oracle), not product code.
 *
 * Elementary fp32 functions of the oracle. GLSL leaves the precision of
 * atan/sin/cos/acos/inversesqrt/normalize implementation-defined (GLSL.std.450,
 * un-pinned driver code, SURVEY 8c); this header pins ONE valid instance of
 * them built only from IEEE-754 correctly-rounded +,-,*,/,sqrt,fma so that the
 * same bits can be produced on x86 (gcc -ffp-contract=off -mfma) and on sm_90a
 * (nvcc -fmad=false, explicit fmaf). The CUDA path carries its OWN
 * implementation of the same definitions (vulkan_renderer_b200/csrc/
 * vkr_device_math.cuh); the two are compared bit-for-bit by tests/.
 *
 * Definitions (the "spec" both sides implement):
 *   rsqrt(x)      = 1.0f / sqrtf(x)
 *   dot3(a,b)     = fma(a.z,b.z, fma(a.y,b.y, a.x*b.x))
 *   dot2(a,b)     = fma(a.y,b.y, a.x*b.x)
 *   cross(a,b).x  = fma(a.y,b.z, -(a.z*b.y))  (cyclic)
 *   normalize(v)  = v * rsqrt(dot(v,v))
 *   M*v (n cols)  = fma chain: ((c0*v0 then fma c1,v1 ...)) in column order
 *   atan(x)       = odd minimax polynomial on [0,1] (9 coefficients in x^2),
 *                   1/x reflection for |x|>1 with a two-term pi/2
 *   sin/cos(x)    = Cody-Waite 3-term reduction by pi/2, Cephes sinf/cosf kernels
 *   acos(x)       = 2*atan(sqrt((1-x)/(1+x)))   for x in [0,1]
 */
#ifndef VKR_ORACLE_MATH_H
#define VKR_ORACLE_MATH_H
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct { float x, y; } v2;
typedef struct { float x, y, z; } v3;

#define VKR_PI 3.1415926535897932384626433832795f
#define VKR_INV_PI 0.31830988618379067153776752674503f
#define VKR_HALF_PI 1.5707963267948966192313216916398f

static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

static inline float vkr_rsqrt(float x) { return 1.0f / sqrtf(x); }
/* GLSL.std.450 FMax/FMin wording: max(x,y) = (x<y)?y:x, min(x,y) = (y<x)?y:x */
static inline float vkr_max(float x, float y) { return (x < y) ? y : x; }
static inline float vkr_min(float x, float y) { return (y < x) ? y : x; }
static inline float vkr_clamp(float x, float lo, float hi) { return vkr_min(vkr_max(x, lo), hi); }

static inline float vkr_atan(float x) {
	float ax = fabsf(x);
	int big = ax > 1.0f;
	float z = big ? (1.0f / ax) : ax;
	float s = z * z;
	float q = 0.002849885728210211f;
	q = fmaf(q, s, -0.016068613156676292f);
	q = fmaf(q, s, 0.042691491544246674f);
	q = fmaf(q, s, -0.07504292577505112f);
	q = fmaf(q, s, 0.10640932619571686f);
	q = fmaf(q, s, -0.14203643798828125f);
	q = fmaf(q, s, 0.1999261975288391f);
	q = fmaf(q, s, -0.3333307206630707f);
	float r = fmaf(z * s, q, z);
	/* pi/2 = 1.57079637050628662109375 (hi) - 4.37113882867379e-8 (lo) */
	if (big) r = (1.57079637050628662109375f - r) + (-4.37113882867379e-8f);
	return (x < 0.0f) ? -r : r;
}

/* Reduces x to r in [-pi/4,pi/4] and quadrant k (x = k*pi/2 + r). Accurate for |x| < ~1e4. */
static inline float vkr_reduce_pio2(float x, int* quadrant) {
	float k = rintf(x * 0.63661977236758134308f);
	float r = fmaf(-k, 1.5707962512969970703125f, x);
	r = fmaf(-k, 7.54978995489188216e-08f, r);
	r = fmaf(-k, 5.39030285815811905e-15f, r);
	*quadrant = (int) k;
	return r;
}
static inline float vkr_sin_kernel(float r) {
	float s = r * r;
	float p = -1.9515295891e-4f;
	p = fmaf(p, s, 8.3321608736e-3f);
	p = fmaf(p, s, -1.6666654611e-1f);
	return fmaf(r * s, p, r);
}
static inline float vkr_cos_kernel(float r) {
	float s = r * r;
	float p = 2.443315711809948e-5f;
	p = fmaf(p, s, -1.388731625493765e-3f);
	p = fmaf(p, s, 4.166664568298827e-2f);
	return fmaf(s * s, p, fmaf(-0.5f, s, 1.0f));
}
static inline float vkr_sin(float x) {
	int q; float r = vkr_reduce_pio2(x, &q);
	float v = (q & 1) ? vkr_cos_kernel(r) : vkr_sin_kernel(r);
	return (q & 2) ? -v : v;
}
static inline float vkr_cos(float x) {
	int q; float r = vkr_reduce_pio2(x, &q);
	float v = (q & 1) ? vkr_sin_kernel(r) : vkr_cos_kernel(r);
	return ((q + 1) & 2) ? -v : v;
}
/* acos for x in [0,1] (callers clamp first, ltc_utility.glsl:61) */
static inline float vkr_acos01(float x) {
	return 2.0f * vkr_atan(sqrtf((1.0f - x) / (1.0f + x)));
}

/* two-argument atan (quadrant-corrected, built on vkr_atan) and acos on [-1,1]: used by the related-work samplers
   (cubic_solver.glsl:52, polygon_sampling_related_work.glsl:148-151, 764-768) */
static inline float vkr_atan2(float y, float x) {
	if (x > 0.0f) return vkr_atan(y / x);
	if (x < 0.0f) return (y >= 0.0f) ? vkr_atan(y / x) + VKR_PI : vkr_atan(y / x) - VKR_PI;
	return (y > 0.0f) ? VKR_HALF_PI : ((y < 0.0f) ? -VKR_HALF_PI : 0.0f);
}
static inline float vkr_acos(float x) { return (x >= 0.0f) ? vkr_acos01(vkr_min(x, 1.0f)) : VKR_PI - vkr_acos01(vkr_min(-x, 1.0f)); }

/* ---- output stage (srgb_utility.glsl, shading_pass.frag.glsl:871-892). GLSL leaves the precision of pow to the driver;
   this is the contract both sides implement: pow(x, y) = exp2(y * log2(x)) for x > 0, 0 for x <= 0, every step in fp32. */
static inline float vkr_log2(float x) { /* x > 0, normal; fdlibm's logf kernel, then one fma by 1/ln 2 */
	uint32_t u = f2u(x) - 0x3f3504f3u;                        /* mantissa in [sqrt(1/2), sqrt(2)) */
	const float e = (float) ((int32_t) u >> 23);
	const float f = u2f((u & 0x007fffffu) + 0x3f3504f3u) - 1.0f;
	const float s = f / (2.0f + f);
	const float z = s * s, w = z * z;
	const float t1 = w * fmaf(w, 0.24279078841f, 0.40000972152f);
	const float t2 = z * fmaf(w, 0.28498786688f, 0.66666662693f);
	const float hfsq = 0.5f * f * f;
	const float ln = f - (hfsq - s * (hfsq + (t2 + t1)));
	return fmaf(ln, 1.44269502162933349609375f, e);
}
static inline float vkr_exp2(float x) { /* x in [-126, 127]; smaller x gives 0 */
	if (!(x >= -126.0f)) return 0.0f;
	const float n = floorf(x + 0.5f);
	const float r = x - n;                                        /* [-0.5, 0.5] */
	float p = 1.52527338e-5f;
	p = fmaf(p, r, 1.54035304e-4f);
	p = fmaf(p, r, 1.33335581e-3f);
	p = fmaf(p, r, 9.61812911e-3f);
	p = fmaf(p, r, 5.55041087e-2f);
	p = fmaf(p, r, 2.40226507e-1f);
	p = fmaf(p, r, 6.93147181e-1f);
	p = fmaf(p, r, 1.0f);
	return p * u2f((uint32_t) ((int32_t) n + 127) << 23);
}
static inline float vkr_pow(float x, float y) { return (x > 0.0f) ? vkr_exp2(y * vkr_log2(x)) : 0.0f; }
/* srgb_utility.glsl:21-26 and 44-49 */
static inline float vkr_linear_to_srgb(float c) {
	c = vkr_clamp(c, 0.0f, 1.0f);
	return (c <= 0.0031308f) ? (12.92f * c) : (1.055f * vkr_pow(c, 1.0f / 2.4f) - 0.055f);
}
static inline float vkr_srgb_to_linear(float c) {
	c = vkr_clamp(c, 0.0f, 1.0f);
	return (c <= 0.04045f) ? ((1.0f / 12.92f) * c) : vkr_pow(fmaf(c, 1.0f / 1.055f, 0.055f / 1.055f), 2.4f);
}
/* IEEE binary32 -> binary16, round to nearest even (packHalf2x16) */
static inline uint32_t vkr_float_to_half(float f) {
	const uint32_t u = f2u(f), sign = (u >> 16) & 0x8000u, a = u & 0x7fffffffu;
	if (a > 0x7f800000u) return sign | 0x7e00u;               /* NaN */
	if (a >= 0x47800000u) return sign | 0x7c00u;              /* >= 65536 (and inf): 65520 <= |f| rounds to inf below */
	if (a < 0x33000001u) return sign;                         /* <= 2^-25: rounds to zero */
	uint32_t exponent = a >> 23, mantissa = (a & 0x007fffffu) | 0x00800000u;
	uint32_t shift, half;
	if (exponent < 113u) { shift = 126u - exponent; half = 0u; }           /* subnormal half */
	else { shift = 13u; half = (exponent - 112u) << 10; mantissa &= 0x007fffffu; }
	const uint32_t kept = mantissa >> shift, rest = mantissa & ((1u << shift) - 1u), halfway = 1u << (shift - 1u);
	half += kept;
	if (rest > halfway || (rest == halfway && (half & 1u))) ++half;        /* carries into the exponent (and to inf) correctly */
	return sign | half;
}
static inline uint32_t vkr_pack_half_2x16(float x, float y) { return vkr_float_to_half(x) | (vkr_float_to_half(y) << 16); }

static inline v2 mk2(float x, float y) { v2 r = {x, y}; return r; }
static inline v3 mk3(float x, float y, float z) { v3 r = {x, y, z}; return r; }
static inline float dot2(v2 a, v2 b) { return fmaf(a.y, b.y, a.x * b.x); }
static inline float dot3(v3 a, v3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
static inline v3 cross3(v3 a, v3 b) {
	return mk3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x)));
}
static inline v3 scale3(v3 a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
static inline v2 scale2(v2 a, float s) { return mk2(a.x * s, a.y * s); }
static inline v3 add3(v3 a, v3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline v3 sub3(v3 a, v3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline v2 add2(v2 a, v2 b) { return mk2(a.x + b.x, a.y + b.y); }
static inline v2 sub2(v2 a, v2 b) { return mk2(a.x - b.x, a.y - b.y); }
static inline v3 normalize3(v3 a) { return scale3(a, vkr_rsqrt(dot3(a, a))); }
static inline v2 normalize2(v2 a) { return scale2(a, vkr_rsqrt(dot2(a, a))); }
/* det of the 3x3 matrix with COLUMNS a,b,c = dot(a, cross(b,c)) */
static inline float det3(v3 a, v3 b, v3 c) { return dot3(a, cross3(b, c)); }

#endif
