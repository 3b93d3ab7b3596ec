// vkr_raster.cuh -- the reference's subpass 0 (src/main.c:1421-1427, visibility_pass.{vert,frag}.glsl) as a rasteriser: back-face culling
// (frontFace = COUNTER_CLOCKWISE), clipping to 0 <= z <= w, one sample at the pixel centre with the top-left rule, and a LESS depth test in
// draw order against a D32_SFLOAT buffer cleared to 1.0. DESIGN.md §5 "Rasterised visibility" states every choice Vulkan leaves open.
//
// Per-triangle and per-pixel functions without warp-level operations: csrc/vkr_raster.cu wraps them into kernels, tests/raster_on_host.cpp
// runs them on the CPU against the brute-force oracle (tests/raster_oracle.h). Integer edge functions, fp64 clipping and depth; compile with -fmad=false.
#pragma once
#include "vkr_gbuffer.cuh"

namespace vkr {

constexpr int kSubPixelBits = 8;                          // NVIDIA's VkPhysicalDeviceLimits::subPixelPrecisionBits
constexpr int kSubPixelScale = 1 << kSubPixelBits;
// Guard band: polygons are also clipped to |x|, |y| <= G w. With at most kRasterMaxDimension pixels per side, snapped coordinates stay below
// (G + 1) / 2 * 2^15 * 2^8 < 2^31 and a 2x2 edge product below 2 (G 2^23)^2 = 2^61 (DESIGN.md §5)
constexpr double kGuardBand = 128.0;
constexpr uint32_t kRasterMaxDimension = 32768;
constexpr int kRasterClipPlanes = 6;
constexpr int kRasterMaxPolygon = 3 + kRasterClipPlanes;  // Sutherland-Hodgman adds at most one vertex per plane
constexpr int kRasterMaxFan = kRasterMaxPolygon - 2;
constexpr unsigned long long kRasterClearKey = ~0ull;     // no fragment: resolves to 0xFFFFFFFF and depth 1.0
enum { G_OFF_WORLD_TO_PROJECTION = 32 };                  // std140 row_major mat4 (shared_constants.glsl:20-26)

struct raster_vertex { double x, y, z, w; };

// one front-facing fan triangle after snapping, its vertices in fan order (first, i, i + 1)
struct raster_triangle {
	int32_t X[3], Y[3];      // framebuffer coordinates in 1/256 pixel
	double z[3];             // z_f = z / w
	long long area;          // -c > 0 (raster_setup_fan)
	int x0, y0, x1, y1;      // pixel bounding box on the screen, inclusive; empty if x0 > x1 or y0 > y1
};

VKR_DEV long long raster_round_even(double v) {
#ifdef __CUDA_ARCH__
	return __double2ll_rn(v);
#else
	return llrint(v);        // the default rounding mode, to nearest even
#endif
}

// vertex stage (visibility_pass.vert.glsl:27-33): the shader's decode, then clip = W2P * (p, 1) as an fma chain over the columns
VKR_DEV raster_vertex raster_transform(uint2 q, const unsigned char* cb) {
	const f3 p = decode_position(q, cb);
	float c[4];
#pragma unroll
	for (int i = 0; i != 4; ++i) {
		const int row = G_OFF_WORLD_TO_PROJECTION + 16 * i;
		c[i] = fmaf(gldf(cb, row + 12), 1.0f, fmaf(gldf(cb, row + 8), p.z, fmaf(gldf(cb, row + 4), p.y, gldf(cb, row) * p.x)));
	}
	raster_vertex v; v.x = c[0]; v.y = c[1]; v.z = c[2]; v.w = c[3];
	return v;
}

// signed distance to clip plane k; inside is >= 0. Order: z >= 0, z <= w, x >= -G w, x <= G w, y >= -G w, y <= G w
VKR_DEV double raster_plane_distance(const raster_vertex& v, int k) {
	switch (k) {
	case 0: return v.z;
	case 1: return v.w - v.z;
	case 2: return kGuardBand * v.w + v.x;
	case 3: return kGuardBand * v.w - v.x;
	case 4: return kGuardBand * v.w + v.y;
	default: return kGuardBand * v.w - v.y;
	}
}

// the point where the edge from the inside vertex to the outside one crosses the plane, always computed from the inside vertex so that two
// triangles sharing the edge get the same point
VKR_DEV raster_vertex raster_intersect(const raster_vertex& in, const raster_vertex& out, double d_in, double d_out) {
	const double t = d_in / (d_in - d_out);
	raster_vertex r;
	r.x = in.x + t * (out.x - in.x); r.y = in.y + t * (out.y - in.y); r.z = in.z + t * (out.z - in.z); r.w = in.w + t * (out.w - in.w);
	return r;
}

// 0 = entirely outside one plane, 1 = inside all planes, 2 = needs clipping. A NaN distance counts as outside.
VKR_DEV int raster_classify(const raster_vertex* v) {
	bool crossing = false;
	for (int k = 0; k != kRasterClipPlanes; ++k) {
		const bool i0 = raster_plane_distance(v[0], k) >= 0.0, i1 = raster_plane_distance(v[1], k) >= 0.0, i2 = raster_plane_distance(v[2], k) >= 0.0;
		if (!i0 && !i1 && !i2) return 0;
		crossing = crossing || !(i0 && i1 && i2);
	}
	return crossing ? 2 : 1;
}

// Sutherland-Hodgman over the six planes in order; v holds kRasterMaxPolygon vertices, the first n are the polygon. Returns the new count.
VKR_DEV int raster_clip(raster_vertex* v, int n) {
	raster_vertex out[kRasterMaxPolygon];
	for (int k = 0; k != kRasterClipPlanes && n != 0; ++k) {
		int m = 0;
		for (int i = 0; i != n; ++i) {
			const raster_vertex& cur = v[i];
			const raster_vertex& prev = v[(i == 0) ? n - 1 : i - 1];
			const double dc = raster_plane_distance(cur, k), dp = raster_plane_distance(prev, k);
			const bool ic = dc >= 0.0, ip = dp >= 0.0;
			if (ic != ip) out[m++] = ip ? raster_intersect(prev, cur, dp, dc) : raster_intersect(cur, prev, dc, dp);
			if (ic) out[m++] = cur;
		}
		for (int i = 0; i != m; ++i) v[i] = out[i];
		n = m;
	}
	return n;
}

// viewport transform and snapping of a clipped polygon; false if a vertex has w <= 0 (only a polygon that degenerates to the eye point can)
VKR_DEV bool raster_snap(const raster_vertex* v, int n, int width, int height, int32_t* X, int32_t* Y, double* z) {
	for (int i = 0; i != n; ++i) {
		if (!(v[i].w > 0.0)) return false;
		X[i] = (int32_t) raster_round_even(((v[i].x / v[i].w * 0.5 + 0.5) * (double) width) * (double) kSubPixelScale);
		Y[i] = (int32_t) raster_round_even(((v[i].y / v[i].w * 0.5 + 0.5) * (double) height) * (double) kSubPixelScale);
		z[i] = v[i].z / v[i].w;
	}
	return true;
}

VKR_DEV long long floor_div_subpixel(long long v) { return v >> kSubPixelBits; }   // arithmetic shift: floor

// fan triangle (0, i, i + 1) of a snapped polygon: false if it is back-facing or has zero area (Vulkan's a <= 0 with frontFace = CCW) or covers
// no pixel centre of the screen's bounding box
VKR_DEV bool raster_setup_fan(const int32_t* X, const int32_t* Y, const double* z, int i, int width, int height, raster_triangle& t) {
	const long long ex1 = (long long) X[i] - X[0], ey1 = (long long) Y[i] - Y[0], ex2 = (long long) X[i + 1] - X[0], ey2 = (long long) Y[i + 1] - Y[0];
	const long long c = ex1 * ey2 - ex2 * ey1;       // = -2a in Vulkan's terms (framebuffer y points down)
	if (c >= 0) return false;
	t.X[0] = X[0]; t.Y[0] = Y[0]; t.z[0] = z[0];
	t.X[1] = X[i]; t.Y[1] = Y[i]; t.z[1] = z[i];
	t.X[2] = X[i + 1]; t.Y[2] = Y[i + 1]; t.z[2] = z[i + 1];
	t.area = -c;
	const long long lo_x = min(t.X[0], min(t.X[1], t.X[2])), hi_x = max(t.X[0], max(t.X[1], t.X[2]));
	const long long lo_y = min(t.Y[0], min(t.Y[1], t.Y[2])), hi_y = max(t.Y[0], max(t.Y[1], t.Y[2]));
	const long long half = kSubPixelScale / 2;
	// pixel x has its centre at 256 x + 128: the first centre >= lo and the last <= hi
	t.x0 = (int) max(-floor_div_subpixel(half - lo_x), 0ll); t.x1 = (int) min(floor_div_subpixel(hi_x - half), (long long) width - 1);
	t.y0 = (int) max(-floor_div_subpixel(half - lo_y), 0ll); t.y1 = (int) min(floor_div_subpixel(hi_y - half), (long long) height - 1);
	return t.x0 <= t.x1 && t.y0 <= t.y1;
}

// edge function of a -> b at p: (b - a) x (p - a). A front-facing triangle has c < 0 (raster_setup_fan), so the edge functions of its edges
// are negative inside; the reversed edge b -> a gives the positive value.
VKR_DEV long long raster_edge(int32_t xa, int32_t ya, int32_t xb, int32_t yb, long long px, long long py) {
	return ((long long) xb - xa) * (py - ya) - ((long long) yb - ya) * (px - xa);
}

// top-left rule with y pointing down, for the reversed edge a -> b (inside on its positive side): a top edge is horizontal with the inside below
// it, a left edge has the inside to its right
VKR_DEV bool raster_owns_zero(int32_t xa, int32_t ya, int32_t xb, int32_t yb) { return yb < ya || (yb == ya && xb > xa); }

// the fragment of triangle t at pixel (x, y) as a depth-test key (depth bits << 32 | primitive), or kRasterClearKey if there is none or its depth
// is not LESS than the clear value 1.0
VKR_DEV unsigned long long raster_fragment(const raster_triangle& t, int x, int y, uint32_t primitive) {
	const long long px = (long long) x * kSubPixelScale + kSubPixelScale / 2, py = (long long) y * kSubPixelScale + kSubPixelScale / 2;
	// w_k > 0 inside: the weight of vertex k, the edge function of the opposite edge reversed
	const long long w0 = raster_edge(t.X[2], t.Y[2], t.X[1], t.Y[1], px, py);
	const long long w1 = raster_edge(t.X[0], t.Y[0], t.X[2], t.Y[2], px, py);
	const long long w2 = raster_edge(t.X[1], t.Y[1], t.X[0], t.Y[0], px, py);
	if (w0 < 0 || (w0 == 0 && !raster_owns_zero(t.X[2], t.Y[2], t.X[1], t.Y[1]))) return kRasterClearKey;
	if (w1 < 0 || (w1 == 0 && !raster_owns_zero(t.X[0], t.Y[0], t.X[2], t.Y[2]))) return kRasterClearKey;
	if (w2 < 0 || (w2 == 0 && !raster_owns_zero(t.X[1], t.Y[1], t.X[0], t.Y[0]))) return kRasterClearKey;
	// screen-space linear depth: fp64 weights from the integer edge functions, one rounding to binary32, clamp to [0, 1] (-0.0 and NaN -> +0.0)
	float depth = (float) (((double) w0 * t.z[0] + (double) w1 * t.z[1] + (double) w2 * t.z[2]) / (double) t.area);
	if (!(depth > 0.0f)) depth = 0.0f;
	if (!(depth < 1.0f)) return kRasterClearKey;    // LESS against the clear value, also for depths clamped to 1.0
	return ((unsigned long long) __float_as_uint(depth) << 32) | primitive;
}

// clipped, snapped polygon of one triangle of the visibility draw
struct raster_polygon {
	int count;                       // 0: nothing to rasterise
	int32_t X[kRasterMaxPolygon], Y[kRasterMaxPolygon];
	double z[kRasterMaxPolygon];
};

VKR_DEV void raster_polygon_of(const uint2* quantized_positions, const unsigned char* cb, uint32_t primitive, int width, int height, raster_polygon& poly) {
	raster_vertex v[kRasterMaxPolygon];
#pragma unroll
	for (int i = 0; i != 3; ++i) v[i] = raster_transform(__ldg(quantized_positions + 3 * (size_t) primitive + i), cb);
	poly.count = 0;
	const int cls = raster_classify(v);
	if (cls == 0) return;
	const int n = (cls == 1) ? 3 : raster_clip(v, 3);
	if (n < 3 || !raster_snap(v, n, width, height, poly.X, poly.Y, poly.z)) return;
	poly.count = n;
}

// the front-facing fan triangles of a polygon that cover a pixel centre's bounding box on the screen, and the union of their boxes
// {x0, y0, x1, y1}; returns their number
VKR_DEV int raster_fans_of(const raster_polygon& poly, int width, int height, raster_triangle* tris, int* box) {
	int count = 0;
	box[0] = width; box[1] = height; box[2] = -1; box[3] = -1;
	for (int i = 1; i + 1 < poly.count; ++i) {
		raster_triangle& t = tris[count];
		if (!raster_setup_fan(poly.X, poly.Y, poly.z, i, width, height, t)) continue;
		box[0] = min(box[0], t.x0); box[1] = min(box[1], t.y0); box[2] = max(box[2], t.x1); box[3] = max(box[3], t.y1);
		++count;
	}
	return count;
}

// the depth-test key of a polygon's fragment at pixel (x, y): the least over its fan triangles (at most one covers the pixel centre)
VKR_DEV unsigned long long raster_polygon_fragment(const raster_triangle* tris, int count, int x, int y, uint32_t primitive) {
	unsigned long long key = kRasterClearKey;
	for (int f = 0; f != count; ++f) {
		const raster_triangle& t = tris[f];
		if (x < t.x0 || x > t.x1 || y < t.y0 || y > t.y1) continue;
		const unsigned long long k = raster_fragment(t, x, y, primitive);
		key = (k < key) ? k : key;
	}
	return key;
}

} // namespace vkr
