/* tests/raster_oracle.h -- TEST INFRASTRUCTURE: brute-force restatement of the rasterised visibility buffer (DESIGN.md §5 "Rasterised visibility"),
 * written from Vulkan's rules rather than from csrc/vkr_raster.cuh. Plain C (gcc's __int128 for exact edge functions).
 *
 * For each triangle in draw order: decode, transform, Sutherland-Hodgman against the six planes, viewport transform and snapping, fan. Each
 * fan triangle is front-facing if Vulkan's signed area a = -1/2 sum(x_i y_(i+1) - x_(i+1) y_i) is positive (frontFace = COUNTER_CLOCKWISE).
 * Then, for every pixel of the screen and every front-facing fan triangle: the pixel centre is covered if it is strictly inside, or on an
 * edge that is a top edge (horizontal, the third vertex below it) or a left edge (not horizontal, the third vertex to its right); its depth is
 * z_f interpolated linearly in screen space, rounded to binary32 and clamped to [0, 1]; it is stored if it is LESS than the stored depth,
 * which starts at 1.0. Slow and simple. tests/raster_on_host.cpp exports it. */
#ifndef VKR_RASTER_ORACLE_H
#define VKR_RASTER_ORACLE_H
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define RO_SUBPIXEL 256.0       /* 8 sub-pixel bits */
#define RO_GUARD_BAND 128.0
#define RO_MAX_POLYGON 9

typedef struct { double x, y, z, w; } ro_vertex;
typedef struct { int64_t X[3], Y[3]; double z[3]; uint32_t primitive; } ro_triangle;

static float ro_float(const unsigned char* constants, int offset) { float f; memcpy(&f, constants + offset, 4); return f; }

/* mesh_quantization.glsl: 21 bits per coordinate, dequantised with fma (factor at byte 0, summand at byte 16), then W2P (byte 32, row-major)
   times (p, 1), accumulated over the columns with fma */
static ro_vertex ro_vertex_stage(const uint32_t* q, const unsigned char* constants) {
	const uint32_t bits[3] = { q[0] & 0x1FFFFFu, (q[0] >> 21) | ((q[1] & 0x3FFu) << 11), (q[1] >> 10) & 0x1FFFFFu };
	float p[3], c[4];
	int i;
	for (i = 0; i < 3; ++i) p[i] = fmaf((float) bits[i], ro_float(constants, 4 * i), ro_float(constants, 16 + 4 * i));
	for (i = 0; i < 4; ++i) {
		const int row = 32 + 16 * i;
		c[i] = ro_float(constants, row) * p[0];
		c[i] = fmaf(ro_float(constants, row + 4), p[1], c[i]);
		c[i] = fmaf(ro_float(constants, row + 8), p[2], c[i]);
		c[i] = fmaf(ro_float(constants, row + 12), 1.0f, c[i]);
	}
	{ ro_vertex v; v.x = c[0]; v.y = c[1]; v.z = c[2]; v.w = c[3]; return v; }
}

/* the clip volume 0 <= z <= w and the guard band |x|, |y| <= G w, one plane after the other */
static double ro_inside(const ro_vertex* v, int plane) {
	if (plane == 0) return v->z;
	if (plane == 1) return v->w - v->z;
	if (plane == 2) return RO_GUARD_BAND * v->w + v->x;
	if (plane == 3) return RO_GUARD_BAND * v->w - v->x;
	if (plane == 4) return RO_GUARD_BAND * v->w + v->y;
	return RO_GUARD_BAND * v->w - v->y;
}

static int ro_clip(ro_vertex* poly, int n) {
	int plane, i;
	for (plane = 0; plane < 6; ++plane) {
		ro_vertex out[RO_MAX_POLYGON];
		int m = 0;
		for (i = 0; i < n; ++i) {
			const ro_vertex a = poly[(i + n - 1) % n], b = poly[i];
			const double da = ro_inside(&a, plane), db = ro_inside(&b, plane);
			if ((da >= 0.0) != (db >= 0.0)) {
				/* interpolate from the vertex inside towards the one outside */
				const ro_vertex in = (da >= 0.0) ? a : b, outside = (da >= 0.0) ? b : a;
				const double d_in = (da >= 0.0) ? da : db, d_out = (da >= 0.0) ? db : da;
				const double t = d_in / (d_in - d_out);
				ro_vertex r;
				r.x = in.x + t * (outside.x - in.x); r.y = in.y + t * (outside.y - in.y); r.z = in.z + t * (outside.z - in.z); r.w = in.w + t * (outside.w - in.w);
				out[m++] = r;
			}
			if (db >= 0.0) out[m++] = b;
		}
		memcpy(poly, out, sizeof(ro_vertex) * (size_t) m);
		n = m;
		if (n == 0) return 0;
	}
	return n;
}

/* all front-facing fan triangles of the draw, in draw order; returns their number (tris holds 7 per triangle) */
static size_t ro_primitives(uint32_t width, uint32_t height, const unsigned char* constants, const uint32_t* quantized_positions, uint64_t triangle_count, ro_triangle* tris) {
	size_t count = 0;
	uint64_t t;
	for (t = 0; t < triangle_count; ++t) {
		ro_vertex poly[RO_MAX_POLYGON];
		int64_t X[RO_MAX_POLYGON], Y[RO_MAX_POLYGON];
		double z[RO_MAX_POLYGON];
		int n, i, ok = 1;
		for (i = 0; i < 3; ++i) poly[i] = ro_vertex_stage(quantized_positions + 2 * (3 * t + i), constants);
		n = ro_clip(poly, 3);
		for (i = 0; i < n; ++i) {
			if (!(poly[i].w > 0.0)) { ok = 0; break; }
			X[i] = llrint(((poly[i].x / poly[i].w * 0.5 + 0.5) * (double) width) * RO_SUBPIXEL);
			Y[i] = llrint(((poly[i].y / poly[i].w * 0.5 + 0.5) * (double) height) * RO_SUBPIXEL);
			z[i] = poly[i].z / poly[i].w;
		}
		if (!ok) continue;
		for (i = 1; i + 1 < n; ++i) {
			const int k[3] = { 0, i, i + 1 };
			__int128 twice_area_neg = 0;   /* sum x_i y_(i+1) - x_(i+1) y_i = -2a */
			int j;
			for (j = 0; j < 3; ++j) twice_area_neg += (__int128) X[k[j]] * Y[k[(j + 1) % 3]] - (__int128) X[k[(j + 1) % 3]] * Y[k[j]];
			if (!(twice_area_neg < 0)) continue;   /* a <= 0: back-facing or zero area */
			for (j = 0; j < 3; ++j) { tris[count].X[j] = X[k[j]]; tris[count].Y[j] = Y[k[j]]; tris[count].z[j] = z[k[j]]; }
			tris[count].primitive = (uint32_t) t;
			++count;
		}
	}
	return count;
}

static __int128 ro_edge(const ro_triangle* t, int a, int b, __int128 px, __int128 py) {
	return (__int128) (t->X[b] - t->X[a]) * (py - t->Y[a]) - (__int128) (t->Y[b] - t->Y[a]) * (px - t->X[a]);
}

/* covered: all three edge functions negative (a > 0 puts the inside on the negative side with y pointing down), or zero on a top or left edge */
static int ro_covers(const ro_triangle* t, __int128 px, __int128 py, __int128 e[3]) {
	int j;
	for (j = 0; j < 3; ++j) {
		const int a = j, b = (j + 1) % 3, c = (j + 2) % 3;
		e[j] = ro_edge(t, a, b, px, py);
		if (e[j] > 0) return 0;
		if (e[j] == 0) {
			const int64_t dy = t->Y[b] - t->Y[a];
			int top_or_left;
			if (dy == 0) top_or_left = t->Y[c] > t->Y[a];
			else {
				const __int128 side = (__int128) (t->X[c] - t->X[a]) * dy - (__int128) (t->Y[c] - t->Y[a]) * (t->X[b] - t->X[a]);
				top_or_left = (side > 0) == (dy > 0);
			}
			if (!top_or_left) return 0;
		}
	}
	return 1;
}

/* depth of a covered pixel centre: weights = edge functions of the opposite edges over the doubled signed area, in fp64, rounded once to binary32,
   clamped to [0, 1]; *depth = 1.0 if it does not pass LESS against the clear value */
static float ro_depth(const ro_triangle* t, const __int128 e[3]) {
	const __int128 area = e[0] + e[1] + e[2];
	const double d = ((double) (int64_t) e[1] * t->z[0] + (double) (int64_t) e[2] * t->z[1] + (double) (int64_t) e[0] * t->z[2]) / (double) (int64_t) area;
	float f = (float) d;
	if (!(f > 0.0f)) f = 0.0f;
	if (f > 1.0f) f = 1.0f;
	return f;
}

/* the visibility buffer and depth buffer of the draw; out_fragments (may be NULL) counts every fragment of each pixel with the depth test off */
static void ro_rasterize(uint32_t width, uint32_t height, const unsigned char* constants, const uint32_t* quantized_positions, uint64_t triangle_count,
	uint32_t* out_visibility, float* out_depth, uint32_t* out_fragments)
{
	ro_triangle* tris = (ro_triangle*) malloc(sizeof(ro_triangle) * 7 * (size_t) (triangle_count ? triangle_count : 1));
	const size_t count = ro_primitives(width, height, constants, quantized_positions, triangle_count, tris);
	uint32_t x, y;
	for (y = 0; y < height; ++y) for (x = 0; x < width; ++x) {
		const size_t pixel = (size_t) y * width + x;
		const __int128 px = (__int128) x * 256 + 128, py = (__int128) y * 256 + 128;
		float stored = 1.0f;
		uint32_t visible = 0xFFFFFFFFu, fragments = 0;
		size_t i;
		for (i = 0; i < count; ++i) {
			__int128 e[3];
			float d;
			if (!ro_covers(&tris[i], px, py, e)) continue;
			d = ro_depth(&tris[i], e);
			++fragments;
			if (d < stored) { stored = d; visible = tris[i].primitive; }
		}
		out_visibility[pixel] = visible;
		out_depth[pixel] = stored;
		if (out_fragments) out_fragments[pixel] = fragments;
	}
	free(tris);
}

#endif
