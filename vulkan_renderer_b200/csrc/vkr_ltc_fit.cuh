// vkr_ltc_fit.cuh -- fitting linearly transformed cosines (LTCs) to the specular BRDF (include/vkr_b200.h, vkr_fit_ltc_table; DESIGN.md §5).
//
// Everything the fit kernel of vkr_ltc_fit.cu computes is written here, in float64, so that a host build (tests/ltc_fit_on_host.cpp, plain g++ with
// -ffp-contract=off) performs the same operations in the same order and gets the same bits. nvcc compiles the library with -fmad=false, so a product
// is fused into an addition only where the source says fma(). Only + - * /, sqrt and fma appear: every cosine and sine the samplers need comes
// from tables the host fills once (make_tables) and hands to both builds.
//
// Target lobe: the specular term of evaluate_brdf (brdfs.glsl:74-87) with scalar F0, times cos(theta_i), over the upper hemisphere, for the outgoing
// direction wo = (sin theta, 0, cos theta). Its integral is the albedo; the fit approximates target / albedo.
// LTC: the density the shader evaluates (evaluate_ltc_density, ltc_utility.glsl:103-108) from the matrix get_ltc_coefficients builds out of what
// vkr_load_ltc_table stores for the five floats {m00, m02, m11, m20, albedo}. That matrix is proportional to the inverse of
//   M = [[m00, 0, m20], [0, m11, 0], [m02, 0, 1]]   (cosine space -> shading space),
// so M is what the fit moves: a = m00, c = m11, b = m20, d = m02. The loader stores (m11, m02 m11, m00 - m02 m20, -m11 m20, m00 m11) over their
// largest magnitude; with a, c > 0, b <= 0 and d >= 0 all of them lie in [0, 1] and the determinant is positive, so the fit keeps to that domain:
// the parameters are those of Heitz et al. in the frame of the lobe's mean direction (matrix_of), and a matrix outside the domain is rejected.
//
// Objective: Heitz et al. 2016's L3 error, the integral over the sphere of |target / albedo - LTC|^3, estimated with the balance heuristic over
// n x n stratified samples of each distribution: visible-normal (VNDF) samples of the GGX lobe (brdfs.glsl:122-162) and cosine samples pushed
// through M. Sample k < n^2 is a VNDF sample, k >= n^2 an LTC sample; within each, row r = (k mod n^2) / n gives u = (r + 1/2) / n and column
// s = k mod n the azimuth 2 pi (s + 1/2) / n.
//
// Summation order: thread t of kThreads sums the samples t, t + kThreads, ... in that order; the threads combine in a fixed halving tree
// (partial[t] += partial[t + s], s = kThreads / 2, ..., 1). Nothing depends on the device.
//
// Minimiser: Nelder-Mead over k = {k11, k22, k13} (one parameter k11 = k22, k13 = 0 on the row theta = 0, where the lobe is rotationally
// symmetric) with reflection 1, expansion 2, contraction 1/2, shrink 1/2, initial simplex k0 and k0 + kSimplexStep * max(|k0_i|, |k0_0|) e_i; it
// stops when (f_worst - f_best) <= kRelTolerance * f_best or after the iteration limit. A chain is one (Fresnel layer, inclination row): its cells
// are fitted from alpha = 1 down, each starting from its neighbour's parameters; the first starts from the cosine lobe on the mean direction.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define VKR_LTC_FN __host__ __device__ inline
#define VKR_LTC_HOST_FN __host__ inline
#else
#include <math.h>
#define VKR_LTC_FN inline
#define VKR_LTC_HOST_FN inline
#endif

namespace vkr_ltc {

constexpr int kThreads = 128;              // threads per chain: part of the summation order
constexpr int kParams = 3;                 // k11, k22, k13
constexpr int kMatrix = 4;                 // a, c, b, d
constexpr int kSlots = 3;                  // moments: albedo, mean direction x, z
constexpr double kAlphaMin = 1.0e-3;       // alpha = 0 is a delta lobe
constexpr double kThetaMaxDegrees = 89.5;  // theta = 90 degrees is grazing: wo in the tangent plane
constexpr double kRelTolerance = 1.0e-6;
constexpr double kSimplexStep = 0.1;
constexpr double kRejected = 1.0e300;       // the objective of a degenerate matrix (a or c zero) or of a NaN
constexpr double kInvPi = 0.318309886183790671537767526745028724;
constexpr double kPi = 3.14159265358979323846264338327950288;

struct Cell { double cos_theta, sin_theta, alpha, f0; };
constexpr int kMomentRefinement = 8;      // the albedo and the mean direction take (kMomentRefinement n)^2 VNDF samples, once per cell
// n azimuths 2 pi (s + 1/2) / n for the objective, kMomentRefinement n for the moments
struct Quadrature { int n; const double* cos_phi; const double* sin_phi; const double* moment_cos_phi; const double* moment_sin_phi; };

VKR_LTC_FN double cell_alpha(uint32_t column, uint32_t resolution) {
	const double r = (double) column / (double) (resolution - 1);
	const double alpha = r * r;
	return alpha < kAlphaMin ? kAlphaMin : alpha;
}
VKR_LTC_FN double cell_f0(uint32_t layer, uint32_t fresnel_count) { return (double) layer / (double) (fresnel_count - 1); }

// ---- the target lobe
VKR_LTC_FN double fresnel_schlick(double f0, double cos_theta) {   // brdfs.glsl:42-46 with F90 = 1
	const double flipped = 1.0 - cos_theta;
	const double flipped_squared = flipped * flipped;
	return f0 + (1.0 - f0) * (flipped_squared * flipped * flipped_squared);
}

// the specular BRDF (brdfs.glsl:58-61, 74-87 with diffuse = false), wo and wi unit vectors in shading space (normal z); cos(theta_i) > 0
VKR_LTC_FN double specular_brdf(const double* wo, const double* wi, double alpha, double f0) {
	double h[3] = { wi[0] + wo[0], wi[1] + wo[1], wi[2] + wo[2] };
	const double rcp_length = 1.0 / sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
	h[0] = h[0] * rcp_length; h[1] = h[1] * rcp_length; h[2] = h[2] * rcp_length;
	const double lambert_incoming = wi[2], lambert_outgoing = wo[2];
	const double outgoing_dot_half = wo[0] * h[0] + wo[1] * h[1] + wo[2] * h[2];
	const double normal_dot_half = h[2];
	const double roughness_squared = alpha * alpha;
	double ggx = fma(fma(normal_dot_half, roughness_squared, -normal_dot_half), normal_dot_half, 1.0);
	ggx = roughness_squared / (ggx * ggx);
	const double masking = lambert_incoming * sqrt(fma(fma(-lambert_outgoing, roughness_squared, lambert_outgoing), lambert_outgoing, roughness_squared));
	const double shadowing = lambert_outgoing * sqrt(fma(fma(-lambert_incoming, roughness_squared, lambert_incoming), lambert_incoming, roughness_squared));
	const double smith = 0.5 / (masking + shadowing);
	const double c = outgoing_dot_half < 0.0 ? 0.0 : (outgoing_dot_half > 1.0 ? 1.0 : outgoing_dot_half);
	return ggx * smith * fresnel_schlick(f0, c) * kInvPi;
}

VKR_LTC_FN double target(const double* wo, const double* wi, double alpha, double f0) {
	return wi[2] > 0.0 ? specular_brdf(wo, wi, alpha, f0) * wi[2] : 0.0;
}

// density of VNDF sampling (get_ggx_reflected_direction_density, brdfs.glsl:180-224) at any unit wi; 0 where no visible normal reflects wo to wi
VKR_LTC_FN double vndf_density(const double* wo, const double* wi, double alpha) {
	double h[3] = { wi[0] + wo[0], wi[1] + wo[1], wi[2] + wo[2] };
	const double length_squared = h[0] * h[0] + h[1] * h[1] + h[2] * h[2];
	if (!(length_squared > 0.0)) return 0.0;
	const double rcp_length = 1.0 / sqrt(length_squared);
	h[0] = h[0] * rcp_length; h[1] = h[1] * rcp_length; h[2] = h[2] * rcp_length;
	const double micro_dot_out = wo[0] * h[0] + wo[1] * h[1] + wo[2] * h[2];
	const double micro_dot_normal = h[2];
	if (!(micro_dot_out > 0.0) || !(micro_dot_normal > 0.0)) return 0.0;
	const double roughness_squared = alpha * alpha;
	double ggx = fma(fma(micro_dot_normal, roughness_squared, -micro_dot_normal), micro_dot_normal, 1.0);
	ggx = roughness_squared / (ggx * ggx);
	ggx = ggx * kInvPi;
	double masking_over_out_z = sqrt(fma(fma(-wo[2], roughness_squared, wo[2]), wo[2], roughness_squared));
	masking_over_out_z = 2.0 / (wo[2] + masking_over_out_z);
	return masking_over_out_z * micro_dot_out * ggx / (4.0 * micro_dot_out);
}

// sample_ggx_reflected_direction (brdfs.glsl:122-162, 200-210) for wo = (sin, 0, cos), isotropic alpha, disk radius sqrt(u), azimuth (cos_phi, sin_phi)
VKR_LTC_FN void sample_vndf(double* wi, const double* wo, double alpha, double u, double cos_phi, double sin_phi) {
	double v[3] = { alpha * wo[0], alpha * wo[1], wo[2] };
	const double rcp_v = 1.0 / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
	v[0] = v[0] * rcp_v; v[1] = v[1] * rcp_v; v[2] = v[2] * rcp_v;
	const double length_sq = v[0] * v[0] + v[1] * v[1];
	double t1[3] = { 1.0, 0.0, 0.0 };
	if (length_sq > 0.0) { const double r = 1.0 / sqrt(length_sq); t1[0] = -v[1] * r; t1[1] = v[0] * r; }
	const double t2[3] = { v[1] * t1[2] - v[2] * t1[1], v[2] * t1[0] - v[0] * t1[2], v[0] * t1[1] - v[1] * t1[0] };
	const double radius = sqrt(u);
	const double dx = radius * cos_phi, dy = radius * sin_phi;
	const double lerp_factor = fma(0.5, v[2], 0.5);
	const double sx = dx;
	const double sy = sqrt(fma(-dx, dx, 1.0)) * (1.0 - lerp_factor) + dy * lerp_factor;
	const double zz = 1.0 - (sx * sx + sy * sy);
	const double sz = sqrt(zz > 0.0 ? zz : 0.0);
	double m[3] = { sx * t1[0] + sy * t2[0] + sz * v[0], sx * t1[1] + sy * t2[1] + sz * v[1], sx * t1[2] + sy * t2[2] + sz * v[2] };
	m[0] = alpha * m[0]; m[1] = alpha * m[1];
	const double rcp_m = 1.0 / sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
	m[0] = m[0] * rcp_m; m[1] = m[1] * rcp_m; m[2] = m[2] * rcp_m;
	const double micro_dot_out = m[0] * wo[0] + m[1] * wo[1] + m[2] * wo[2];
	const double two_dot = 2.0 * micro_dot_out;
	wi[0] = fma(two_dot, m[0], -wo[0]); wi[1] = fma(two_dot, m[1], -wo[1]); wi[2] = fma(two_dot, m[2], -wo[2]);
}

// ---- the LTC of M = [[a, 0, b], [0, c, 0], [d, 0, 1]], x = {a, c, b, d}
// the density evaluate_ltc_density computes with shading_to_cosine_space = adj(M), normalised to 1 over the sphere
VKR_LTC_FN double ltc_density(const double* x, const double* w) {
	const double a = x[0], c = x[1], b = x[2], d = x[3];
	const double s00 = c, s02 = -(c * b), s11 = a - d * b, s20 = -(d * c), s22 = a * c;
	const double v0 = s00 * w[0] + s02 * w[2], v1 = s11 * w[1], v2 = s20 * w[0] + s22 * w[2];
	if (!(v2 > 0.0)) return 0.0;
	const double determinant = s11 * (s00 * s22 - s20 * s02);
	const double length_squared = v0 * v0 + v1 * v1 + v2 * v2;
	return v2 * determinant / (length_squared * length_squared) * kInvPi;
}

// a cosine sample (disk radius sqrt(u), azimuth phi) pushed through M and normalised
VKR_LTC_FN void sample_ltc(double* w, const double* x, double u, double cos_phi, double sin_phi) {
	const double radius = sqrt(u);
	const double zz = 1.0 - u;
	const double cx = radius * cos_phi, cy = radius * sin_phi, cz = sqrt(zz > 0.0 ? zz : 0.0);
	const double m0 = x[0] * cx + x[2] * cz, m1 = x[1] * cy, m2 = x[3] * cx + cz;
	const double r = 1.0 / sqrt(m0 * m0 + m1 * m1 + m2 * m2);
	w[0] = m0 * r; w[1] = m1 * r; w[2] = m2 * r;
}

// the matrix of the fit's parameters k = {k11, k22, k13} in the frame of the lobe's mean direction (mx, 0, mz), mx <= 0 < mz:
// M = [X Y Z] [[|k11|, 0, k13], [0, |k22|, 0], [0, 0, 1]] with Z = (mx, 0, mz), X = (mz, 0, -mx), divided by its entry M[2][2]. false where M
// leaves the domain the loader represents without clamping (M[2][2] <= 0, a or c not positive, b > 0; d >= 0 follows).
VKR_LTC_FN bool matrix_of(double* x, const double* k, double mx, double mz) {
	const double k11 = k[0] < 0.0 ? -k[0] : k[0], k22 = k[1] < 0.0 ? -k[1] : k[1];
	const double m22 = mz - k[2] * mx;
	if (!(m22 > 0.0)) return false;
	const double rcp = 1.0 / m22;
	x[0] = k11 * mz * rcp; x[1] = k22 * rcp; x[2] = (k[2] * mz + mx) * rcp; x[3] = -(k11 * mx) * rcp;
	return x[0] > 0.0 && x[1] > 0.0 && x[2] <= 0.0 && x[3] >= 0.0;
}

// ---- per-thread partial sums
VKR_LTC_FN void sample_point(int n, int k, double& u, int& s) {
	const int nn = n * n;
	const int local = k < nn ? k : k - nn;
	u = (double) (2 * (local / n) + 1) / (double) (2 * n);
	s = local % n;
}

// thread t: sum over its VNDF samples (m = kMomentRefinement n per axis) of target / density, and of that times wi.x, wi.z (the albedo and the
// lobe's mean direction, times m^2)
VKR_LTC_FN void thread_moment_terms(double* out, const Cell& cell, const Quadrature& q, int thread) {
	out[0] = 0.0; out[1] = 0.0; out[2] = 0.0;
	const double wo[3] = { cell.sin_theta, 0.0, cell.cos_theta };
	const int m = kMomentRefinement * q.n, mm = m * m;
	for (int k = thread; k < mm; k += kThreads) {
		double u; int s; sample_point(m, k, u, s);
		double wi[3]; sample_vndf(wi, wo, cell.alpha, u, q.moment_cos_phi[s], q.moment_sin_phi[s]);
		const double p = vndf_density(wo, wi, cell.alpha);
		if (!(wi[2] > 0.0) || !(p > 0.0)) continue;
		const double weight = target(wo, wi, cell.alpha, cell.f0) / p;
		out[0] = out[0] + weight; out[1] = out[1] + weight * wi[0]; out[2] = out[2] + weight * wi[2];
	}
}

// thread t: sum over its samples of both distributions of |target / albedo - LTC|^3 / (VNDF density + LTC density)
VKR_LTC_FN double thread_objective_term(const double* x, const Cell& cell, const Quadrature& q, double rcp_albedo, int thread) {
	const double wo[3] = { cell.sin_theta, 0.0, cell.cos_theta };
	const int nn = q.n * q.n;
	double sum = 0.0;
	for (int k = thread; k < 2 * nn; k += kThreads) {
		double u; int s; sample_point(q.n, k, u, s);
		double w[3];
		if (k < nn) sample_vndf(w, wo, cell.alpha, u, q.cos_phi[s], q.sin_phi[s]);
		else sample_ltc(w, x, u, q.cos_phi[s], q.sin_phi[s]);
		const double lobe = target(wo, w, cell.alpha, cell.f0) * rcp_albedo;
		const double ltc = ltc_density(x, w);
		const double pdf = vndf_density(wo, w, cell.alpha) + ltc;
		if (!(pdf > 0.0)) continue;
		const double e = lobe > ltc ? lobe - ltc : ltc - lobe;
		sum = sum + e * e * e / pdf;
	}
	return sum;
}

// ---- one cell and one chain. Reducer provides moments(out[kSlots], cell, q) and objective(x, cell, q, rcp_albedo), both the totals of the
// halving tree (the kernel's reducer runs the tree in shared memory, the host's loops over the threads). Every thread runs this code with the
// same values.
struct CellFit { double k[kParams]; double x[kMatrix]; double error; double albedo; uint32_t evaluations; uint32_t iterations; };

struct Problem { Cell cell; Quadrature q; double mx, mz, rcp_albedo, rcp_count; int isotropic; };

template <class Reducer> VKR_LTC_FN double evaluate(Reducer& reducer, const double* p, const Problem& problem, uint32_t& evaluations) {
	const double k[kParams] = { p[0], problem.isotropic ? p[0] : p[1], problem.isotropic ? 0.0 : p[2] };
	double x[kMatrix];
	++evaluations;
	if (!matrix_of(x, k, problem.mx, problem.mz)) return kRejected;
	const double f = reducer.objective(x, problem.cell, problem.q, problem.rcp_albedo) * problem.rcp_count;
	return f == f ? f : kRejected;
}

// start: the previous cell's parameters, or NULL for the first cell of a chain (k = {1, 1, 0}: the cosine lobe on the mean direction).
// isotropic (the row theta = 0): one parameter, k11 = k22, k13 = 0, and the mean direction is the normal.
template <class Reducer> VKR_LTC_FN void fit_cell(CellFit& out, Reducer& reducer, const Cell& cell, const Quadrature& q, const double* start, int isotropic, uint32_t iteration_limit) {
	double moments[kSlots];
	reducer.moments(moments, cell, q);
	Problem problem = { cell, q, moments[1], moments[2], 0.0, 1.0 / (double) (q.n * q.n), isotropic };
	const double albedo = moments[0] / ((double) (kMomentRefinement * q.n) * (double) (kMomentRefinement * q.n));
	out.albedo = albedo;
	problem.rcp_albedo = albedo > 0.0 ? 1.0 / albedo : 0.0;
	if (isotropic || problem.mx > 0.0) problem.mx = 0.0;
	const double rcp_length = 1.0 / sqrt(problem.mx * problem.mx + problem.mz * problem.mz);
	problem.mx = problem.mx * rcp_length; problem.mz = problem.mz * rcp_length;
	const int dim = isotropic ? 1 : kParams;
	double v[kParams + 1][kParams], f[kParams + 1];
	v[0][0] = 1.0; v[0][1] = 1.0; v[0][2] = 0.0;
	if (start) { v[0][0] = start[0]; v[0][1] = start[1]; v[0][2] = start[2]; }
	if (isotropic) { v[0][1] = v[0][0]; v[0][2] = 0.0; }
	double x[kMatrix];
	if (!matrix_of(x, v[0], problem.mx, problem.mz)) v[0][2] = 0.0;   // k13 = 0 is always representable
	uint32_t evaluations = 0;
	const double scale = v[0][0] < 0.0 ? -v[0][0] : v[0][0];
	for (int i = 1; i <= dim; ++i) {
		for (int j = 0; j != kParams; ++j) v[i][j] = v[0][j];
		const double m = v[0][i - 1] < 0.0 ? -v[0][i - 1] : v[0][i - 1];
		v[i][i - 1] = v[i][i - 1] + kSimplexStep * (m > scale ? m : scale);
	}
	for (int i = 0; i <= dim; ++i) f[i] = evaluate(reducer, v[i], problem, evaluations);
	uint32_t iteration = 0;
	for (;; ++iteration) {
		for (int i = 1; i <= dim; ++i)   // stable insertion sort by value
			for (int j = i; j > 0 && f[j] < f[j - 1]; --j) {
				const double t = f[j]; f[j] = f[j - 1]; f[j - 1] = t;
				for (int k = 0; k != kParams; ++k) { const double w = v[j][k]; v[j][k] = v[j - 1][k]; v[j - 1][k] = w; }
			}
		if (iteration >= iteration_limit || f[dim] - f[0] <= kRelTolerance * f[0]) break;
		double centroid[kParams], xr[kParams], xt[kParams];
		for (int k = 0; k != kParams; ++k) {
			double sum = v[0][k];
			for (int i = 1; i < dim; ++i) sum = sum + v[i][k];
			centroid[k] = sum / (double) dim;
			xr[k] = centroid[k] + (centroid[k] - v[dim][k]);
		}
		const double fr = evaluate(reducer, xr, problem, evaluations);
		bool shrink = false;
		if (fr < f[0]) {
			for (int k = 0; k != kParams; ++k) xt[k] = centroid[k] + 2.0 * (centroid[k] - v[dim][k]);
			const double fe = evaluate(reducer, xt, problem, evaluations);
			const bool expand = fe < fr;
			for (int k = 0; k != kParams; ++k) v[dim][k] = expand ? xt[k] : xr[k];
			f[dim] = expand ? fe : fr;
		}
		else if (fr < f[dim - 1]) {
			for (int k = 0; k != kParams; ++k) v[dim][k] = xr[k];
			f[dim] = fr;
		}
		else {
			const bool outside = fr < f[dim];
			for (int k = 0; k != kParams; ++k) xt[k] = centroid[k] + 0.5 * ((outside ? xr[k] : v[dim][k]) - centroid[k]);
			const double fc = evaluate(reducer, xt, problem, evaluations);
			if (outside ? fc <= fr : fc < f[dim]) {
				for (int k = 0; k != kParams; ++k) v[dim][k] = xt[k];
				f[dim] = fc;
			}
			else shrink = true;
		}
		if (shrink)
			for (int i = 1; i <= dim; ++i) {
				for (int k = 0; k != kParams; ++k) v[i][k] = v[0][k] + 0.5 * (v[i][k] - v[0][k]);
				f[i] = evaluate(reducer, v[i], problem, evaluations);
			}
	}
	out.k[0] = v[0][0]; out.k[1] = isotropic ? v[0][0] : v[0][1]; out.k[2] = isotropic ? 0.0 : v[0][2];
	matrix_of(out.x, out.k, problem.mx, problem.mz);
	out.error = f[0];
	out.evaluations = evaluations;
	out.iterations = iteration;
}

// the five floats of the file format, {m00, m02, m11, m20, albedo}
VKR_LTC_FN void store_cell(float* texel, const CellFit& fit) {
	texel[0] = (float) fit.x[0]; texel[1] = (float) fit.x[3]; texel[2] = (float) fit.x[1]; texel[3] = (float) fit.x[2]; texel[4] = (float) fit.albedo;
}

// chain = layer * resolution + row; cells from column resolution - 1 down to 0. fits: the chain's row, resolution texels of 5 floats;
// errors, evaluations: resolution entries each, by column; limit_hits: cells that stopped at the iteration limit. NULL outputs: nothing is stored.
template <class Reducer> VKR_LTC_FN void fit_chain(Reducer& reducer, uint32_t chain, uint32_t resolution, uint32_t fresnel_count, const double* cos_theta, const double* sin_theta,
	const Quadrature& q, uint32_t iteration_limit, float* fits, double* errors, uint32_t* evaluations, uint32_t* limit_hits)
{
	const uint32_t layer = chain / resolution, row = chain % resolution;
	Cell cell = { cos_theta[row], sin_theta[row], 0.0, cell_f0(layer, fresnel_count) };
	CellFit fit = {};
	uint32_t hits = 0;
	for (uint32_t step = 0; step != resolution; ++step) {
		const uint32_t column = resolution - 1 - step;
		cell.alpha = cell_alpha(column, resolution);
		double start[kParams];
		for (int k = 0; k != kParams; ++k) start[k] = fit.k[k];
		fit_cell(fit, reducer, cell, q, step ? start : nullptr, row == 0, iteration_limit);
		if (fits) { store_cell(fits + 5 * column, fit); errors[column] = fit.error; evaluations[column] = fit.evaluations; }
		if (fit.iterations >= iteration_limit) ++hits;
	}
	if (limit_hits) *limit_hits = hits;
}

// ---- host only: the trigonometric tables both builds read (the library's host code and the CPU build call the same libm)
// tables: table_size(n, resolution) doubles: cos, sin of n azimuths (the objective), of kMomentRefinement n azimuths (the moments), then cos, sin
// theta of the rows (theta = row / (resolution - 1) * pi / 2, at most kThetaMaxDegrees)
VKR_LTC_FN uint64_t table_size(uint32_t n, uint32_t resolution) { return 2 * (uint64_t) n * (1 + kMomentRefinement) + 2 * (uint64_t) resolution; }
VKR_LTC_FN Quadrature quadrature_of(const double* tables, uint32_t n) {
	const uint64_t m = (uint64_t) kMomentRefinement * n;
	const Quadrature q = { (int) n, tables, tables + n, tables + 2 * n, tables + 2 * n + m };
	return q;
}
VKR_LTC_FN const double* cos_theta_of(const double* tables, uint32_t n) { return tables + 2 * (uint64_t) n * (1 + kMomentRefinement); }
VKR_LTC_HOST_FN void make_tables(double* tables, uint32_t n, uint32_t resolution) {
	const uint32_t m = kMomentRefinement * n;
	for (uint32_t s = 0; s != n; ++s) {
		const double phi = 2.0 * kPi * ((double) s + 0.5) / (double) n;
		tables[s] = cos(phi); tables[n + s] = sin(phi);
	}
	for (uint32_t s = 0; s != m; ++s) {
		const double phi = 2.0 * kPi * ((double) s + 0.5) / (double) m;
		tables[2 * n + s] = cos(phi); tables[2 * n + m + s] = sin(phi);
	}
	double* cos_theta = tables + 2 * (uint64_t) n * (1 + kMomentRefinement);
	double* sin_theta = cos_theta + resolution;
	const double theta_max = kThetaMaxDegrees * (kPi / 180.0);
	for (uint32_t i = 0; i != resolution; ++i) {
		double theta = (double) i / (double) (resolution - 1) * (0.5 * kPi);
		if (theta > theta_max) theta = theta_max;
		cos_theta[i] = cos(theta); sin_theta[i] = sin(theta);
	}
}

#ifndef __CUDACC__
// the kernel's reductions as one CPU thread runs them
struct HostReducer {
	double partial[kThreads][kSlots];
	void tree() {
		for (int s = kThreads / 2; s > 0; s >>= 1)
			for (int t = 0; t < s; ++t)
				for (int k = 0; k != kSlots; ++k) partial[t][k] = partial[t][k] + partial[t + s][k];
	}
	void moments(double* out, const Cell& cell, const Quadrature& q) {
		for (int t = 0; t != kThreads; ++t) thread_moment_terms(partial[t], cell, q, t);
		tree();
		for (int k = 0; k != kSlots; ++k) out[k] = partial[0][k];
	}
	double objective(const double* x, const Cell& cell, const Quadrature& q, double rcp_albedo) {
		for (int t = 0; t != kThreads; ++t) { partial[t][0] = thread_objective_term(x, cell, q, rcp_albedo, t); partial[t][1] = partial[t][2] = 0.0; }
		tree();
		return partial[0][0];
	}
};
#endif

} // namespace vkr_ltc
