// tests/ltc_fit_on_host.cpp -- TEST INFRASTRUCTURE: the LTC fit (vulkan_renderer_b200/csrc/vkr_ltc_fit.cuh) compiled for the CPU. The loops stand in for
// the launch: chain by chain, and within an objective evaluation thread by thread, then the same halving tree, so every float64 operation happens in
// the order the kernel performs it. -ffp-contract=off stands in for nvcc's -fmad=false. tests/test_ltc_fit_on_host.py holds this against numpy and
// scipy float64; the -m gpu tests hold the kernel against this bit for bit. Built by __graft_entry__.build() into tests/build/libltc_fit_on_host.so.
// Nothing in the product links against it.
#include <cstdint>
#include <vector>

#include "vkr_ltc_fit.cuh"

using namespace vkr_ltc;

// the specular BRDF of brdfs.glsl:74-87 (without cos(theta_i)) for count direction pairs {wo xyz, wi xyz}
extern "C" void vkr_host_ltc_specular_brdf(uint64_t count, const double* directions, const double* alpha, const double* f0, double* out) {
	for (uint64_t i = 0; i != count; ++i) out[i] = specular_brdf(directions + 6 * i, directions + 6 * i + 3, alpha[i], f0[i]);
}

// the albedo of the lobe at wo = (sin_theta, 0, cos_theta) from the quadrature of VNDF samples, as the fit computes it
extern "C" double vkr_host_ltc_albedo(uint32_t n, double cos_theta, double sin_theta, double alpha, double f0) {
	std::vector<double> tables(table_size(n, 2));
	make_tables(tables.data(), n, 2);
	const Cell cell = { cos_theta, sin_theta, alpha, f0 };
	const Quadrature q = quadrature_of(tables.data(), n);
	HostReducer reducer;
	double moments[kSlots];
	reducer.moments(moments, cell, q);
	return moments[0] / ((double) (kMomentRefinement * n) * (double) (kMomentRefinement * n));
}

// the chains chains[0 .. chain_count) (chain = layer * resolution + row), as the kernel fits them; per chain: fits resolution x 5 floats,
// errors and evaluations resolution entries, limit_hits one entry
extern "C" void vkr_host_ltc_fit_chains(uint32_t resolution, uint32_t fresnel_count, uint32_t n, uint32_t iteration_limit, uint32_t chain_count, const uint32_t* chains,
	float* fits, double* errors, uint32_t* evaluations, uint32_t* limit_hits)
{
	std::vector<double> tables(table_size(n, resolution));
	make_tables(tables.data(), n, resolution);
	const Quadrature q = quadrature_of(tables.data(), n);
	const double* cos_theta = cos_theta_of(tables.data(), n);
	#pragma omp parallel for schedule(dynamic, 1)
	for (int64_t c = 0; c < (int64_t) chain_count; ++c) {
		HostReducer reducer;
		fit_chain(reducer, chains[c], resolution, fresnel_count, cos_theta, cos_theta + resolution, q, iteration_limit,
			fits + (uint64_t) c * resolution * 5, errors + (uint64_t) c * resolution, evaluations + (uint64_t) c * resolution, limit_hits + c);
	}
}
