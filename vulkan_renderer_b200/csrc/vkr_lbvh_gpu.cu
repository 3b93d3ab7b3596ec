// vkr_lbvh_gpu.cu -- linear BVH built on the GPU (SURVEY 8 row f2; replaces the driver's acceleration-structure build,
// vkCmdBuildAccelerationStructuresKHR at src/scene.c:354-378, which also runs on the GPU).
//
// The parallel form of vkr_lbvh.cpp, step for step, so that both produce the same bytes:
//   1. triangle boxes, centroids, scene / centroid bounds            one thread per triangle, atomicMin/Max on order-preserving keys
//   2. 63-bit Morton codes, stable radix sort by code                 cub::DeviceRadixSort (values start as 0..n-1, so ties keep the index order)
//   3. triangle slots (v0, e1, e2) and original indices in that order one thread per slot
//   4. binary radix tree (Karras, HPG 2012)                           one thread per internal node, no synchronisation
//   5. boxes bottom-up                                                 one thread per leaf walks up; the second arrival at a node merges
//   6. collapse subtrees of <= 4 triangles, number the rest           exclusive prefix sum over "has more than four triangles"
//   7. node pairs (centre + half extent rounded up, child references)  one thread per internal node
//   8. depth in node pairs                                             one thread per internal node walks up, atomicMax
// Everything is integer or exact min/max work except the box encoding of step 7, which repeats the host's double-precision
// arithmetic (-fmad=false: no contraction). HBM traffic ~ 0.4 KB per triangle; the radix sort (8 passes over 12-byte pairs) dominates.
// Selected with VKR_BVH_BUILDER=lbvh_gpu; the default builder stays the binned-SAH one (better trees for the benchmark).
#include "vkr_bvh.h"
#include "vkr_lbvh.cuh"
#include "vkr_trace.cuh"
#include "vkr_kernels.h"
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace vkr {
namespace {

constexpr int kThreads = 256;
constexpr int kLeafSize = kLbvhLeafSize;

struct bounds_keys { uint32_t scene_lo[3], scene_hi[3], centroid_lo[3], centroid_hi[3]; };

__global__ void __launch_bounds__(kThreads) triangle_bounds_kernel(const float* __restrict__ vertices, uint32_t n, float* __restrict__ box_lo, float* __restrict__ box_hi, float* __restrict__ centroid, bounds_keys* keys) {
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	const bool valid = t < n;
	float lo[3], hi[3], c[3];
	lbvh_triangle_bounds(vertices, valid ? t : 0u, lo, hi, c);
#pragma unroll
	for (int a = 0; a != 3; ++a) {
		if (valid) { box_lo[3 * (size_t) t + a] = lo[a]; box_hi[3 * (size_t) t + a] = hi[a]; centroid[3 * (size_t) t + a] = c[a]; }
		// one atomic per warp and bound: min / max over the warp first (lanes past the end contribute the neutral keys)
		const uint32_t k_lo = __reduce_min_sync(0xffffffffu, valid ? float_to_ordered(lo[a]) : 0xffffffffu), k_hi = __reduce_max_sync(0xffffffffu, valid ? float_to_ordered(hi[a]) : 0u);
		const uint32_t k_clo = __reduce_min_sync(0xffffffffu, valid ? float_to_ordered(c[a]) : 0xffffffffu), k_chi = __reduce_max_sync(0xffffffffu, valid ? float_to_ordered(c[a]) : 0u);
		if ((threadIdx.x & 31) == 0) {
			atomicMin(&keys->scene_lo[a], k_lo); atomicMax(&keys->scene_hi[a], k_hi);
			atomicMin(&keys->centroid_lo[a], k_clo); atomicMax(&keys->centroid_hi[a], k_chi);
		}
	}
}

__global__ void __launch_bounds__(kThreads) morton_kernel(const float* __restrict__ centroid, uint32_t n, f3 lo, f3 inv_extent, uint64_t* __restrict__ codes, uint32_t* __restrict__ indices) {
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	if (t >= n) return;
	codes[t] = lbvh_morton(centroid + 3 * (size_t) t, lo, inv_extent);
	indices[t] = t;
}

__global__ void __launch_bounds__(kThreads) slots_kernel(const float* __restrict__ vertices, const uint32_t* __restrict__ order, uint32_t n, float4* __restrict__ tris, uint32_t* __restrict__ tri_ids) {
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s >= n) return;
	const uint32_t t = order[s];
	float slot[12];
	lbvh_slot(vertices, t, slot);
	tris[3 * (size_t) s] = make_float4(slot[0], slot[1], slot[2], slot[3]);
	tris[3 * (size_t) s + 1] = make_float4(slot[4], slot[5], slot[6], slot[7]);
	tris[3 * (size_t) s + 2] = make_float4(slot[8], slot[9], slot[10], slot[11]);
	tri_ids[s] = t;
}

__global__ void __launch_bounds__(kThreads) radix_tree_kernel(const uint64_t* __restrict__ codes, uint32_t n, int32_t* __restrict__ first, int32_t* __restrict__ last, int32_t* __restrict__ split,
	int32_t* __restrict__ parent, int32_t* __restrict__ leaf_parent)
{
	const int64_t i = (int64_t) blockIdx.x * kThreads + threadIdx.x;
	if (i < (int64_t) n - 1) lbvh_radix_tree_node(codes, n, i, first, last, split, parent, leaf_parent);
}

__global__ void __launch_bounds__(kThreads) refit_kernel(uint32_t n, const uint32_t* __restrict__ order, const float* __restrict__ box_lo, const float* __restrict__ box_hi,
	const int32_t* __restrict__ first, const int32_t* __restrict__ last, const int32_t* __restrict__ split, const int32_t* __restrict__ parent, const int32_t* __restrict__ leaf_parent,
	float* node_lo, float* node_hi, uint32_t* arrivals)
{
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s < n) lbvh_refit_from_leaf(s, order, box_lo, box_hi, first, last, split, parent, leaf_parent, node_lo, node_hi, arrivals);
}

__global__ void __launch_bounds__(kThreads) used_kernel(uint32_t internal_count, const int32_t* __restrict__ first, const int32_t* __restrict__ last, uint32_t* __restrict__ used) {
	const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
	if (i < internal_count) used[i] = lbvh_is_used(first[i], last[i]);
}

__global__ void __launch_bounds__(kThreads) emit_kernel(uint32_t internal_count, const uint32_t* __restrict__ order, const float* __restrict__ box_lo, const float* __restrict__ box_hi,
	const float* __restrict__ node_lo, const float* __restrict__ node_hi, const int32_t* __restrict__ first, const int32_t* __restrict__ last, const int32_t* __restrict__ split,
	const uint32_t* __restrict__ used, const uint32_t* __restrict__ rank, float pad, float* __restrict__ nodes)
{
	const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
	if (i >= internal_count || !used[i]) return;
	float out[16];
	lbvh_emit_pair(i, order, box_lo, box_hi, node_lo, node_hi, first, last, split, used, rank, pad, out);
	float4* dst = reinterpret_cast<float4*>(nodes + 16 * (size_t) rank[i]);
#pragma unroll
	for (int k = 0; k != 4; ++k) dst[k] = make_float4(out[4 * k], out[4 * k + 1], out[4 * k + 2], out[4 * k + 3]);
}

__global__ void __launch_bounds__(kThreads) depth_kernel(uint32_t internal_count, const uint32_t* __restrict__ used, const int32_t* __restrict__ parent, uint32_t* max_depth) {
	const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
	if (i < internal_count && used[i]) atomicMax(max_depth, lbvh_depth(i, parent));
}

inline float key_to_float(uint32_t k) { const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k; float f; memcpy(&f, &u, 4); return f; } // ordered_to_float() on the host

struct scratch { // device allocations that live as long as one build
	static constexpr int kCapacity = 32;
	void* ptr[kCapacity] = {};
	int count = 0;
	template <class T> bool alloc(T** p, size_t elements) {
		*p = nullptr;
		if (count == kCapacity || cudaMalloc((void**) p, sizeof(T) * (elements ? elements : 1)) != cudaSuccess) { *p = nullptr; return false; }
		ptr[count++] = *p;
		return true;
	}
	~scratch() { for (int i = 0; i != count; ++i) cudaFree(ptr[i]); }
};

} // namespace

// Builds on the current device. vertices: HOST pointer, 9 floats per triangle. On success *d_nodes (16 floats per pair), *d_tris (12 floats per slot)
// and *d_tri_ids are device allocations owned by the caller (cudaFree). Returns non-zero (and allocates nothing) on failure or if there are
// fewer than five triangles (the host builder handles those).
int build_lbvh_device(const float* vertices, uint64_t triangle_count, void* stream_handle, void** d_nodes, void** d_tris, void** d_tri_ids, uint64_t* node_count, uint32_t* max_depth) {
	cudaStream_t stream = (cudaStream_t) stream_handle;
	*d_nodes = *d_tris = *d_tri_ids = nullptr; *node_count = 0; *max_depth = 0;
	if (triangle_count <= (uint64_t) kLeafSize || triangle_count >= (1ull << 27)) return 1;
	const uint32_t n = (uint32_t) triangle_count, internal_count = n - 1;
	const uint32_t blocks = (n + kThreads - 1) / kThreads;
	scratch s;
	float *d_vertices, *box_lo, *box_hi, *centroid, *node_lo, *node_hi;
	uint64_t *codes_in, *codes; uint32_t *index_in, *order, *arrivals, *used, *rank, *d_depth; bounds_keys* keys;
	int32_t *first, *last, *split, *parent, *leaf_parent;
	if (!s.alloc(&d_vertices, 9 * (size_t) n) || !s.alloc(&box_lo, 3 * (size_t) n) || !s.alloc(&box_hi, 3 * (size_t) n) || !s.alloc(&centroid, 3 * (size_t) n)
		|| !s.alloc(&codes_in, n) || !s.alloc(&codes, n) || !s.alloc(&index_in, n) || !s.alloc(&order, n) || !s.alloc(&keys, 1)) return 1;
	if (cudaMemcpyAsync(d_vertices, vertices, sizeof(float) * 9 * (size_t) n, cudaMemcpyHostToDevice, stream) != cudaSuccess) return 1;
	// 1. boxes and bounds
	bounds_keys init;
	for (int a = 0; a != 3; ++a) { init.scene_lo[a] = init.centroid_lo[a] = 0xffffffffu; init.scene_hi[a] = init.centroid_hi[a] = 0u; }
	cudaMemcpyAsync(keys, &init, sizeof(init), cudaMemcpyHostToDevice, stream);
	triangle_bounds_kernel<<<blocks, kThreads, 0, stream>>>(d_vertices, n, box_lo, box_hi, centroid, keys);
	bounds_keys found;
	if (cudaMemcpyAsync(&found, keys, sizeof(found), cudaMemcpyDeviceToHost, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess) return 1;
	float extent = 0.0f; f3 lo, inv; float* lo_a[3] = { &lo.x, &lo.y, &lo.z }; float* inv_a[3] = { &inv.x, &inv.y, &inv.z };
	for (int a = 0; a != 3; ++a) {
		extent = fmaxf(extent, fmaxf(fabsf(key_to_float(found.scene_lo[a])), fabsf(key_to_float(found.scene_hi[a]))));
		const float c_lo = key_to_float(found.centroid_lo[a]), e = key_to_float(found.centroid_hi[a]) - c_lo;
		*lo_a[a] = c_lo; *inv_a[a] = (e > 0.0f) ? 1.0f / e : 0.0f;
	}
	const float pad = extent * (1.0f / 65536.0f);
	// 2. Morton codes and their order
	morton_kernel<<<blocks, kThreads, 0, stream>>>(centroid, n, lo, inv, codes_in, index_in);
	size_t sort_bytes = 0;
	if (cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, codes_in, codes, index_in, order, (int) n, 0, 63, stream) != cudaSuccess) return 1;
	size_t scan_bytes = 0;
	if (cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t*) nullptr, (uint32_t*) nullptr, (int) internal_count, stream) != cudaSuccess) return 1;
	unsigned char* cub_temp;
	if (!s.alloc(&cub_temp, sort_bytes > scan_bytes ? sort_bytes : scan_bytes)) return 1;
	if (cub::DeviceRadixSort::SortPairs(cub_temp, sort_bytes, codes_in, codes, index_in, order, (int) n, 0, 63, stream) != cudaSuccess) return 1;
	// 3. slots (outputs)
	float4* tris; uint32_t* tri_ids;
	if (cudaMalloc((void**) &tris, sizeof(float) * 12 * (size_t) n) != cudaSuccess) return 1;
	if (cudaMalloc((void**) &tri_ids, sizeof(uint32_t) * (size_t) n) != cudaSuccess) { cudaFree(tris); return 1; }
	auto fail = [&]() { cudaFree(tris); cudaFree(tri_ids); return 1; };
	slots_kernel<<<blocks, kThreads, 0, stream>>>(d_vertices, order, n, tris, tri_ids);
	// 4. radix tree
	if (!s.alloc(&first, internal_count) || !s.alloc(&last, internal_count) || !s.alloc(&split, internal_count) || !s.alloc(&parent, internal_count) || !s.alloc(&leaf_parent, n)
		|| !s.alloc(&node_lo, 3 * (size_t) internal_count) || !s.alloc(&node_hi, 3 * (size_t) internal_count) || !s.alloc(&arrivals, internal_count)
		|| !s.alloc(&used, internal_count) || !s.alloc(&rank, internal_count) || !s.alloc(&d_depth, 1)) return fail();
	cudaMemsetAsync(parent, 0xff, sizeof(int32_t) * (size_t) internal_count, stream);   // -1: the root has no parent
	cudaMemsetAsync(arrivals, 0, sizeof(uint32_t) * (size_t) internal_count, stream);
	cudaMemsetAsync(d_depth, 0, sizeof(uint32_t), stream);
	radix_tree_kernel<<<blocks, kThreads, 0, stream>>>(codes, n, first, last, split, parent, leaf_parent);
	// 5. boxes
	refit_kernel<<<blocks, kThreads, 0, stream>>>(n, order, box_lo, box_hi, first, last, split, parent, leaf_parent, node_lo, node_hi, arrivals);
	// 6. collapse + numbering
	used_kernel<<<blocks, kThreads, 0, stream>>>(internal_count, first, last, used);
	if (cub::DeviceScan::ExclusiveSum(cub_temp, scan_bytes, used, rank, (int) internal_count, stream) != cudaSuccess) return fail();
	uint32_t last_rank = 0, last_used = 0;
	if (cudaMemcpyAsync(&last_rank, rank + (internal_count - 1), 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess
		|| cudaMemcpyAsync(&last_used, used + (internal_count - 1), 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess) return fail();
	const uint32_t used_count = last_rank + last_used;
	// 7. node pairs, 8. depth
	float* nodes;
	if (cudaMalloc((void**) &nodes, sizeof(float) * 16 * (size_t) (used_count ? used_count : 1)) != cudaSuccess) return fail();
	emit_kernel<<<blocks, kThreads, 0, stream>>>(internal_count, order, box_lo, box_hi, node_lo, node_hi, first, last, split, used, rank, pad, nodes);
	depth_kernel<<<blocks, kThreads, 0, stream>>>(internal_count, used, parent, d_depth);
	uint32_t depth = 0;
	if (cudaMemcpyAsync(&depth, d_depth, 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) {
		cudaFree(nodes); return fail();
	}
	*d_nodes = nodes; *d_tris = tris; *d_tri_ids = tri_ids; *node_count = used_count; *max_depth = depth;
	return 0;
}

} // namespace vkr


// ------------------------------------------------------------------------------------------------
// Interleaved node pairs for the trace warps (vkr_trace.cuh): one thread per pair
namespace vkr {
__global__ void interleave_pairs_kernel(const float4* __restrict__ nodes, unsigned long long count, float4* __restrict__ out) {
	const unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count) return;
	float w[16];
	interleave_node_pair(nodes + 4 * i, w);
	for (int k = 0; k != 4; ++k) out[4 * i + k] = make_float4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
}
} // namespace vkr

cudaError_t vkr_interleave_node_pairs(const float4* d_nodes, uint64_t pair_count, float4* d_nodes_i, cudaStream_t stream) {
	if (!pair_count) return cudaSuccess;
	vkr::interleave_pairs_kernel<<<(unsigned) ((pair_count + 255) / 256), 256, 0, stream>>>(d_nodes, (unsigned long long) pair_count, d_nodes_i);
	return cudaGetLastError();
}

namespace vkr {
// For the host code (vkr_host.cpp): allocates the interleaved pairs and fills them from the float pairs on the device
int interleave_node_pairs_device(const void* d_nodes, uint64_t pair_count, void** d_nodes_i, void* stream) {
	*d_nodes_i = nullptr;
	if (cudaMalloc(d_nodes_i, 64 * (size_t) (pair_count ? pair_count : 1)) != cudaSuccess) { *d_nodes_i = nullptr; return 1; }
	if (vkr_interleave_node_pairs((const float4*) d_nodes, pair_count, (float4*) *d_nodes_i, (cudaStream_t) stream) != cudaSuccess || cudaStreamSynchronize((cudaStream_t) stream) != cudaSuccess) {
		cudaFree(*d_nodes_i); *d_nodes_i = nullptr; return 1;
	}
	return 0;
}
}
