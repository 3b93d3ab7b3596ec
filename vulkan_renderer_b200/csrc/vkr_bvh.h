// vkr_bvh.h -- host-side BVH2 builder producing the node-pair layout of vkr_trace.cuh.
// Replaces the driver's acceleration-structure build (vkCmdBuildAccelerationStructuresKHR,
// src/scene.c:354-378) for a triangle soup with stride 12 (scene.c:197-209).
#pragma once
#include <stdint.h>
#include <vector>

namespace vkr {

struct host_bvh {
	std::vector<float> nodes;       // 16 floats per inner node (4 x float4)
	std::vector<float> tris;        // 12 floats per triangle slot (3 x float4)
	std::vector<uint32_t> tri_ids;  // original triangle index per slot
	uint32_t max_depth = 0;
	uint64_t node_count = 0;
};

// vertices: 9 floats per triangle. The result is deterministic for a given input.
void build_bvh(host_bvh& out, const float* vertices, uint64_t triangle_count);

// Linear BVH (Morton order + Karras' radix tree + leaves of up to four triangles), vkr_lbvh.cpp: the sequential reference of the GPU
// builder. Same output layout, lower tree quality, identical traversal results.
void build_lbvh(host_bvh& out, const float* vertices, uint64_t triangle_count);
uint64_t lbvh_morton_code(const float centroid[3], const float lo[3], const float inv_extent[3]);

// The same builder on the GPU (vkr_lbvh_gpu.cu). vertices: HOST pointer; outputs: device allocations owned by the caller. stream: a cudaStream_t
// (void* like vkr_device_t::stream, so that this header needs no CUDA headers).
int build_lbvh_device(const float* vertices, uint64_t triangle_count, void* stream, void** d_nodes, void** d_tris, void** d_tri_ids, uint64_t* node_count, uint32_t* max_depth);

// Interleaved node pairs (vkr_trace.cuh: the two children's numbers side by side, 64 bytes per pair), made on the device from the float pairs (vkr_lbvh_gpu.cu)
int interleave_node_pairs_device(const void* d_nodes, uint64_t pair_count, void** d_nodes_i, void* stream);
// The grid of the quantised node pairs (vkr_trace.cuh: quantise_node_pair) for a tree whose root pair (16 floats) is given: the scene's bounding box
// with two cells to spare on every side, 65536 cells per axis; grid = minimum xyz, cells per world unit xyz
void shadow_grid_from_root(const float* root_pair, float grid[6]);

// 4-wide nodes collapsed from a BVH2 (vkr_bvh.cpp: build_bvh4_from_bvh2): groundwork for a traversal with half as many, fatter steps
// (DESIGN.md section 7). node = 128 B = 8 x float4: child c has centre and half extent at floats [6c, 6c + 6), its reference (same
// encoding as in the node pairs) as int bits at float 24 + c; unused children are empty leaves with a negative half extent.
struct host_bvh4 {
	std::vector<float> nodes;   // 32 floats per node
	uint32_t max_depth = 0;
	uint64_t node_count = 0;
};
void build_bvh4_from_bvh2(host_bvh4& out, const host_bvh& in);

enum bvh_builder { bvh_builder_sah = 0, bvh_builder_lbvh = 1, bvh_builder_lbvh_gpu = 2 };
// VKR_BVH_BUILDER = sah (default) | lbvh | lbvh_gpu
bvh_builder bvh_builder_from_environment();

} // namespace vkr
