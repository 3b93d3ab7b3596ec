// vkr_kernels.h -- host-visible launch interface of the CUDA kernels (internal to the library).
#pragma once
#ifndef VKR_DEVICE_CODE_ON_HOST   // tests/device_on_host.cpp supplies the few CUDA types itself
#include <cuda_runtime.h>
#endif
#include <stdint.h>

// numeric values = the reference's sampling_strategies_t / mis_heuristic_t (src/main.h:45-92)
enum { VKR_STRATEGY_DIFFUSE_ONLY = 0, VKR_STRATEGY_DIFFUSE_GGX_MIS = 1, VKR_STRATEGY_DIFFUSE_SPECULAR_SEPARATELY = 2,
	VKR_STRATEGY_DIFFUSE_SPECULAR_MIS = 3, VKR_STRATEGY_DIFFUSE_SPECULAR_RANDOM = 4 };
enum { VKR_MIS_BALANCE = 0, VKR_MIS_POWER = 1, VKR_MIS_WEIGHTED = 2, VKR_MIS_OPTIMAL_CLAMPED = 3, VKR_MIS_OPTIMAL = 4 };

namespace vkr {

struct shading_kernel_params {
	// frame
	int width, height;
	// Which 16x8 screen tiles this launch shades (multi-GPU: every GPU takes a share of the tiles, vkr_api.cu): CTA b shades tile
	// tile_list[b] (= ty * tiles_x + tx), or tile b of the whole frame when the list is null. The list is also the launch ORDER: the
	// pass sorts it by the cost measured in the previous frame, dearest first, so that the last wave of CTAs is made of cheap tiles.
	int tile_count; const uint32_t* tile_list;
	uint32_t* tile_cost;             // per tile of the frame: nanoseconds the CTA spent on it (atomicMax over its shading warps); null = not recorded
	// Multi-GPU frame exchange (vkr_frame_exchange_t): finished pixels are also stored into the frames of the other GPUs (peer
	// memory over NVLink) from the kernel's epilogue, so no gather pass follows. out_peer_count = 0 on a single GPU.
	int out_peer_count; float4* out_peers[7];
	const float4* gbuffer;           // 4 planes of width*height float4
	float4* out;                     // width*height float4, linear radiance * exposure, alpha 1
	const unsigned char* constants;  // device copy of the reference's constant block
	uint32_t constants_bytes;        // 256 + light_count * light_stride (multiple of 16)
	uint32_t constants_smem_bytes;   // constants_bytes rounded up to 128
	// what the reference passes as -D defines (src/main.c:752-792)
	int light_count, max_light_vertex_count, sample_count;
	int sampling_strategies, mis_heuristic, biased_sampling, trace_shadow_rays, show_polygonal_lights;
	int output_srgb;                 // !OUTPUT_LINEAR_RGB (src/main.c:790); the half-bit split follows frame_bits in the constant block
	// tables
	const uint16_t* noise; int noise_w, noise_h, noise_layers;
	const uint16_t* ltc0; const uint16_t* ltc1; int ltc_res, ltc_layers;
	// acceleration structure
	const float4* bvh_nodes; const float4* bvh_tris; uint32_t tri_count;
	const float4* bvh_nodes_i;       // the same node pairs with the two children interleaved (vkr_trace.cuh): what the trace warps walk
	int stack_depth;                 // traversal stack entries per lane (BVH depth + 2)
	int polygon_sampling_technique;  // sample_polygon_technique_t (src/polygonal_light.h:30-66); 0..10 run vkr_related_work_kernel.cu
	int error_display;               // error_display_t (src/main.h:92-112); != 0 runs error_display_kernel (vkr_related_work_kernel.cu)
	// light textures (vkr_light_textures_t); only the kernels of vkr_textured_light_kernel.cu read them. dims = {width, height, mip_count, -}, offsets in texels
	const float4* light_texture_texels; const uint4* light_texture_dims; const unsigned long long* light_texture_offsets; uint32_t light_texture_count;
	unsigned long long* stats;       // VKR_TRACE_COUNTER_COUNT device counters, only written by the counters edition of the kernels (-DVKR_TRACE_STATS); else null
};

struct gbuffer_kernel_params {
	int width, height;
	const unsigned char* constants;          // device copy of the 256-byte fixed block
	const uint2* quantized_positions;        // 3 per triangle (scene.h:56-62)
	const ushort4* normals_and_tex_coords;   // 3 per triangle
	const uint8_t* material_indices;         // 1 per triangle
	const float* material_params;            // 8 floats per material (materials whose textures are constant)
	const float4* bvh_nodes; const float4* bvh_tris; const uint32_t* bvh_tri_ids; uint32_t tri_count; // primary-ray BVH (shader-decoded vertices)
	uint32_t* visibility;                    // width*height primitive indices (0xFFFFFFFF = background)
	float4* gbuffer;                         // 4 planes
	// material textures that need filtering (vkr_texture.cuh), 3 per material {base colour, specular, normal}; null for constant materials
	const float4* texture_data; const uint4* texture_dims; const unsigned long long* texture_offsets; // dims = {width, height, mip_count, -}, offsets in texels
};

} // namespace vkr

cudaError_t vkr_launch_shading_kernel(const vkr::shading_kernel_params& p, cudaStream_t stream);   // dispatches on max_light_vertex_count (vkr_api.cu)
// The tile kernels' entry points: one object per kernel family and light vertex bound MAX_POLYGONAL_LIGHT_VERTEX_COUNT = 3 .. 7 (__graft_entry__.py)
typedef cudaError_t vkr_tile_launcher_t(const vkr::shading_kernel_params& p, cudaStream_t stream);
// vkr_shading_kernel.cu: projected solid angle sampling, and the counters edition of its quad-light kernels (-DVKR_TRACE_STATS)
vkr_tile_launcher_t vkr_launch_shading_kernel_v3, vkr_launch_shading_kernel_v4, vkr_launch_shading_kernel_v5, vkr_launch_shading_kernel_v6, vkr_launch_shading_kernel_v7;
vkr_tile_launcher_t vkr_launch_shading_kernel_stats_v4;
// vkr_textured_light_kernel.cu: the same for frames with textured lights
vkr_tile_launcher_t vkr_launch_textured_light_kernel_v3, vkr_launch_textured_light_kernel_v4, vkr_launch_textured_light_kernel_v5, vkr_launch_textured_light_kernel_v6, vkr_launch_textured_light_kernel_v7;
// vkr_related_work_kernel.cu: the related-work sampling techniques and the error display
vkr_tile_launcher_t vkr_launch_related_work_kernel_v3, vkr_launch_related_work_kernel_v4, vkr_launch_related_work_kernel_v5, vkr_launch_related_work_kernel_v6, vkr_launch_related_work_kernel_v7;
// and the sampling probe of the same samplers (vkr_sample_related_work_batch), one thread per sample. All pointers are device pointers;
// position_frame = 3 + 12 floats, out_ggx_lit = {GGX density factor, 1 if lit else 0}.
typedef cudaError_t vkr_related_work_probe_launcher_t(uint32_t technique, const unsigned char* light_block, const float* position_frame, uint32_t n, const float* random_numbers,
	float* out_dirs, float* out_densities, float* out_ggx_lit, cudaStream_t stream);
vkr_related_work_probe_launcher_t vkr_launch_related_work_probe_v3, vkr_launch_related_work_probe_v4, vkr_launch_related_work_probe_v5, vkr_launch_related_work_probe_v6, vkr_launch_related_work_probe_v7;
// vkr_textured_related_work_kernel.cu: the related-work sampling techniques for frames with textured lights
vkr_tile_launcher_t vkr_launch_textured_related_work_kernel_v3, vkr_launch_textured_related_work_kernel_v4, vkr_launch_textured_related_work_kernel_v5, vkr_launch_textured_related_work_kernel_v6, vkr_launch_textured_related_work_kernel_v7;
// float node pairs -> interleaved node pairs (vkr_lbvh_gpu.cu); d_nodes_i: 64 bytes per pair
cudaError_t vkr_interleave_node_pairs(const float4* d_nodes, uint64_t pair_count, float4* d_nodes_i, cudaStream_t stream);
cudaError_t vkr_launch_visibility_kernel(const vkr::gbuffer_kernel_params& p, cudaStream_t stream);
cudaError_t vkr_launch_gbuffer_kernel(const vkr::gbuffer_kernel_params& p, cudaStream_t stream);
