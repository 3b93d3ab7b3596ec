// vkr_api.cu -- frame-side C-ABI: G-buffer producer passes, the shading pass object and the
// device probes used by the parity tests. Replaces create_shading_pass (src/main.c:598-940), the
// subpass-1 draw (src/main.c:1429-1434) and the per-frame part of render_frame (src/main.c:2197-2270).
// Compile with -fmad=false (the probe kernels call the same device math as the megakernel).
#include "../../include/vkr_b200.h"
#include "vkr_internal.h"
#include "vkr_kernels.h"
#include "vkr_psa.cuh"
#include "vkr_trace.cuh"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

using namespace vkr;

uint32_t vkr_share_first_column(const vkr_shading_pass_desc_t& d, uint32_t band);

#define VKR_CUDA_OK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { printf("%s: %s\n", what, cudaGetErrorString(e_)); return 1; } } while (0)

extern "C" size_t vkr_gbuffer_size(uint32_t width, uint32_t height) { return (size_t) width * height * 4 * sizeof(float) * 4; }

// ------------------------------------------------------------------------------------------------
// G-buffer producer
// ------------------------------------------------------------------------------------------------
static int fill_gbuffer_params(gbuffer_kernel_params& p, void** d_constants, const vkr_device_t* device, const vkr_scene_t* scene, const void* constants, uint32_t width, uint32_t height) {
	memset(&p, 0, sizeof(p));
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaMallocAsync(d_constants, 256, stream), "Failed to allocate constants for the G-buffer producer");
	VKR_CUDA_OK(cudaMemcpyAsync(*d_constants, constants, 256, cudaMemcpyHostToDevice, stream), "Failed to upload constants for the G-buffer producer");
	p.width = (int) width; p.height = (int) height;
	p.constants = (const unsigned char*) *d_constants;
	p.quantized_positions = (const uint2*) scene->d_quantized_positions;
	p.normals_and_tex_coords = (const ushort4*) scene->d_normals_and_tex_coords;
	p.material_indices = (const uint8_t*) scene->d_material_indices;
	p.material_params = (const float*) scene->d_material_params;
	if (scene->textured) {
		p.texture_data = (const float4*) scene->d_texture_data; p.texture_dims = (const uint4*) scene->d_texture_dims; p.texture_offsets = (const unsigned long long*) scene->d_texture_offsets;
	}
	p.bvh_nodes = (const float4*) scene->d_primary_nodes; p.bvh_tris = (const float4*) scene->d_primary_tris; p.bvh_tri_ids = (const uint32_t*) scene->d_primary_tri_ids;
	p.tri_count = (uint32_t) scene->triangle_count;
	return 0;
}

extern "C" int vkr_run_visibility_pass(const vkr_device_t* device, const vkr_scene_t* scene, const void* constants, uint32_t width, uint32_t height, void* d_visibility) {
	if (!scene->d_primary_nodes) { printf("Cannot run the visibility pass: the scene was loaded without acceleration structure.\n"); return 1; }
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	gbuffer_kernel_params p; void* d_constants = nullptr;
	if (fill_gbuffer_params(p, &d_constants, device, scene, constants, width, height)) return 1;
	p.visibility = (uint32_t*) d_visibility;
	cudaError_t err = vkr_launch_visibility_kernel(p, (cudaStream_t) device->stream);
	cudaFreeAsync(d_constants, (cudaStream_t) device->stream);
	VKR_CUDA_OK(err, "Failed to launch the visibility kernel");
	return 0;
}

extern "C" int vkr_run_gbuffer_pass(const vkr_device_t* device, const vkr_scene_t* scene, const void* constants, uint32_t width, uint32_t height, const void* d_visibility, void* d_gbuffer) {
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	gbuffer_kernel_params p; void* d_constants = nullptr;
	if (fill_gbuffer_params(p, &d_constants, device, scene, constants, width, height)) return 1;
	p.visibility = (uint32_t*) d_visibility;
	p.gbuffer = (float4*) d_gbuffer;
	cudaError_t err = vkr_launch_gbuffer_kernel(p, (cudaStream_t) device->stream);
	cudaFreeAsync(d_constants, (cudaStream_t) device->stream);
	VKR_CUDA_OK(err, "Failed to launch the G-buffer kernel");
	return 0;
}

// ------------------------------------------------------------------------------------------------
// shading pass
// ------------------------------------------------------------------------------------------------
extern "C" void vkr_destroy_shading_pass(vkr_shading_pass_t* pass, const vkr_device_t* device) {
	(void) device;
	if (pass->d_constants) cudaFree(pass->d_constants);
	if (pass->h_constants_pinned) cudaFreeHost(pass->h_constants_pinned);
	if (pass->d_gbuffer_staging) cudaFree(pass->d_gbuffer_staging);
	if (pass->d_out_staging) cudaFree(pass->d_out_staging);
	if (pass->event_begin) cudaEventDestroy((cudaEvent_t) pass->event_begin);
	if (pass->event_end) cudaEventDestroy((cudaEvent_t) pass->event_end);
	if (pass->event_constants) cudaEventDestroy((cudaEvent_t) pass->event_constants);
	if (pass->event_costs) cudaEventDestroy((cudaEvent_t) pass->event_costs);
	if (pass->d_tile_list) cudaFree(pass->d_tile_list);
	if (pass->h_tile_list) cudaFreeHost(pass->h_tile_list);
	if (pass->d_tile_cost) cudaFree(pass->d_tile_cost);
	if (pass->h_tile_cost) cudaFreeHost(pass->h_tile_cost);
	memset(pass, 0, sizeof(*pass));
}

extern "C" int vkr_create_shading_pass(vkr_shading_pass_t* pass, const vkr_device_t* device, const vkr_shading_pass_desc_t* desc) {
	memset(pass, 0, sizeof(*pass));
	pass->desc = *desc;
	vkr_shading_pass_desc_t& d = pass->desc;
	if (d.stripe_count == 0) d.stripe_count = 1;
	// Legality rules of the reference's settings panel (src/user_interface.cpp:90-180), plus what this library implements
	const int technique = (int) d.polygon_sampling_technique;
	if (technique < (int) vkr_sample_polygon_baseline || technique > (int) vkr_sample_polygon_projected_solid_angle_biased) {
		printf("Failed to create the shading pass: unknown polygon sampling technique %d.\n", technique);
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	if (technique < (int) vkr_sample_polygon_projected_solid_angle) {
		// the related-work techniques sample the diffuse lobe only; GGX MIS needs a density that can be evaluated on its own
		const bool ggx_ok = technique == vkr_sample_polygon_rectangle_solid_angle_urena || technique == vkr_sample_polygon_solid_angle_arvo || technique == vkr_sample_polygon_solid_angle
			|| technique == vkr_sample_polygon_clipped_solid_angle || technique == vkr_sample_polygon_projected_solid_angle_arvo;
		if (!(d.sampling_strategies == vkr_sampling_strategies_diffuse_only || (d.sampling_strategies == vkr_sampling_strategies_diffuse_ggx_mis && ggx_ok))) {
			printf("Failed to create the shading pass: polygon sampling technique %d does not support sampling strategy %d.\n", technique, (int) d.sampling_strategies);
			memset(pass, 0, sizeof(*pass)); return 1;
		}
	}
	if (d.error_display != vkr_error_display_none) {
		// the shader evaluates ERROR_DISPLAY_* in its projected solid angle branches only (shading_pass.frag.glsl:468, 489, 549, 555)
		const int e = (int) d.error_display;
		const bool combined = (int) d.sampling_strategies >= (int) vkr_sampling_strategies_diffuse_specular_separately;
		if (e < 0 || e > 6 || technique < (int) vkr_sample_polygon_projected_solid_angle_arvo || (e >= 4 && (!combined || technique == (int) vkr_sample_polygon_projected_solid_angle_arvo))
			|| (technique == (int) vkr_sample_polygon_projected_solid_angle_arvo && e == (int) vkr_error_display_diffuse_forward))
		{
			printf("Failed to create the shading pass: error display %d is not available with polygon sampling technique %d and sampling strategy %d.\n", e, technique, (int) d.sampling_strategies);
			memset(pass, 0, sizeof(*pass)); return 1;
		}
	}
	if ((int) d.sampling_strategies < 0 || (int) d.sampling_strategies > 4 || (int) d.mis_heuristic < 0 || (int) d.mis_heuristic > 4) {
		printf("Failed to create the shading pass: invalid sampling strategy or MIS heuristic.\n");
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	if (d.sampling_strategies == vkr_sampling_strategies_diffuse_ggx_mis && d.mis_heuristic != vkr_mis_heuristic_balance && d.mis_heuristic != vkr_mis_heuristic_power) {
		printf("Failed to create the shading pass: GGX importance sampling supports the balance and power heuristics only.\n");
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	if (d.max_polygonal_light_vertex_count < 3 || d.max_polygonal_light_vertex_count > 7 || d.min_polygonal_light_vertex_count < 3 || d.min_polygonal_light_vertex_count > d.max_polygonal_light_vertex_count) {
		printf("Failed to create the shading pass: polygonal lights must have 3 to 7 vertices (got min %u, max %u).\n", d.min_polygonal_light_vertex_count, d.max_polygonal_light_vertex_count);
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	if (!d.width || !d.height || d.stripe_index >= d.stripe_count || !d.sample_count || !d.ltc_table || !d.noise_table || !d.ltc_table->d_table0 || !d.noise_table->d_noise) {
		printf("Failed to create the shading pass: invalid resolution, stripe, sample count or missing LTC / noise tables.\n");
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	if (d.trace_shadow_rays && (!d.scene || !d.scene->d_shadow_nodes)) {
		printf("Failed to create the shading pass: shadow rays requested but the scene has no acceleration structure.\n");
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	if (cudaSetDevice(device->cuda_device) != cudaSuccess) { memset(pass, 0, sizeof(*pass)); return 1; }
	const uint32_t v = d.max_polygonal_light_vertex_count;
	pass->constants_size = 256 + (size_t) d.polygonal_light_count * (160 + 16 * (size_t) v * 2 + 16 * (size_t) (v - 2));
	if (pass->constants_size > 160 * 1024) {
		printf("Failed to create the shading pass: %u lights do not fit into shared memory.\n", d.polygonal_light_count);
		memset(pass, 0, sizeof(*pass)); return 1;
	}
	cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr, e3 = nullptr;
	// The tiles of this instance (column tx of every tile row with tx % stripe_count == stripe_index), row-major: the launch order of the first frame
	const uint32_t tiles_x = (d.width + VKR_TILE_WIDTH - 1) / VKR_TILE_WIDTH, tiles_y = (d.height + VKR_TILE_ROW_HEIGHT - 1) / VKR_TILE_ROW_HEIGHT;
	std::vector<uint32_t> tiles;
	for (uint32_t ty = 0; ty != tiles_y; ++ty) // the columns of a share move on by one every VKR_TILE_BAND_ROWS tile rows (see vkr_share_first_column)
		for (uint32_t tx = vkr_share_first_column(d, ty / VKR_TILE_BAND_ROWS); tx < tiles_x; tx += d.stripe_count) tiles.push_back(ty * tiles_x + tx);
	pass->tile_count = (uint32_t) tiles.size();
	const size_t list_bytes = sizeof(uint32_t) * (tiles.empty() ? 1 : tiles.size()), cost_bytes = sizeof(uint32_t) * (size_t) tiles_x * tiles_y;
	if (cudaMalloc(&pass->d_constants, pass->constants_size) != cudaSuccess || cudaMallocHost(&pass->h_constants_pinned, pass->constants_size) != cudaSuccess
		|| cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess
		|| cudaEventCreateWithFlags(&e2, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e3, cudaEventDisableTiming) != cudaSuccess
		|| cudaMalloc(&pass->d_tile_list, list_bytes) != cudaSuccess || cudaMallocHost(&pass->h_tile_list, list_bytes) != cudaSuccess
		|| cudaMalloc(&pass->d_tile_cost, cost_bytes) != cudaSuccess || cudaMallocHost(&pass->h_tile_cost, cost_bytes) != cudaSuccess
		|| cudaMemset(pass->d_tile_cost, 0, cost_bytes) != cudaSuccess)
	{
		printf("Failed to allocate constant buffers for the shading pass.\n");
		pass->event_begin = e0; pass->event_end = e1; pass->event_constants = e2; pass->event_costs = e3;
		vkr_destroy_shading_pass(pass, device); return 1;
	}
	pass->event_begin = e0; pass->event_end = e1; pass->event_constants = e2; pass->event_costs = e3;
	memcpy(pass->h_tile_list, tiles.data(), sizeof(uint32_t) * tiles.size());
	if (cudaMemcpy(pass->d_tile_list, pass->h_tile_list, list_bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
		printf("Failed to upload the tile list of the shading pass.\n");
		vkr_destroy_shading_pass(pass, device); return 1;
	}
	const char* order = getenv("VKR_TILE_ORDER");   // "static": keep the row-major order (tuning experiments)
	pass->reorder_tiles = !(order && !strcmp(order, "static"));
	return 0;
}

// Launch order of the next frame: the tiles of this instance sorted by what they cost in the frame before, dearest first (longest processing time first:
// the hardware hands out CTAs in index order, so the frame ends on cheap tiles instead of on whatever the bottom rows hold). Called when the costs of the
// previous frame have arrived on the host; equal costs keep their row-major order, so the order is deterministic.
static void reorder_tiles_by_cost(vkr_shading_pass_t* pass) {
	uint32_t* list = (uint32_t*) pass->h_tile_list;
	const uint32_t* cost = (const uint32_t*) pass->h_tile_cost;
	std::sort(list, list + pass->tile_count); // row-major first: ties below are then independent of the previous order
	std::stable_sort(list, list + pass->tile_count, [cost](uint32_t a, uint32_t b) { return cost[a] > cost[b]; });
}

cudaError_t vkr_launch_shading_kernel(const vkr::shading_kernel_params& p, cudaStream_t stream) {
	if (p.light_texture_count != 0 && p.polygon_sampling_technique < 11 && p.error_display == 0) { // related-work techniques under textured lights
		switch (p.max_light_vertex_count) {
		case 3: return vkr_launch_textured_related_work_kernel_maxv3(p, stream);
		case 4: return vkr_launch_textured_related_work_kernel_maxv4(p, stream);
		case 5: return vkr_launch_textured_related_work_kernel_maxv5(p, stream);
		case 6: return vkr_launch_textured_related_work_kernel_maxv6(p, stream);
		case 7: return vkr_launch_textured_related_work_kernel_maxv7(p, stream);
		default: return cudaErrorInvalidValue;
		}
	}
	if (p.polygon_sampling_technique < 11 || p.error_display != 0) { // related-work techniques and error display (SURVEY 8 f4)
		switch (p.max_light_vertex_count) {
		case 3: return vkr_launch_related_work_kernel_maxv3(p, stream);
		case 4: return vkr_launch_related_work_kernel_maxv4(p, stream);
		case 5: return vkr_launch_related_work_kernel_maxv5(p, stream);
		case 6: return vkr_launch_related_work_kernel_maxv6(p, stream);
		case 7: return vkr_launch_related_work_kernel_maxv7(p, stream);
		default: return cudaErrorInvalidValue;
		}
	}
	if (p.light_texture_count != 0) { // at least one textured light in this frame (vkr_textured_light_kernel.cu)
		switch (p.max_light_vertex_count) {
		case 3: return vkr_launch_textured_light_kernel_maxp4(p, stream);
		case 4: return vkr_launch_textured_light_kernel_maxp5(p, stream);
		case 5: return vkr_launch_textured_light_kernel_maxp6(p, stream);
		case 6: return vkr_launch_textured_light_kernel_maxp7(p, stream);
		case 7: return vkr_launch_textured_light_kernel_maxp8(p, stream);
		default: return cudaErrorInvalidValue;
		}
	}
	switch (p.max_light_vertex_count) { // MAX_POLYGONAL_LIGHT_VERTEX_COUNT, a compile-time bound of the kernels
	case 3: return vkr_launch_shading_kernel_maxp4(p, stream);
	case 4: return vkr_launch_shading_kernel_maxp5(p, stream);
	case 5: return vkr_launch_shading_kernel_maxp6(p, stream);
	case 6: return vkr_launch_shading_kernel_maxp7(p, stream);
	case 7: return vkr_launch_shading_kernel_maxp8(p, stream);
	default: return cudaErrorInvalidValue;
	}
}

// exchange: when not null, the pixels also go into the frames of the other GPUs (vkr_exchange.cu fills peer_outs)
int vkr_launch_shading(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out, unsigned long long* d_stats,
	int peer_count, void* const* peer_outs)
{
	const vkr_shading_pass_desc_t& d = pass->desc;
	if (constants_size != pass->constants_size) {
		printf("The constant block has %llu bytes but the shading pass was created for %llu bytes (%u lights with up to %u vertices).\n",
			(unsigned long long) constants_size, (unsigned long long) pass->constants_size, d.polygonal_light_count, d.max_polygonal_light_vertex_count);
		return 1;
	}
	bool any_textured_light = false;
	{ // light blocks must match what the pass was created for (the reference recompiles the shader when they change)
		const uint32_t v = d.max_polygonal_light_vertex_count;
		const size_t stride = 160 + 16 * (size_t) v * 2 + 16 * (size_t) (v - 2);
		for (uint32_t i = 0; i != d.polygonal_light_count; ++i) {
			uint32_t vertex_count, texturing_technique, texture_index;
			memcpy(&vertex_count, (const char*) constants + 256 + stride * i + 80, 4);
			memcpy(&texturing_technique, (const char*) constants + 256 + stride * i + 84, 4);
			memcpy(&texture_index, (const char*) constants + 256 + stride * i + 88, 4);
			if (vertex_count < d.min_polygonal_light_vertex_count || vertex_count > v) {
				printf("Polygonal light %u has %u vertices but the shading pass was created for %u to %u.\n", i, vertex_count, d.min_polygonal_light_vertex_count, v);
				return 1;
			}
			if (texturing_technique != 0) { // polygon_texturing_technique_t: 1 area, 2 portal, 3 IES profile
				any_textured_light = true;
				if (texturing_technique > 3 || !d.light_textures || !d.light_textures->d_texels || texture_index >= d.light_textures->texture_count) {
					printf("Polygonal light %u is textured (technique %u, texture %u) but the shading pass has %u light textures on the device.\n", i, texturing_technique, texture_index,
						(d.light_textures && d.light_textures->d_texels) ? d.light_textures->texture_count : 0u);
					return 1;
				}
			}
		}
		if (any_textured_light && d.error_display != 0) { // the error display shows no radiance; it has no textured variant
			printf("The error display (%d) is not available with textured polygonal lights.\n", (int) d.error_display);
			return 1;
		}
	}
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	// The call is asynchronous: the previous frame's copy out of the pinned staging buffer may not have run yet (it queues behind that frame's kernel)
	if (pass->kernel_launches) VKR_CUDA_OK(cudaEventSynchronize((cudaEvent_t) pass->event_constants), "Failed to wait for the previous upload of the constant block");
	memcpy(pass->h_constants_pinned, constants, constants_size);
	VKR_CUDA_OK(cudaMemcpyAsync(pass->d_constants, pass->h_constants_pinned, constants_size, cudaMemcpyHostToDevice, stream), "Failed to upload the constant block");
	VKR_CUDA_OK(cudaEventRecord((cudaEvent_t) pass->event_constants, stream), "Failed to record the upload of the constant block");
	shading_kernel_params p; memset(&p, 0, sizeof(p));
	p.width = (int) d.width; p.height = (int) d.height;
	p.tile_count = (int) pass->tile_count;
	const bool whole_frame = d.stripe_count == 1;
	if (pass->reorder_tiles && pass->costs_pending && cudaEventQuery((cudaEvent_t) pass->event_costs) == cudaSuccess) {
		// the costs of an earlier frame are here: new launch order. The list's last upload ran before that frame's kernel, so the staging buffer is free.
		pass->costs_pending = 0;
		reorder_tiles_by_cost(pass);
		VKR_CUDA_OK(cudaMemcpyAsync(pass->d_tile_list, pass->h_tile_list, sizeof(uint32_t) * pass->tile_count, cudaMemcpyHostToDevice, stream), "Failed to upload the tile order");
	}
	p.tile_list = (whole_frame && !pass->reorder_tiles) ? nullptr : (const uint32_t*) pass->d_tile_list;
	const bool record_costs = pass->reorder_tiles && !pass->costs_pending && !d_stats;
	if (record_costs) {
		const size_t cost_bytes = sizeof(uint32_t) * (size_t) ((d.width + VKR_TILE_WIDTH - 1) / VKR_TILE_WIDTH) * ((d.height + VKR_TILE_ROW_HEIGHT - 1) / VKR_TILE_ROW_HEIGHT);
		VKR_CUDA_OK(cudaMemsetAsync(pass->d_tile_cost, 0, cost_bytes, stream), "Failed to clear the tile costs");
		p.tile_cost = (uint32_t*) pass->d_tile_cost;
	}
	if (peer_count < 0 || peer_count > 7) return 1;
	p.out_peer_count = peer_count;
	for (int k = 0; k != peer_count; ++k) p.out_peers[k] = (float4*) peer_outs[k];
	p.gbuffer = (const float4*) d_gbuffer; p.out = (float4*) d_out;
	p.constants = (const unsigned char*) pass->d_constants;
	p.constants_bytes = (uint32_t) constants_size;
	p.constants_smem_bytes = (uint32_t) ((constants_size + 127) / 128 * 128);
	p.light_count = (int) d.polygonal_light_count; p.max_light_vertex_count = (int) d.max_polygonal_light_vertex_count; p.sample_count = (int) d.sample_count;
	p.sampling_strategies = (int) d.sampling_strategies; p.mis_heuristic = (int) d.mis_heuristic;
	p.biased_sampling = d.polygon_sampling_technique == vkr_sample_polygon_projected_solid_angle_biased;
	p.polygon_sampling_technique = (int) d.polygon_sampling_technique;
	p.error_display = (int) d.error_display;
	p.trace_shadow_rays = d.trace_shadow_rays; p.show_polygonal_lights = d.show_polygonal_lights; p.output_srgb = d.output_srgb;
	p.noise = (const uint16_t*) d.noise_table->d_noise; p.noise_w = (int) d.noise_table->width; p.noise_h = (int) d.noise_table->height; p.noise_layers = (int) d.noise_table->layers;
	p.ltc0 = (const uint16_t*) d.ltc_table->d_table0; p.ltc1 = (const uint16_t*) d.ltc_table->d_table1;
	p.ltc_res = (int) d.ltc_table->roughness_count; p.ltc_layers = (int) d.ltc_table->fresnel_count;
	p.stack_depth = 4;
	if (d.trace_shadow_rays) {
		p.bvh_nodes = (const float4*) d.scene->d_shadow_nodes; p.bvh_tris = (const float4*) d.scene->d_shadow_tris; p.tri_count = (uint32_t) d.scene->triangle_count;
		p.stack_depth = (int) d.scene->shadow_max_depth + 2;
		p.bvh_width = d.scene->shadow_bvh_width ? (int) d.scene->shadow_bvh_width : 2;
		p.bvh_nodes_q = (const uint4*) d.scene->d_shadow_nodes_quantised;
		p.bvh_nodes_i = (const float4*) d.scene->d_shadow_nodes_interleaved;
		if (p.bvh_width == 2 && !p.bvh_nodes_i) { printf("The scene holds no interleaved node pairs for the shadow rays (a scene object that was not made by this library?).\n"); return 1; }
		for (int k = 0; k != 6; ++k) p.bvh_grid[k] = d.scene->shadow_grid[k];
	}
	if (any_textured_light) {
		p.light_texture_texels = (const float4*) d.light_textures->d_texels; p.light_texture_dims = (const uint4*) d.light_textures->d_dims;
		p.light_texture_offsets = (const unsigned long long*) d.light_textures->d_offsets; p.light_texture_count = d.light_textures->texture_count;
	}
	if (d_stats) { // the counters edition exists for the projected solid angle kernels of quad lights (what the benchmark configurations run)
		if (p.max_light_vertex_count != 4 || p.polygon_sampling_technique < 11 || p.error_display != 0 || any_textured_light) {
			printf("Trace counters are available for projected solid angle sampling of untextured lights with up to 4 vertices only.\n");
			return 1;
		}
		p.stats = d_stats;
	}
	if (pass->timing_enabled) cudaEventRecord((cudaEvent_t) pass->event_begin, stream);
	cudaError_t err = d_stats ? vkr_launch_shading_kernel_stats_maxp5(p, stream) : vkr_launch_shading_kernel(p, stream);
	if (pass->timing_enabled) cudaEventRecord((cudaEvent_t) pass->event_end, stream);
	VKR_CUDA_OK(err, "Failed to launch the shading kernel");
	++pass->kernel_launches;
	if (record_costs) { // read back what the tiles cost; looked at when a later frame is launched
		const size_t cost_bytes = sizeof(uint32_t) * (size_t) ((d.width + VKR_TILE_WIDTH - 1) / VKR_TILE_WIDTH) * ((d.height + VKR_TILE_ROW_HEIGHT - 1) / VKR_TILE_ROW_HEIGHT);
		if (cudaMemcpyAsync(pass->h_tile_cost, pass->d_tile_cost, cost_bytes, cudaMemcpyDeviceToHost, stream) == cudaSuccess && cudaEventRecord((cudaEvent_t) pass->event_costs, stream) == cudaSuccess)
			pass->costs_pending = 1;
	}
	return 0;
}

static int launch_shading(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out, unsigned long long* d_stats = nullptr) {
	return vkr_launch_shading(pass, device, constants, constants_size, d_gbuffer, d_out, d_stats, 0, nullptr);
}

// First tile column of this instance in band `band` (VKR_TILE_BAND_ROWS tile rows): column tx of the band belongs to instance (tx + band) % stripe_count.
uint32_t vkr_share_first_column(const vkr_shading_pass_desc_t& d, uint32_t band) {
	return (d.stripe_index + d.stripe_count - band % d.stripe_count) % d.stripe_count;
}

// This instance's part of one plane (or of the frame), host <-> device. A plane is rows of `texel` bytes per pixel; the instance owns tile column tx of
// every row if tx % stripe_count == stripe_index, which makes its part a 2D array of 16-pixel segments with a pitch of stripe_count segments: one strided copy.
int vkr_copy_tile_columns(const vkr_shading_pass_desc_t& d, void* dst, const void* src, size_t texel, cudaMemcpyKind kind, cudaStream_t stream) {
	const size_t row_bytes = (size_t) d.width * texel, seg = (size_t) VKR_TILE_WIDTH * texel;
	if (d.stripe_count == 1) return cudaMemcpyAsync(dst, src, row_bytes * d.height, kind, stream) != cudaSuccess;
	const size_t pitch = seg * d.stripe_count;
	const uint32_t band_rows = VKR_TILE_BAND_ROWS * VKR_TILE_ROW_HEIGHT;
	for (uint32_t y0 = 0, band = 0; y0 < d.height; y0 += band_rows, ++band) { // one band of tile rows: the instance owns the same columns in all of its rows
		const uint32_t rows = (y0 + band_rows <= d.height) ? band_rows : d.height - y0;
		const size_t first = seg * vkr_share_first_column(d, band), base = row_bytes * y0;
		if (row_bytes % pitch == 0) { // every row holds the same number of whole segments of this instance: the rows of the band chain into one 2D array
			if (cudaMemcpy2DAsync((char*) dst + base + first, pitch, (const char*) src + base + first, pitch, seg, (row_bytes / pitch) * rows, kind, stream) != cudaSuccess) return 1;
			continue;
		}
		for (uint32_t y = 0; y != rows; ++y) { // ragged rows: whole segments as a 2D copy per row, then the narrow last segment if it is ours
			const size_t row = base + row_bytes * y;
			size_t whole = 0, tail_at = 0, tail = 0;
			for (size_t at = first; at < row_bytes; at += pitch) { if (at + seg <= row_bytes) ++whole; else { tail_at = at; tail = row_bytes - at; } }
			if (whole && cudaMemcpy2DAsync((char*) dst + row + first, pitch, (const char*) src + row + first, pitch, seg, whole, kind, stream) != cudaSuccess) return 1;
			if (tail && cudaMemcpyAsync((char*) dst + row + tail_at, (const char*) src + row + tail_at, tail, kind, stream) != cudaSuccess) return 1;
		}
	}
	return 0;
}

extern "C" int vkr_shading_pass_run(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out_rgba32f) {
	return launch_shading(pass, device, constants, constants_size, d_gbuffer, d_out_rgba32f);
}

extern "C" int vkr_shading_pass_run_with_counters(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out_rgba32f, uint64_t* out_counters) {
	static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "counter type");
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	unsigned long long* d_stats = nullptr;
	VKR_CUDA_OK(cudaMalloc(&d_stats, sizeof(uint64_t) * VKR_TRACE_COUNTER_COUNT), "Failed to allocate the trace counters");
	cudaMemsetAsync(d_stats, 0, sizeof(uint64_t) * VKR_TRACE_COUNTER_COUNT, stream);
	int rc = launch_shading(pass, device, constants, constants_size, d_gbuffer, d_out_rgba32f, d_stats);
	if (!rc && cudaMemcpyAsync(out_counters, d_stats, sizeof(uint64_t) * VKR_TRACE_COUNTER_COUNT, cudaMemcpyDeviceToHost, stream) != cudaSuccess) rc = 1;
	if (cudaStreamSynchronize(stream) != cudaSuccess) { printf("The shading pass with trace counters failed: %s\n", cudaGetErrorString(cudaGetLastError())); rc = 1; }
	cudaFree(d_stats);
	if (!rc && pass->timing_enabled) { float ms = 0.0f; if (cudaEventElapsedTime(&ms, (cudaEvent_t) pass->event_begin, (cudaEvent_t) pass->event_end) == cudaSuccess) pass->last_kernel_ms = ms; }
	return rc;
}

extern "C" int vkr_shading_pass_wait(vkr_shading_pass_t* pass, const vkr_device_t* device) {
	VKR_CUDA_OK(cudaStreamSynchronize((cudaStream_t) device->stream), "Failed to wait for the shading pass");
	if (pass->timing_enabled && pass->kernel_launches) {
		float ms = 0.0f;
		if (cudaEventElapsedTime(&ms, (cudaEvent_t) pass->event_begin, (cudaEvent_t) pass->event_end) == cudaSuccess) pass->last_kernel_ms = ms;
	}
	return 0;
}

extern "C" int vkr_shading_pass_run_host(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const float* gbuffer, float* out_rgba32f) {
	const vkr_shading_pass_desc_t& d = pass->desc;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	const size_t plane_bytes = (size_t) d.width * d.height * 16;
	if (!pass->d_gbuffer_staging) {
		if (cudaMalloc(&pass->d_gbuffer_staging, 4 * plane_bytes) != cudaSuccess || cudaMalloc(&pass->d_out_staging, plane_bytes) != cudaSuccess) {
			printf("Failed to allocate device staging buffers for the shading pass.\n");
			return 1;
		}
	}
	// Upload only the tiles of this instance, plane by plane
	for (int k = 0; k != 4; ++k)
		if (vkr_copy_tile_columns(d, (char*) pass->d_gbuffer_staging + k * plane_bytes, (const char*) gbuffer + k * plane_bytes, 16, cudaMemcpyHostToDevice, stream)) { printf("Failed to upload the G-buffer.\n"); return 1; }
	if (launch_shading(pass, device, constants, constants_size, pass->d_gbuffer_staging, pass->d_out_staging)) return 1;
	if (vkr_copy_tile_columns(d, out_rgba32f, pass->d_out_staging, 16, cudaMemcpyDeviceToHost, stream)) { printf("Failed to download the frame.\n"); return 1; }
	return vkr_shading_pass_wait(pass, device);
}

// ------------------------------------------------------------------------------------------------
// probes for the parity tests
// ------------------------------------------------------------------------------------------------
namespace vkr {

__global__ void __launch_bounds__(128) trace_probe_kernel(bvh_view bvh, uint32_t ray_count, const float* rays, uint8_t* out) {
	__shared__ int stack[kMaxStackDepth * 128];
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= ray_count) return;
	const float* r = rays + 8 * (size_t) i;
	out[i] = occluded(bvh, make3(r[0], r[1], r[2]), make3(r[3], r[4], r[5]), r[6], r[7], stack + threadIdx.x, 128) ? 1 : 0;
}

template <int MAXP, bool BIASED>
__global__ void sample_probe_kernel(int vertex_count, const float* vertices, uint32_t n, const float* rnd, float* out_dirs, float* out_info) {
	f3 v[MAXP];
#pragma unroll
	for (int i = 0; i != MAXP; ++i) v[i] = (i < vertex_count) ? make3(vertices[3 * i], vertices[3 * i + 1], vertices[3 * i + 2]) : make3(0.0f, 0.0f, 0.0f);
	const int vc = clip_polygon<MAXP>(vertex_count, v);
	psa_polygon<MAXP> p;
	p.psa = 0.0f; p.inner_ellipse_0 = make2(0.0f, 0.0f);
#pragma unroll
	for (int i = 0; i != MAXP; ++i) p.sector_psa[i] = 0.0f;
	if (vc) prepare_psa<MAXP, BIASED>(p, vc, v);
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i == 0 && out_info) {
		out_info[0] = p.psa; out_info[1] = (vc && p.inner_ellipse_0.x > 0.0f) ? 1.0f : 0.0f; out_info[2] = (float) vc;
#pragma unroll
		for (int k = 0; k != 8; ++k) out_info[3 + k] = (k < MAXP) ? p.sector_psa[k < MAXP ? k : 0] : 0.0f;
	}
	if (i >= n || !vc) return;
	const f3 d = sample_psa<MAXP, BIASED>(p, make2(rnd[2 * i], rnd[2 * i + 1]));
	out_dirs[3 * i] = d.x; out_dirs[3 * i + 1] = d.y; out_dirs[3 * i + 2] = d.z;
}

// every float through rsqrt_ieee() and through its definition (vkr_device_math.cuh); a NaN answers a NaN, everything else has to agree bit for bit
__global__ void rsqrt_probe_kernel(unsigned long long* mismatches, unsigned int* first_bad) {
	const unsigned long long stride = (unsigned long long) gridDim.x * blockDim.x;
	unsigned local = 0;
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < (1ull << 32); i += stride) {
		const float x = __uint_as_float((unsigned) i);
		const float a = rsqrt_ieee(x), b = rsqrt_ieee_reference(x);
		if (__float_as_uint(a) != __float_as_uint(b) && !(a != a && b != b)) { ++local; atomicMin(first_bad, (unsigned) i); }
	}
	if (local) atomicAdd(mismatches, (unsigned long long) local);
}

} // namespace vkr

extern "C" int vkr_probe_rsqrt_exhaustive(const vkr_device_t* device, uint64_t* out_mismatches, uint32_t* out_first_mismatch_bits) {
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	cudaStream_t stream = (cudaStream_t) device->stream;
	unsigned long long* d_count = nullptr; unsigned int* d_first = nullptr;
	VKR_CUDA_OK(cudaMalloc(&d_count, sizeof(unsigned long long)), "Failed to allocate the probe's counter");
	if (cudaMalloc(&d_first, sizeof(unsigned int)) != cudaSuccess) { cudaFree(d_count); printf("Failed to allocate the probe's result.\n"); return 1; }
	cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), stream); cudaMemsetAsync(d_first, 0xff, sizeof(unsigned int), stream);
	vkr::rsqrt_probe_kernel<<<(device->sm_count > 0 ? device->sm_count : 132) * 8, 256, 0, stream>>>(d_count, d_first);
	cudaError_t err = cudaGetLastError();
	unsigned long long count = 0; unsigned int first = 0;
	cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, stream); cudaMemcpyAsync(&first, d_first, sizeof(first), cudaMemcpyDeviceToHost, stream);
	cudaError_t err2 = cudaStreamSynchronize(stream);
	cudaFree(d_count); cudaFree(d_first);
	VKR_CUDA_OK(err, "Failed to launch the reciprocal square root probe");
	VKR_CUDA_OK(err2, "The reciprocal square root probe failed");
	*out_mismatches = (uint64_t) count; *out_first_mismatch_bits = (uint32_t) first;
	return 0;
}

extern "C" int vkr_trace_shadow_rays(const vkr_device_t* device, const vkr_scene_t* scene, uint32_t ray_count, const float* rays, uint8_t* out_occluded) {
	if (!scene->d_shadow_nodes) { printf("Cannot trace shadow rays: the scene was loaded without acceleration structure.\n"); return 1; }
	if (scene->shadow_bvh_width == 4) { printf("The shadow-ray probe walks node pairs; the scene was loaded with 4-wide nodes (VKR_BVH_WIDTH=4).\n"); return 1; }
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	cudaStream_t stream = (cudaStream_t) device->stream;
	float* d_rays = nullptr; uint8_t* d_out = nullptr;
	VKR_CUDA_OK(cudaMalloc(&d_rays, sizeof(float) * 8 * (size_t) (ray_count ? ray_count : 1)), "Failed to allocate rays");
	if (cudaMalloc(&d_out, ray_count ? ray_count : 1) != cudaSuccess) { cudaFree(d_rays); printf("Failed to allocate ray results.\n"); return 1; }
	cudaMemcpyAsync(d_rays, rays, sizeof(float) * 8 * (size_t) ray_count, cudaMemcpyHostToDevice, stream);
	bvh_view bvh; bvh.nodes = (const float4*) scene->d_shadow_nodes; bvh.tris = (const float4*) scene->d_shadow_tris; bvh.tri_ids = nullptr; bvh.tri_count = (uint32_t) scene->triangle_count;
	if (ray_count) trace_probe_kernel<<<(ray_count + 127) / 128, 128, 0, stream>>>(bvh, ray_count, d_rays, d_out);
	cudaError_t err = cudaGetLastError();
	cudaMemcpyAsync(out_occluded, d_out, ray_count, cudaMemcpyDeviceToHost, stream);
	cudaError_t err2 = cudaStreamSynchronize(stream);
	cudaFree(d_rays); cudaFree(d_out);
	VKR_CUDA_OK(err, "Failed to launch the shadow ray probe");
	VKR_CUDA_OK(err2, "The shadow ray probe failed");
	return 0;
}

extern "C" int vkr_sample_polygon_batch(const vkr_device_t* device, uint32_t vertex_count, const float* vertices_xyz, int biased, uint32_t n, const float* random_numbers, float* out_dirs, float* out_info) {
	if (vertex_count < 3 || vertex_count > 7) { printf("The sampling probe supports 3 to 7 vertices.\n"); return 1; }
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	cudaStream_t stream = (cudaStream_t) device->stream;
	float *d_v = nullptr, *d_r = nullptr, *d_d = nullptr, *d_i = nullptr;
	const size_t nn = n ? n : 1;
	if (cudaMalloc(&d_v, sizeof(float) * 3 * 7) != cudaSuccess || cudaMalloc(&d_r, sizeof(float) * 2 * nn) != cudaSuccess || cudaMalloc(&d_d, sizeof(float) * 3 * nn) != cudaSuccess || cudaMalloc(&d_i, sizeof(float) * 11) != cudaSuccess) {
		cudaFree(d_v); cudaFree(d_r); cudaFree(d_d); cudaFree(d_i);
		printf("Failed to allocate buffers for the sampling probe.\n"); return 1;
	}
	if (cudaMemcpyAsync(d_v, vertices_xyz, sizeof(float) * 3 * vertex_count, cudaMemcpyHostToDevice, stream) != cudaSuccess
		|| cudaMemcpyAsync(d_r, random_numbers, sizeof(float) * 2 * (size_t) n, cudaMemcpyHostToDevice, stream) != cudaSuccess
		|| cudaMemsetAsync(d_d, 0, sizeof(float) * 3 * nn, stream) != cudaSuccess)
	{
		cudaFree(d_v); cudaFree(d_r); cudaFree(d_d); cudaFree(d_i);
		printf("Failed to upload the inputs of the sampling probe.\n"); return 1;
	}
	const unsigned blocks = (unsigned) ((nn + 127) / 128);
#define VKR_PROBE(V) case V: if (biased) sample_probe_kernel<V + 1, true><<<blocks, 128, 0, stream>>>(V, d_v, n, d_r, d_d, d_i); else sample_probe_kernel<V + 1, false><<<blocks, 128, 0, stream>>>(V, d_v, n, d_r, d_d, d_i); break;
	switch (vertex_count) { VKR_PROBE(3) VKR_PROBE(4) VKR_PROBE(5) VKR_PROBE(6) VKR_PROBE(7) default: break; }
#undef VKR_PROBE
	cudaError_t err = cudaGetLastError();
	cudaMemcpyAsync(out_dirs, d_d, sizeof(float) * 3 * (size_t) n, cudaMemcpyDeviceToHost, stream);
	if (out_info) cudaMemcpyAsync(out_info, d_i, sizeof(float) * 11, cudaMemcpyDeviceToHost, stream);
	cudaError_t err2 = cudaStreamSynchronize(stream);
	cudaFree(d_v); cudaFree(d_r); cudaFree(d_d); cudaFree(d_i);
	VKR_CUDA_OK(err, "Failed to launch the sampling probe");
	VKR_CUDA_OK(err2, "The sampling probe failed");
	return 0;
}
