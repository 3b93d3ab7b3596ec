/* vkr_b200.h -- C-ABI of the H100-native (sm_90a) shading pass (libvkr_b200.so).
 *
 * Drop-in boundary for ONE path of MomentsInGraphics/vulkan_renderer: the per-pixel shading
 * pass (src/shaders/shading_pass.frag.glsl + polygon_sampling.glsl + the ray-query shadow test).
 * Conventions mirror the reference's C host code (SURVEY 8b): caller-owned structs, int return
 * (0 = success), a printf diagnostic on failure, the callee destroys what it built and leaves the
 * struct zeroed, destroy_* tolerates partially-built or zeroed objects, single caller thread.
 * No torch / C++ types appear here; device pointers are plain void*.
 *
 * Every entry point names the reference interface it replaces (file:line under /root/reference).
 */
#ifndef VKR_B200_H
#define VKR_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VKR_B200_ABI_VERSION 1
#define VKR_TILE_ROW_HEIGHT 8 /* pixel rows per screen-tile row */
#define VKR_TILE_WIDTH 16     /* pixel columns per screen tile: the unit of the multi-GPU split */
#define VKR_TILE_BAND_ROWS 8  /* tile rows per band of the multi-GPU split: the tile columns of a share move on by one from band to band */
#define VKR_MAX_GPUS 8        /* GPUs of one box that can share a frame (vkr_frame_exchange_t) */

/* ---- enums: numeric values equal the reference's (src/main.h:45-92, src/polygonal_light.h:28-67,
        src/noise_table.h:20-54) so that render_settings_t fields can be passed through unchanged */
typedef enum vkr_sampling_strategies_e {
	vkr_sampling_strategies_diffuse_only = 0,
	vkr_sampling_strategies_diffuse_ggx_mis = 1,
	vkr_sampling_strategies_diffuse_specular_separately = 2,
	vkr_sampling_strategies_diffuse_specular_mis = 3,
	vkr_sampling_strategies_diffuse_specular_random = 4
} vkr_sampling_strategies_t;

typedef enum vkr_mis_heuristic_e {
	vkr_mis_heuristic_balance = 0, vkr_mis_heuristic_power = 1, vkr_mis_heuristic_weighted = 2,
	vkr_mis_heuristic_optimal_clamped = 3, vkr_mis_heuristic_optimal = 4
} vkr_mis_heuristic_t;

/* sample_polygon_technique_t (src/polygonal_light.h:28-67). 11 and 12 work with every sampling strategy; the related-work
   techniques 0..10 (SURVEY 8 f4) with vkr_sampling_strategies_diffuse_only, and 2, 3, 4, 5, 10 also with
   vkr_sampling_strategies_diffuse_ggx_mis -- the rules of src/user_interface.cpp:124-175 */
typedef enum vkr_sample_polygon_technique_e {
	vkr_sample_polygon_baseline = 0,
	vkr_sample_polygon_area_turk = 1,
	vkr_sample_polygon_rectangle_solid_angle_urena = 2,
	vkr_sample_polygon_solid_angle_arvo = 3,
	vkr_sample_polygon_solid_angle = 4,
	vkr_sample_polygon_clipped_solid_angle = 5,
	vkr_sample_polygon_bilinear_cosine_warp_hart = 6,
	vkr_sample_polygon_bilinear_cosine_warp_clipping_hart = 7,
	vkr_sample_polygon_biquadratic_cosine_warp_hart = 8,
	vkr_sample_polygon_biquadratic_cosine_warp_clipping_hart = 9,
	vkr_sample_polygon_projected_solid_angle_arvo = 10,
	vkr_sample_polygon_projected_solid_angle = 11,
	vkr_sample_polygon_projected_solid_angle_biased = 12
} vkr_sample_polygon_technique_t;

/* error_display_t (src/main.h:92-112): colour-coded error of the first sample of projected solid angle sampling instead of shading.
   Available with techniques 10 (diffuse, backward errors only), 11 and 12; the specular variants need a diffuse + specular strategy. */
typedef enum vkr_error_display_e {
	vkr_error_display_none = 0,
	vkr_error_display_diffuse_backward = 1, vkr_error_display_diffuse_backward_scaled = 2, vkr_error_display_diffuse_forward = 3,
	vkr_error_display_specular_backward = 4, vkr_error_display_specular_backward_scaled = 5, vkr_error_display_specular_forward = 6
} vkr_error_display_t;

typedef enum vkr_noise_type_e { vkr_noise_type_white = 0, vkr_noise_type_blue = 1, vkr_noise_type_ahmed = 2 } vkr_noise_type_t;

/* ---- device (replaces create_vulkan_device, src/vulkan_basics.c:24; device_t, vulkan_basics.h:40-77) */
typedef struct vkr_device_s {
	int cuda_device;               /* ordinal handed to cudaSetDevice */
	int sm_count;                  /* 132 on H100 SXM */
	int ray_tracing_supported;     /* always 1: the software BVH needs no RT cores (scene.c:485 gate) */
	void* stream;                  /* cudaStream_t all asynchronous work is enqueued on */
	int owns_stream;
	char name[64];
} vkr_device_t;

/* stream may be NULL (the library creates one) or a caller's cudaStream_t (e.g. torch's current stream) */
int vkr_create_device(vkr_device_t* device, int cuda_device, void* stream);
void vkr_destroy_device(vkr_device_t* device);
/* blocks until everything enqueued on device->stream has finished (vkQueueWaitIdle, scene.c:395) */
int vkr_device_wait_idle(const vkr_device_t* device);

/* ---- scene (replaces load_scene / destroy_scene, src/scene.h:181-184, src/scene.c:409-581) */
typedef struct vkr_scene_s {
	uint64_t triangle_count, material_count;
	float dequantization_factor[3], dequantization_summand[3];
	char** material_names;                 /* material_count malloc'ed strings */
	float* material_params;                /* host: 8 floats per material {base.rgb, linear roughness, metalicity, normal.xy, 0} */
	/* device buffers, byte-identical to the reference's three mesh buffers (scene.h:56-83) */
	void* d_quantized_positions;           /* uint32[2] * 3 * triangle_count */
	void* d_normals_and_tex_coords;        /* uint16[4] * 3 * triangle_count */
	void* d_material_indices;              /* uint8 * triangle_count */
	void* d_material_params;
	/* software acceleration structures (replace VkAccelerationStructureKHR, scene.c:142-406) */
	void* d_shadow_nodes; void* d_shadow_tris;                 /* over the scene.c:175-187 float soup (a*b+c) */
	void* d_primary_nodes; void* d_primary_tris; void* d_primary_tri_ids; /* over shader-decoded (fma) vertices */
	uint64_t shadow_node_count, primary_node_count;
	uint32_t shadow_max_depth, primary_max_depth;
	double build_seconds;
	/* material textures (src/scene.c:529-540): if any of the 3 * material_count textures is not constant, all of them live on the device as RGBA32F
	   mip chains and the G-buffer producer filters them (textured = 1); otherwise material_params above is all there is */
	int textured;
	void* d_texture_data;      /* float4 per texel, all chains back to back */
	void* d_texture_dims;      /* uint32[4] per texture: width, height, mip_count, 0; order: material-major, {base colour, specular, normal} */
	void* d_texture_offsets;   /* uint64 per texture: first texel of level 0 in d_texture_data */
	uint64_t texture_texel_count;
	uint32_t shadow_bvh_width;  /* children per node of d_shadow_nodes: 2 (64-byte node pairs); 4 only with VKR_BVH_WIDTH=4 in the environment, for the experimental kernel variant */
	/* the node pairs of d_shadow_nodes once more, 32 bytes each: child boxes as 16-bit coordinates on a grid over the scene, rounded outwards (what the trace
	   warps of the shading kernels fetch; the float pairs serve the probes and the tests). shadow_grid = minimum xyz, cells per world unit xyz */
	void* d_shadow_nodes_quantised;
	float shadow_grid[6];
	/* and once more as interleaved pairs (64 bytes, the two children's numbers side by side: the packed-FMA edition of the trace warps, vkr_trace.cuh) */
	void* d_shadow_nodes_interleaved;
} vkr_scene_t;

/* device may be NULL for vkr_load_scene / vkr_load_ltc_table / vkr_load_noise_table: the files are parsed and the host
   members filled, no device buffers or acceleration structures are created (loader tests without a GPU).
   file_path: a *.vks file; texture_path: directory with <material>_{BaseColor,Specular,Normal}.vkt.
   request_acceleration_structure mirrors load_scene's flag; without it shadow rays cannot be traced. */
int vkr_load_scene(vkr_scene_t* scene, const vkr_device_t* device, const char* file_path, const char* texture_path, int request_acceleration_structure);
void vkr_destroy_scene(vkr_scene_t* scene, const vkr_device_t* device);

/* ---- material textures (replaces load_2d_textures for *.vkt files, src/textures.c:111-169, and the texture units' format decode):
        all mip levels decoded to RGBA32F on the host. Formats: R16G16B16(A16)_SFLOAT, R32G32B32(A32)_SFLOAT, R8G8B8A8_UNORM / SRGB,
        BC1_RGB_UNORM / SRGB, BC5_UNORM (tools/texture_conversion/main.c:27-35). */
typedef struct vkr_texture_s {
	uint32_t width, height, mip_count, vk_format;
	float* h_texels;             /* level 0 first; level l is max(width >> l, 1) x max(height >> l, 1) RGBA32F */
	uint64_t texel_float_count;
	int is_constant;             /* every texel of every level has the same value */
} vkr_texture_t;
int vkr_load_texture(vkr_texture_t* texture, const char* file_path);
void vkr_destroy_texture(vkr_texture_t* texture);
/* Boundary B1: the mip levels of an image as the reference's load_2d_textures() holds them (raw bytes of vk_format per level, src/textures.c:111-169) */
int vkr_texture_from_levels(vkr_texture_t* texture, uint32_t width, uint32_t height, uint32_t mip_count, uint32_t vk_format, const void* const* level_data, const uint64_t* level_sizes);

/* ---- boundary B1 (SURVEY 8b): the reference's UNCHANGED loaders -- load_scene (src/scene.c:409-581), load_ltc_table (src/ltc_table.c:23-200),
        load_noise_table (src/noise_table.c:46-168) -- compiled against shim/ leave their staging buffers, images and the triangle soup of the
        acceleration structure build (the vkCmdBuildAccelerationStructuresKHR hook, src/scene.c:354-378) in host memory; these entry points take
        them over: device copies byte for byte, the software BVH built from the very vertices the reference hands to the driver.
        INTEGRATION.md (Route B) and tests/c_host/route_b.c show the calls. */
typedef struct vkr_scene_buffers_s {
	uint64_t triangle_count, material_count;
	float dequantization_factor[3], dequantization_summand[3];   /* mesh_t, src/scene.h:85-95 */
	const char* const* material_names;               /* materials_t::material_names; may be NULL if material_textures is given */
	const uint32_t* quantized_positions;             /* mesh.positions: uint32[2] per vertex (src/scene.h:56-62) */
	const uint16_t* normals_and_tex_coords;          /* mesh.normals_and_tex_coords: uint16[4] per vertex */
	const uint8_t* material_indices;                 /* mesh.material_indices: one per triangle */
	const float* acceleration_structure_vertices;    /* 9 floats per triangle as passed to the bottom-level build (src/scene.c:175-209); NULL: dequantised the same way here */
	const vkr_texture_t* material_textures;          /* 3 per material {base colour, specular, normal} (vkr_texture_from_levels), or NULL: read from texture_path */
	const char* texture_path;
} vkr_scene_buffers_t;
int vkr_scene_from_buffers(vkr_scene_t* scene, const vkr_device_t* device, const vkr_scene_buffers_t* buffers, int request_acceleration_structure);

/* ---- LTC table (replaces load_ltc_table / destroy_ltc_table, src/ltc_table.h:69-72, ltc_table.c:23-200) */
typedef struct vkr_ltc_constants_s { /* = ltc_constants_t, src/ltc_table.h:23-35 */
	float fresnel_index_factor, fresnel_index_summand;
	float roughness_factor, roughness_summand;
	float inclination_factor, inclination_summand;
	float padding[2];
} vkr_ltc_constants_t;

typedef struct vkr_ltc_table_s {
	uint32_t roughness_count, inclination_count, fresnel_count;
	void* d_table0;    /* RGBA16_UNORM [fresnel][inclination][roughness] = (inv00, -inv02, inv11, inv20) */
	void* d_table1;    /* RG16_UNORM   (inv22, albedo) */
	uint16_t* h_table0; uint16_t* h_table1; /* host copies (for inspection / tests) */
	vkr_ltc_constants_t constants;
} vkr_ltc_table_t;

int vkr_load_ltc_table(vkr_ltc_table_t* table, const vkr_device_t* device, const char* directory, uint32_t fresnel_count);
/* Boundary B1: the two texture arrays as load_ltc_table() uploads them (RGBA16_UNORM, RG16_UNORM; src/ltc_table.c:86-141) and its constants */
int vkr_ltc_table_from_images(vkr_ltc_table_t* table, const vkr_device_t* device, uint32_t roughness_count, uint32_t inclination_count, uint32_t fresnel_count,
	const uint16_t* table0_rgba16, const uint16_t* table1_rg16, const vkr_ltc_constants_t* constants);
void vkr_destroy_ltc_table(vkr_ltc_table_t* table, const vkr_device_t* device);

/* ---- fitting the LTC table (no counterpart in the reference, which reads fit<i>.dat from its data download): the specular BRDF of
        brdfs.glsl:74-87 (GGX, height-correlated Smith, Fresnel-Schlick with scalar F0) times cos(theta_i), fitted cell by cell with Heitz et al.
        2016's L3 error on the device, in float64 and a fixed summation order (csrc/vkr_ltc_fit.cuh, DESIGN.md §5): bit-identical from call to call
        and from device to device. Cell (layer f, row i, column j): F0 = f / (F - 1), theta = i / (N - 1) * pi / 2 (at most 89.5 degrees),
        alpha = (j / (N - 1))^2 (at least 1e-3) -- the cells vkr_load_ltc_table's texture coordinates address. Files are the interchange:
        vkr_write_ltc_fits, then vkr_load_ltc_table. */
#define VKR_LTC_FIT_MAX_RESOLUTION 4096      /* the loader's limit */
#define VKR_LTC_FIT_MAX_FRESNEL_COUNT 1024
#define VKR_LTC_FIT_MAX_QUADRATURE_SIZE 256
#define VKR_LTC_FIT_MAX_ITERATION_LIMIT 100000
typedef struct vkr_ltc_fit_desc_s {
	uint32_t resolution;        /* N: roughness and inclination count, 2 .. VKR_LTC_FIT_MAX_RESOLUTION (default 64) */
	uint32_t fresnel_count;     /* F: layers, one fit<i>.dat each, 2 .. VKR_LTC_FIT_MAX_FRESNEL_COUNT (default 51) */
	uint32_t quadrature_size;   /* n: each objective evaluation takes n x n stratified samples of the BRDF and of the LTC, 2 .. 256 (default 32) */
	uint32_t iteration_limit;   /* Nelder-Mead iterations per cell, 1 .. VKR_LTC_FIT_MAX_ITERATION_LIMIT (default 400) */
} vkr_ltc_fit_desc_t;
typedef struct vkr_ltc_fit_stats_s {
	uint64_t cell_count;
	uint64_t objective_evaluations;   /* summed over the cells */
	uint64_t iteration_limit_hits;    /* cells whose minimiser stopped at the iteration limit */
	double max_error, median_error, mean_error;   /* the final L3 error of the cells (integral of |lobe / albedo - LTC|^3 over the sphere) */
	float fit_ms;                     /* device time of the fit kernel (CUDA events) */
	double* cell_errors;              /* set by the caller: NULL, or F * N * N doubles that receive the final L3 error per cell, [F][N][N] */
} vkr_ltc_fit_stats_t;
void vkr_ltc_fit_default_desc(vkr_ltc_fit_desc_t* desc);
/* Synchronous. out_fits: HOST array [F][N][N][5] of {m00, m02, m11, m20, albedo}, texel row * N + column as in the file. stats may be NULL. */
int vkr_fit_ltc_table(const vkr_device_t* device, const vkr_ltc_fit_desc_t* desc, float* out_fits, vkr_ltc_fit_stats_t* stats);
/* Writes directory/fit<i>.dat, i < fresnel_count, as src/ltc_table.c:46-84 reads them: uint64 resolution, then N * N records of 5 float32.
   The directory must exist. */
int vkr_write_ltc_fits(const char* directory, uint32_t resolution, uint32_t fresnel_count, const float* fits);

/* ---- noise table (replaces load_noise_table / set_noise_constants, src/noise_table.h:81-89, noise_table.c:46-168) */
typedef struct vkr_noise_table_s {
	uint32_t width, height, layers;
	void* d_noise;        /* RGBA16_UNORM [layer][y][x] */
	uint16_t* h_noise;
	uint32_t random_seed;
} vkr_noise_table_t;

int vkr_load_noise_table(vkr_noise_table_t* noise, const vkr_device_t* device, uint32_t width, uint32_t height, uint32_t layers, vkr_noise_type_t noise_type);
/* Boundary B1: the texture array as load_noise_table() uploads it (RGBA16_UNORM, layer-major; src/noise_table.c:105-160) and noise_table_t::random_seed */
int vkr_noise_table_from_image(vkr_noise_table_t* noise, const vkr_device_t* device, uint32_t width, uint32_t height, uint32_t layers, const uint16_t* texels_rgba16, uint32_t random_seed);
void vkr_destroy_noise_table(vkr_noise_table_t* noise, const vkr_device_t* device);
void vkr_set_noise_constants(uint32_t resolution_mask[2], uint32_t* texture_index_mask, uint32_t random_numbers[4], vkr_noise_table_t* noise, int animate_noise);

/* ---- generating the file-backed noise tables (no counterpart in the reference, which reads data/noise/<name>.blob from its data download): tables of
        the kind vkr_noise_type_blue and vkr_noise_type_ahmed name, made on the device in integer arithmetic (csrc/vkr_noise_gen.cuh, DESIGN.md §5),
        bit-identical from call to call and from device to device. They are this project's tables, not the paper's files. Files are the
        interchange: vkr_write_noise_table, then vkr_load_noise_table.
        ahmed: W = H = 2^m <= 256; each (layer, RG / BA pair) is an Owen-scrambled 2D Sobol sequence in a hierarchical pixel order, so every aligned
               2^j x 2^j block holds a (0, 2j, 2)-net.
        blue:  W * H <= VKR_NOISE_GEN_MAX_BLUE_PIXELS; each channel of each layer is an independent void-and-cluster dither array. */
#define VKR_NOISE_GEN_MAX_AHMED_SIZE 256
#define VKR_NOISE_GEN_MAX_BLUE_PIXELS 16384
typedef struct vkr_noise_gen_desc_s {
	vkr_noise_type_t type;          /* vkr_noise_type_blue or vkr_noise_type_ahmed */
	uint32_t width, height, layers; /* powers of two the loader accepts (at most 9999) */
	uint32_t seed;                  /* different seeds give independent tables */
} vkr_noise_gen_desc_t;
typedef struct vkr_noise_gen_stats_s {
	float kernel_ms;                /* device time of the generating kernel (CUDA events) */
	uint32_t relaxation_limit_hits; /* blue: dither arrays whose initial pattern stopped relaxing at the iteration limit (W * H iterations) */
} vkr_noise_gen_stats_t;
/* the reference's default resolution of a type (get_default_noise_resolution, src/noise_table.c:22-40): blue 64 x 64 x 64, otherwise 256 x 256 x 64 */
void vkr_noise_gen_default_desc(vkr_noise_type_t type, vkr_noise_gen_desc_t* desc);
/* Synchronous. texels_rgba16: HOST array of width * height * layers * 4 uint16, [layer][y][x][4] as the file holds it. stats may be NULL.
   Refuses, before any device work: the white type, sizes the loader refuses, non-square or larger Ahmed tables, larger dither arrays, no device. */
int vkr_generate_noise_table(const vkr_device_t* device, const vkr_noise_gen_desc_t* desc, uint16_t* texels_rgba16, vkr_noise_gen_stats_t* stats);
/* Writes root/data/noise/blue_noise_rgba_WWxHH_LL.blob or ahmed_2d_rgba_WWxHH_LL.blob, the path vkr_load_noise_table opens relative to the working
   directory, creating root, root/data and root/data/noise as needed (root's parent must exist). */
int vkr_write_noise_table(const char* root, vkr_noise_type_t type, uint32_t width, uint32_t height, uint32_t layers, const uint16_t* texels_rgba16);

/* ---- camera and lights (host-only; same binary layout as src/camera.h:24-44, src/polygonal_light.h:100-129) */
typedef struct vkr_first_person_camera_s {
	float position_world_space[3];
	float rotation_z, rotation_x, vertical_fov;
	float near_plane, far_plane;
	float speed;
	int rotate_camera;
	float rotation_x_0, rotation_z_0;
} vkr_first_person_camera_t;

typedef struct vkr_polygonal_light_s {
	float rotation_angles[3]; float scaling_x;
	float translation[3]; float scaling_y;
	float radiant_flux[3]; float inv_scaling_x;
	float surface_radiance[3]; float inv_scaling_y;
	float plane[4];
	uint32_t vertex_count; uint32_t texturing_technique; uint32_t texture_index; uint32_t padding_0;
	float rotation[3][4];
	float area, rcp_area; float padding_1[2];
	char* texture_file_path;
	float* vertices_plane_space;
	float* vertices_world_space;
	float* fan_areas;
} vkr_polygonal_light_t;

typedef struct vkr_scene_specification_s { /* camera + lights of scene_specification_t, src/main.h:29-42 */
	vkr_first_person_camera_t camera;
	uint32_t polygonal_light_count;
	vkr_polygonal_light_t* polygonal_lights;
} vkr_scene_specification_t;

void vkr_update_polygonal_light(vkr_polygonal_light_t* light);                       /* update_polygonal_light, polygonal_light.c:46-104 */
void vkr_set_polygonal_light_vertex_count(vkr_polygonal_light_t* light, uint32_t n); /* polygonal_light.c:24-43 */
void vkr_destroy_polygonal_light(vkr_polygonal_light_t* light);
void vkr_get_world_to_projection_space(float world_to_projection_space[4][4], const vkr_first_person_camera_t* camera, float aspect_ratio); /* camera.c:74-83 */
/* quick_load / quick_save, src/main.c:49-130 (same *.save files) */
int vkr_quick_load(vkr_scene_specification_t* spec, const char* quick_save_path);
int vkr_quick_save(const vkr_scene_specification_t* spec, const char* quick_save_path);
void vkr_destroy_scene_specification(vkr_scene_specification_t* spec);

/* ---- light textures (replaces create_and_assign_light_textures / destroy_light_textures, src/main.c:364-418; sampled by
        get_polygon_radiance(), src/shaders/shading_pass.frag.glsl:151-185). The unique texture_file_path entries of the lights, in the
        order of their first use, each decoded to an RGBA32F mip chain (level 0 is what the shader reads); lights without a path or
        with a path that cannot be opened share a white texture (the reference's data/white.vkt), with the reference's message.
        Sets polygonal_lights[i].texture_index. light_textures = NULL: indices only (as the reference does at src/main.c:2167);
        device = NULL: host copies only. */
typedef struct vkr_light_textures_s {
	uint32_t texture_count;
	vkr_texture_t* textures;
	void* d_texels;      /* float4 texels of all textures, chain after chain */
	void* d_dims;        /* uint4 {width, height, mip_count, 0} per texture */
	void* d_offsets;     /* uint64 index of the first texel of each texture in d_texels */
	uint64_t texel_count;
} vkr_light_textures_t;
int vkr_create_and_assign_light_textures(vkr_light_textures_t* light_textures, const vkr_device_t* device, vkr_scene_specification_t* spec);
void vkr_destroy_light_textures(vkr_light_textures_t* light_textures, const vkr_device_t* device);

/* ---- render settings (the subset of render_settings_t, src/main.h:128-159, the shading pass consumes) */
typedef struct vkr_render_settings_s {
	float exposure_factor, roughness_factor;
	uint32_t sample_count;
	vkr_sampling_strategies_t sampling_strategies;
	vkr_mis_heuristic_t mis_heuristic;
	float mis_visibility_estimate;
	vkr_sample_polygon_technique_t polygon_sampling_technique;
	float error_min_exponent;
	int animate_noise;
	int trace_shadow_rays;
	int show_polygonal_lights;
} vkr_render_settings_t;

void vkr_specify_default_render_settings(vkr_render_settings_t* settings); /* main.c:232-249 */

/* Size of the constant block for the given lights: 256 + light_count * (160 + 16*V + 16*V + 16*(V-2)),
   V = max vertex count over the lights (main.c:334). */
size_t vkr_get_constants_size(const vkr_scene_specification_t* spec);
/* Writes the per-frame constants exactly as write_constants() does (src/main.c:2114-2188). Returns bytes written. */
size_t vkr_write_constants(void* data, const vkr_scene_specification_t* spec, const vkr_render_settings_t* settings,
	const vkr_scene_t* scene, const vkr_ltc_table_t* ltc, vkr_noise_table_t* noise, uint32_t width, uint32_t height);
/* HDR screenshots (src/main.c:1702-1750, :2132): write_constants() copies app->screenshot.frame_bits into the block;
   0 = normal frame, 1 / 2 = the frame carries the low / high bytes of the half-precision colours */
void vkr_set_frame_bits(void* constants, uint32_t frame_bits);

/* ---- G-buffer producer (stands in for subpass 0 + get_shading_data(), src/main.c:1422-1427,
        src/shaders/shading_pass.frag.glsl:721-822). Layout: 4 planes of width*height float4:
        {position.xyz, roughness} {normal.xyz, 1 if surface else 0} {diffuse_albedo.rgb, 0} {fresnel_0.rgb, 0} */
size_t vkr_gbuffer_size(uint32_t width, uint32_t height);
/* d_visibility (uint32 per pixel, 0xFFFFFFFF = background) is written by a primary-ray cast; constants = first 256 bytes of the block (host) */
int vkr_run_visibility_pass(const vkr_device_t* device, const vkr_scene_t* scene, const void* constants, uint32_t width, uint32_t height, void* d_visibility);
int vkr_run_gbuffer_pass(const vkr_device_t* device, const vkr_scene_t* scene, const void* constants, uint32_t width, uint32_t height, const void* d_visibility, void* d_gbuffer);

/* ---- render targets (replaces create_render_targets / destroy_render_targets, src/main.c:253-315, and the swapchain image the
        shading pass writes): device images of one resolution, owned by the library so that a host application needs no CUDA
        allocator of its own. The reference's depth buffer has no counterpart (visibility comes from primary rays). */
typedef struct vkr_render_targets_s {
	uint32_t width, height;
	void* d_visibility;   /* uint32 per pixel, 0xFFFFFFFF = background (the clear value, src/main.c:1409) */
	void* d_gbuffer;      /* vkr_gbuffer_size(width, height) bytes */
	void* d_frame;        /* width * height float4: what the shading pass writes */
} vkr_render_targets_t;
int vkr_create_render_targets(vkr_render_targets_t* targets, const vkr_device_t* device, uint32_t width, uint32_t height);
void vkr_destroy_render_targets(vkr_render_targets_t* targets, const vkr_device_t* device);
/* Copies the frame (width * height float4) / the G-buffer to HOST memory and waits for it */
int vkr_download_frame(const vkr_render_targets_t* targets, const vkr_device_t* device, float* out_rgba32f);
int vkr_download_gbuffer(const vkr_render_targets_t* targets, const vkr_device_t* device, uint32_t* out_visibility, float* out_gbuffer);
/* Copies a G-buffer from HOST memory into the targets (e.g. one made elsewhere) */
int vkr_upload_gbuffer(vkr_render_targets_t* targets, const vkr_device_t* device, const float* gbuffer);

/* ---- the shading pass (replaces create_shading_pass src/main.c:598-940, the subpass-1 draw
        src/main.c:1429-1434 and the per-frame part of render_frame src/main.c:2197-2270) */
typedef struct vkr_shading_pass_desc_s {
	uint32_t width, height;
	/* what the reference bakes into the shader as -D defines (src/main.c:752-792) */
	uint32_t polygonal_light_count;
	uint32_t min_polygonal_light_vertex_count, max_polygonal_light_vertex_count;
	uint32_t sample_count;
	vkr_sampling_strategies_t sampling_strategies;
	vkr_mis_heuristic_t mis_heuristic;
	vkr_sample_polygon_technique_t polygon_sampling_technique;
	int trace_shadow_rays;
	int show_polygonal_lights;
	/* multi-GPU split: this pass instance shades the 16x8 screen tiles (tx, ty) with (tx + ty / VKR_TILE_BAND_ROWS) % stripe_count ==
	   stripe_index (SURVEY 8e asks for tile rows per GPU; the rows are cut further into tiles and dealt out column-wise because
	   135 tile rows of uneven cost do not balance over 8 GPUs; the columns of a share move on by one every 8 tile rows so that no
	   share sits on one set of screen columns -- at 1920x1080 every GPU of 8 visits each column phase twice. Every GPU gets the
	   same number of tiles from all over the screen, and its part of a G-buffer plane is one strided 2D copy per band);
	   stripe_count = 0 or 1 means the whole frame */
	uint32_t stripe_index, stripe_count;
	/* resources */
	const vkr_scene_t* scene;
	const vkr_ltc_table_t* ltc_table;
	const vkr_noise_table_t* noise_table;
	/* output stage (shading_pass.frag.glsl:866-892): 0 = linear RGB, what the shader writes when the swapchain converts to
	   sRGB itself (OUTPUT_LINEAR_RGB=1, src/main.c:790); 1 = the shader converts to sRGB (OUTPUT_LINEAR_RGB=0). The
	   half-bit split for HDR screenshots follows g_frame_bits in the constant block (vkr_set_frame_bits). Output stays
	   float4: the values the render target receives before its UNORM quantisation. */
	int output_srgb;
	/* ERROR_DISPLAY_DIFFUSE / ERROR_DISPLAY_SPECULAR / ERROR_INDEX (src/main.c:735-750, 788-790); the scale comes from error_min_exponent
	   in the render settings via g_error_factor in the constant block */
	vkr_error_display_t error_display;
	/* textures of the polygonal lights (g_light_textures); may be NULL as long as no light of a frame's constant block is textured.
	   Every sampling technique works with textured lights; the error display does not (it shows no radiance). */
	const vkr_light_textures_t* light_textures;
} vkr_shading_pass_desc_t;

typedef struct vkr_shading_pass_s {
	vkr_shading_pass_desc_t desc;
	size_t constants_size;
	void* d_constants;         /* device staging of the constant block */
	void* h_constants_pinned;
	void* d_gbuffer_staging;   /* used by vkr_shading_pass_run_host only */
	void* d_out_staging;
	uint64_t kernel_launches;  /* number of kernels this pass has launched so far */
	float last_kernel_ms;      /* device time of the most recent shading kernel (CUDA events), if timing is enabled */
	void* event_begin; void* event_end;
	int timing_enabled;
	void* event_constants;     /* recorded after the upload of the constant block: the staging buffer is not rewritten before */
	/* The tiles this instance shades, in launch order. After every frame the pass reads back what each tile cost (nanoseconds) and
	   launches the next frame dearest tile first, so that the last wave of CTAs consists of cheap tiles (frames of an animation
	   resemble their predecessors; the order never changes a pixel). reorder_tiles = 0 keeps the order fixed (row-major). */
	uint32_t tile_count;
	void* d_tile_list; void* h_tile_list;
	void* d_tile_cost; void* h_tile_cost;
	void* event_costs; int costs_pending;
	int reorder_tiles;
} vkr_shading_pass_t;

int vkr_create_shading_pass(vkr_shading_pass_t* pass, const vkr_device_t* device, const vkr_shading_pass_desc_t* desc);
void vkr_destroy_shading_pass(vkr_shading_pass_t* pass, const vkr_device_t* device);
/* Asynchronous on device->stream. constants: HOST pointer to the block written by vkr_write_constants() (or by the
   reference's write_constants()). d_gbuffer / d_out_rgba32f: DEVICE pointers (out = width*height float4, pixels outside
   the tiles of this instance untouched). */
int vkr_shading_pass_run(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out_rgba32f);
/* End-to-end variant with HOST buffers: uploads the G-buffer tiles of this instance, shades, downloads them, waits. */
int vkr_shading_pass_run_host(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const float* gbuffer, float* out_rgba32f);
int vkr_shading_pass_wait(vkr_shading_pass_t* pass, const vkr_device_t* device);

/* ---- one frame on several GPUs (replaces nothing in the reference, which drives one GPU; SURVEY 8e). Every GPU of the box runs its
        own pass instance (stripe_index = rank, stripe_count = world) and owns a vkr_frame_exchange_t. The shading kernel stores each
        finished pixel into the frame of EVERY GPU -- its own and, through peer mappings over NVLink, the others' -- so when the
        kernels are done each GPU holds the whole frame; no gather pass, no collective library. Two one-block kernels per frame
        make the barrier: signal (release, system scope) increments this GPU's arrival counter on every peer, wait (acquire) spins
        until all peers of this frame have arrived. Frames alternate between two buffers, so a GPU may start frame f + 1 while a
        slower one still reads frame f.
        One process per GPU: create, vkr_frame_exchange_get_handle, exchange the 64-byte handles by whatever means the host has
        (MPI, a socket, torch.distributed), vkr_frame_exchange_connect. One process for all GPUs: vkr_frame_exchange_connect_local. */
typedef struct vkr_frame_exchange_s {
	uint32_t width, height, rank, world;
	void* d_block;                          /* one cudaMalloc: two frames (width * height float4 each), then 2 * VKR_MAX_GPUS arrival counters */
	void* d_peer_blocks[VKR_MAX_GPUS];      /* [rank] = d_block; the others: mappings of the peers' blocks */
	int peer_is_ipc[VKR_MAX_GPUS];          /* mapping came from cudaIpcOpenMemHandle (to be closed) */
	uint64_t frames_exchanged;              /* frames completed so far; the frame in flight lives in buffer frames_exchanged & 1 */
	int* h_status;                          /* pinned, device-visible: set by the wait kernel when a peer did not arrive in time */
	uint64_t timeout_ns;                    /* how long the wait kernel waits for the peers (default 20 s) */
} vkr_frame_exchange_t;
int vkr_create_frame_exchange(vkr_frame_exchange_t* exchange, const vkr_device_t* device, uint32_t width, uint32_t height, uint32_t rank, uint32_t world);
void vkr_destroy_frame_exchange(vkr_frame_exchange_t* exchange, const vkr_device_t* device);
/* the cudaIpcMemHandle_t of this GPU's block, to be sent to the other processes */
int vkr_frame_exchange_get_handle(const vkr_frame_exchange_t* exchange, const vkr_device_t* device, unsigned char out_handle[64]);
/* handles: world * 64 bytes in rank order (the entry of this rank is ignored) */
int vkr_frame_exchange_connect(vkr_frame_exchange_t* exchange, const vkr_device_t* device, const unsigned char* handles);
/* all GPUs driven by this process: d_blocks[r] = the d_block of rank r's exchange (peer access is enabled here) */
int vkr_frame_exchange_connect_local(vkr_frame_exchange_t* exchange, const vkr_device_t* device, void* const* d_blocks);
/* device pointer to the most recently completed frame (width * height float4), valid until the frame after the next is started */
void* vkr_frame_exchange_frame(const vkr_frame_exchange_t* exchange);
/* Shades this GPU's tiles of one frame into every GPU's frame, signals, waits for the peers: asynchronous on device->stream; once the
   stream has passed this call vkr_frame_exchange_frame() holds the whole frame. All GPUs must call it once per frame. */
int vkr_shading_pass_run_exchange(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, vkr_frame_exchange_t* exchange);
/* Host-buffer variant: uploads this GPU's tile columns of the G-buffer (one strided copy per plane and band of tile rows), shades and exchanges as above, and
   if out_rgba32f is not NULL downloads the WHOLE frame; waits. Returns non-zero if a peer failed to arrive. */
int vkr_shading_pass_run_host_exchange(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const float* gbuffer,
	vkr_frame_exchange_t* exchange, float* out_rgba32f);
/* copies the most recently completed frame (the whole frame) to HOST memory and waits */
int vkr_frame_exchange_download(vkr_frame_exchange_t* exchange, const vkr_device_t* device, float* out_rgba32f);
/* waits for the stream and reports whether the exchange has failed (a peer did not arrive in time) */
int vkr_frame_exchange_wait(vkr_frame_exchange_t* exchange, const vkr_device_t* device);

/* Measurement aid (no counterpart in the reference, which reads such numbers from vendor profilers): shades the frame with the counters
   edition of the kernel -- same frame, bit for bit -- and returns what the trace warps did. Synchronous; quad lights, projected solid
   angle sampling, untextured lights only. Sums over the whole launch; "lane" counters count per ray, "warp" counters per warp. */
typedef enum vkr_trace_counter_e {
	vkr_trace_counter_rays = 0,             /* shadow rays traced (entries whose visibility was not known beforehand) */
	vkr_trace_counter_occluded = 1,         /* of these, rays that hit something */
	vkr_trace_counter_cache_hits = 2,       /* of these, rays ended by the occluder cache before any traversal */
	vkr_trace_counter_node_visits = 3,      /* BVH nodes fetched, summed over rays */
	vkr_trace_counter_leaf_visits = 4,      /* leaves whose triangles were tested, summed over rays */
	vkr_trace_counter_triangle_tests = 5,   /* ray/triangle predicates evaluated */
	vkr_trace_counter_warp_rounds = 6,      /* rounds of the trace warps' outer loop (warp) */
	vkr_trace_counter_warp_node_steps = 7,  /* iterations of the node loop (warp): node_visits / this = lanes busy per step */
	vkr_trace_counter_known_occluded = 8,   /* ring entries that needed no ray (n.w <= 0; optimal MIS only) */
	vkr_trace_counter_idle_polls = 9,       /* times a trace warp found nothing to do and slept (warp) */
	vkr_trace_counter_entries = 10,         /* ring entries submitted by the shading warps */
	vkr_trace_counter_resolve_polls = 11,   /* times a shading warp slept waiting for shadow ray results (warp) */
	vkr_trace_counter_candidates = 12,      /* candidate samples with a contribution (before the n.w > 0 test) */
	VKR_TRACE_COUNTER_COUNT = 16
} vkr_trace_counter_t;
int vkr_shading_pass_run_with_counters(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out_rgba32f,
	uint64_t out_counters[VKR_TRACE_COUNTER_COUNT]);

/* ---- after the pass: screenshots and frame times (SURVEY 8 f3; replaces take_screenshot / implement_screenshot,
        src/main.c:1550-1770, the stb_image_write calls in them and src/frame_timer.c) */
/* What an 8-bit UNORM render target stores for a float frame: round(clamp(x, 0, 1) * 255) per channel, alpha dropped */
void vkr_quantize_unorm8(const float* rgba32f, uint32_t width, uint32_t height, uint8_t* out_rgb8);
/* combine_ldr_screenshots_into_hdr, src/main.c:1696-1707: low / high bytes of half-precision values -> float */
void vkr_combine_ldr_screenshots_into_hdr(const uint8_t* low_bytes, const uint8_t* high_bytes, size_t entry_count, float* out_hdr);
/* stbi_write_png / stbi_write_hdr as called at src/main.c:1734, 1755: tightly packed 8-bit RGB / float RGB */
int vkr_write_png(const char* file_path, uint32_t width, uint32_t height, const uint8_t* rgb8);
int vkr_write_hdr(const char* file_path, uint32_t width, uint32_t height, const float* rgb32f);
/* Shades the frame and stores it: *.png (the shader converts to sRGB, 8-bit quantisation) or *.hdr (two frames with the low and
   high half-float bytes, g_frame_bits = 1 / 2, combined on the host like the reference does). Exactly one path must be given.
   constants: HOST pointer; d_gbuffer: DEVICE pointer. Synchronous. */
int vkr_take_screenshot(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer,
	const char* path_png, const char* path_hdr);
/* record_frame_time / get_frame_time, src/frame_timer.c:28-75: median of the differences of the last 100 recorded times (seconds) */
void vkr_record_frame_time(double time_in_seconds);
float vkr_get_frame_time(void);
void vkr_reset_frame_times(void);

/* ---- averaging frames and measuring their error (no counterpart in the reference, which shows one frame at a time). What is accumulated is the
        frame as the shading pass stores it: linear radiance times the exposure factor, RGB; alpha is ignored. A pixel whose radiance was NaN has been
        painted pink by the pass (as the reference does), so it counts as that colour. Accumulate frames of a pass with output_srgb = 0 and
        g_frame_bits = 0 (vkr_set_frame_bits); sRGB or half-bit frames are not radiance. Frames of independent noise come from animate_noise = 1 in
        the render settings: each vkr_write_constants() call then draws new random numbers.
        All arithmetic is float64 and every sum has a fixed order (csrc/vkr_accumulate.cuh), so results are bit-identical from call to call and from
        device to device. Asynchronous on device->stream unless marked synchronous; those wait for device->stream only. */
typedef struct vkr_accumulator_s {
	uint32_t width, height;
	uint64_t frame_count;   /* frames added since create / reset */
	void* d_state;          /* 6 planes of width*height double: mean rgb, m2 rgb (Welford) */
	void* d_partials; void* h_partials;   /* reduction scratch, pinned host copy */
} vkr_accumulator_t;
/* 48 bytes of state per pixel (99.5 MB at 1920x1080) */
int vkr_create_accumulator(vkr_accumulator_t* accumulator, const vkr_device_t* device, uint32_t width, uint32_t height);
void vkr_destroy_accumulator(vkr_accumulator_t* accumulator, const vkr_device_t* device);
/* frame_count = 0; the next frame replaces the state */
int vkr_accumulator_reset(vkr_accumulator_t* accumulator, const vkr_device_t* device);
/* d_frame_rgba32f: DEVICE pointer, width*height float4 (16-byte aligned), e.g. vkr_render_targets_t::d_frame after vkr_shading_pass_run. Per pixel and
   channel, frame n = frame_count + 1: d = x - mean; mean += d / n; m2 += d * (x - mean) (the first frame is stored as it is) */
int vkr_accumulate_frame(vkr_accumulator_t* accumulator, const vkr_device_t* device, const void* d_frame_rgba32f);
/* DEVICE pointers, width*height float4 each, either may be NULL: the mean rounded to float (alpha 1) and the per-frame sample variance
   m2 / (frame_count - 1) rounded to float (alpha 0). Refuses frame_count == 0, and a variance with frame_count < 2. */
int vkr_accumulator_resolve(const vkr_accumulator_t* accumulator, const vkr_device_t* device, void* d_mean_rgba32f, void* d_variance_rgba32f);
/* synchronous: per channel, the mean over all pixels of the per-frame sample variance -- the noise level of a setting, no reference needed. frame_count >= 2. */
int vkr_accumulator_mean_variance(const vkr_accumulator_t* accumulator, const vkr_device_t* device, double out_mean_variance[3]);
/* A frame x against a reference r, over the pixels whose six RGB inputs are finite (N = pixel_count), in float64 from the exactly converted floats:
   mse[c] = sum (x-r)^2 / N; rel_mse[c] = sum (x-r)^2 / (r^2 + 0.01) / N; mae[c] = sum |x-r| / N; max_abs_error over all channels. The means are
   NaN if N = 0. nonfinite_pixels: pixels left out. */
typedef struct vkr_frame_error_s {
	double mse[3], rel_mse[3], mae[3], max_abs_error;
	uint64_t pixel_count, nonfinite_pixels;
} vkr_frame_error_t;
/* synchronous; both frames are DEVICE pointers to width*height float4 */
int vkr_compare_frames(const vkr_device_t* device, uint32_t width, uint32_t height, const void* d_frame_rgba32f, const void* d_reference_rgba32f, vkr_frame_error_t* out);

/* ---- shadow-ray probe (tests / KATs): rays = {ox,oy,oz,dx,dy,dz,tmin,tmax} per ray on the HOST, out = 1 byte per ray */
int vkr_trace_shadow_rays(const vkr_device_t* device, const vkr_scene_t* scene, uint32_t ray_count, const float* rays, uint8_t* out_occluded);
/* ---- sampling probe (tests / KATs): clip + prepare + sample in the polygon's local space on the device */
int vkr_sample_polygon_batch(const vkr_device_t* device, uint32_t vertex_count, const float* vertices_xyz, int biased,
	uint32_t n, const float* random_numbers, float* out_dirs, float* out_info);

/* ---- arithmetic probe: the kernels' reciprocal square root (one range check in front of the square root's and the reciprocal's fast paths, csrc/vkr_device_math.cuh)
        against its definition 1.0f / sqrtf(x) for all 2^32 floats on the device; mismatches must come back 0 */
int vkr_probe_rsqrt_exhaustive(const vkr_device_t* device, uint64_t* out_mismatches, uint32_t* out_first_mismatch_bits);

/* ---- BVH builder probe (structural tests on the host; arrays are malloc'ed, release with vkr_bvh_free_probe).
        nodes: 16 floats per node pair, tris: 12 floats per slot, tri_ids: original index per slot (layout: csrc/vkr_trace.cuh) */
/* builder: 0 = binned SAH (the default of vkr_load_scene), 1 = linear BVH (the host reference of the GPU builder; VKR_BVH_BUILDER=lbvh) */
int vkr_bvh_build_probe_with(int builder, const float* vertices, uint64_t triangle_count, float** out_nodes, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth);
/* the linear BVH built on the GPU (vkr_lbvh_gpu.cu; VKR_BVH_BUILDER=lbvh_gpu), copied to the host: must equal builder 1 array for array */
int vkr_bvh_build_probe_device(const vkr_device_t* device, const float* vertices, uint64_t triangle_count, float** out_nodes, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth);
/* builder 0's tree collapsed into 4-wide nodes (32 floats each; layout: csrc/vkr_bvh.h) -- groundwork for a 4-wide trace loop, not used by the kernels yet */
int vkr_bvh4_build_probe(const float* vertices, uint64_t triangle_count, float** out_nodes4, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth,
	uint64_t* out_bvh2_node_count, uint32_t* out_bvh2_max_depth);
int vkr_bvh_build_probe(const float* vertices, uint64_t triangle_count, float** out_nodes, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth);
void vkr_bvh_free_probe(float* nodes, float* tris, uint32_t* tri_ids);

uint32_t vkr_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif
