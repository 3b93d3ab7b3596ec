"""ctypes binding of libvkr_b200.so (include/vkr_b200.h).

This is the host-side mirror used by tests/, bench.py and smoke(); it adds nothing to the C-ABI.
The product path is the CUDA library: loading fails loudly when it has not been built, and every
compute entry point needs a visible CUDA device (vkr_create_device reports the absence).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvkr_b200.so")

# Every symbol include/vkr_b200.h declares
EXPORTED_SYMBOLS = [
	"vkr_abi_version", "vkr_create_device", "vkr_destroy_device", "vkr_device_wait_idle",
	"vkr_load_scene", "vkr_destroy_scene", "vkr_load_ltc_table", "vkr_destroy_ltc_table",
	"vkr_load_noise_table", "vkr_destroy_noise_table", "vkr_set_noise_constants",
	"vkr_update_polygonal_light", "vkr_set_polygonal_light_vertex_count", "vkr_destroy_polygonal_light",
	"vkr_get_world_to_projection_space", "vkr_quick_load", "vkr_quick_save", "vkr_destroy_scene_specification",
	"vkr_specify_default_render_settings", "vkr_get_constants_size", "vkr_write_constants", "vkr_set_frame_bits",
	"vkr_gbuffer_size", "vkr_run_visibility_pass", "vkr_run_gbuffer_pass",
	"vkr_create_shading_pass", "vkr_destroy_shading_pass", "vkr_shading_pass_run", "vkr_shading_pass_run_host", "vkr_shading_pass_wait", "vkr_shading_pass_run_with_counters", "vkr_shading_pass_run_tiles",
	"vkr_create_frame_exchange", "vkr_destroy_frame_exchange", "vkr_frame_exchange_get_handle", "vkr_frame_exchange_connect", "vkr_frame_exchange_connect_local",
	"vkr_frame_exchange_frame", "vkr_shading_pass_run_exchange", "vkr_shading_pass_run_host_exchange", "vkr_frame_exchange_wait", "vkr_frame_exchange_download",
	"vkr_trace_shadow_rays", "vkr_sample_polygon_batch", "vkr_sample_related_work_batch", "vkr_probe_rsqrt_exhaustive", "vkr_bvh_build_probe", "vkr_bvh_build_probe_with", "vkr_bvh_build_probe_device", "vkr_bvh4_build_probe", "vkr_bvh_free_probe",
	"vkr_quantize_unorm8", "vkr_combine_ldr_screenshots_into_hdr", "vkr_write_png", "vkr_write_hdr", "vkr_take_screenshot",
	"vkr_record_frame_time", "vkr_get_frame_time", "vkr_reset_frame_times",
	"vkr_load_texture", "vkr_destroy_texture", "vkr_texture_from_levels", "vkr_scene_from_buffers", "vkr_ltc_table_from_images", "vkr_noise_table_from_image", "vkr_create_and_assign_light_textures", "vkr_destroy_light_textures",
	"vkr_create_render_targets", "vkr_destroy_render_targets", "vkr_download_frame", "vkr_download_gbuffer", "vkr_upload_gbuffer",
	"vkr_create_accumulator", "vkr_destroy_accumulator", "vkr_accumulator_reset", "vkr_accumulate_frame", "vkr_accumulator_resolve", "vkr_accumulator_mean_variance", "vkr_compare_frames",
	"vkr_create_adaptive_accumulator", "vkr_destroy_adaptive_accumulator", "vkr_adaptive_accumulator_reset", "vkr_adaptive_accumulate_frame", "vkr_adaptive_update_tiles",
	"vkr_adaptive_tile_frames", "vkr_adaptive_resolve", "vkr_adaptive_estimated_rel_mse",
	"vkr_ltc_fit_default_desc", "vkr_fit_ltc_table", "vkr_write_ltc_fits",
	"vkr_noise_gen_default_desc", "vkr_generate_noise_table", "vkr_write_noise_table",
	"vkr_take_screenshot_formats", "vkr_quantize_unorm8_device", "vkr_encode_jpg", "vkr_write_jpg",
	"vkr_create_rasterizer", "vkr_destroy_rasterizer", "vkr_rasterize_visibility",
]

# enums (values = the reference's)
ERROR_DISPLAY_NONE, ERROR_DISPLAY_DIFFUSE_BACKWARD, ERROR_DISPLAY_DIFFUSE_BACKWARD_SCALED, ERROR_DISPLAY_DIFFUSE_FORWARD, \
	ERROR_DISPLAY_SPECULAR_BACKWARD, ERROR_DISPLAY_SPECULAR_BACKWARD_SCALED, ERROR_DISPLAY_SPECULAR_FORWARD = range(7)
STRATEGY_DIFFUSE_ONLY, STRATEGY_DIFFUSE_GGX_MIS, STRATEGY_DIFFUSE_SPECULAR_SEPARATELY, STRATEGY_DIFFUSE_SPECULAR_MIS, STRATEGY_DIFFUSE_SPECULAR_RANDOM = range(5)
MIS_BALANCE, MIS_POWER, MIS_WEIGHTED, MIS_OPTIMAL_CLAMPED, MIS_OPTIMAL = range(5)
TECHNIQUE_PSA, TECHNIQUE_PSA_BIASED = 11, 12
# the related-work techniques (sample_polygon_technique_t, src/polygonal_light.h:30-66), SURVEY 8 f4
(TECHNIQUE_BASELINE, TECHNIQUE_AREA_TURK, TECHNIQUE_RECTANGLE_SOLID_ANGLE_URENA, TECHNIQUE_SOLID_ANGLE_ARVO, TECHNIQUE_SOLID_ANGLE, TECHNIQUE_CLIPPED_SOLID_ANGLE,
	TECHNIQUE_BILINEAR_COSINE_WARP_HART, TECHNIQUE_BILINEAR_COSINE_WARP_CLIPPING_HART, TECHNIQUE_BIQUADRATIC_COSINE_WARP_HART,
	TECHNIQUE_BIQUADRATIC_COSINE_WARP_CLIPPING_HART, TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO) = range(11)
NOISE_WHITE, NOISE_BLUE, NOISE_AHMED = 0, 1, 2


class Device(C.Structure):
	_fields_ = [("cuda_device", C.c_int), ("sm_count", C.c_int), ("ray_tracing_supported", C.c_int), ("stream", C.c_void_p),
		("owns_stream", C.c_int), ("name", C.c_char * 64)]


class Scene(C.Structure):
	_fields_ = [("triangle_count", C.c_uint64), ("material_count", C.c_uint64),
		("dequantization_factor", C.c_float * 3), ("dequantization_summand", C.c_float * 3),
		("material_names", C.POINTER(C.c_char_p)), ("material_params", C.POINTER(C.c_float)),
		("d_quantized_positions", C.c_void_p), ("d_normals_and_tex_coords", C.c_void_p), ("d_material_indices", C.c_void_p), ("d_material_params", C.c_void_p),
		("d_shadow_nodes", C.c_void_p), ("d_shadow_tris", C.c_void_p),
		("d_primary_nodes", C.c_void_p), ("d_primary_tris", C.c_void_p), ("d_primary_tri_ids", C.c_void_p),
		("shadow_node_count", C.c_uint64), ("primary_node_count", C.c_uint64),
		("shadow_max_depth", C.c_uint32), ("primary_max_depth", C.c_uint32), ("build_seconds", C.c_double),
		("textured", C.c_int), ("d_texture_data", C.c_void_p), ("d_texture_dims", C.c_void_p), ("d_texture_offsets", C.c_void_p), ("texture_texel_count", C.c_uint64), ("shadow_bvh_width", C.c_uint32),
		("d_shadow_nodes_quantised", C.c_void_p), ("shadow_grid", C.c_float * 6), ("d_shadow_nodes_interleaved", C.c_void_p)]


class LtcConstants(C.Structure):
	_fields_ = [("fresnel_index_factor", C.c_float), ("fresnel_index_summand", C.c_float), ("roughness_factor", C.c_float), ("roughness_summand", C.c_float),
		("inclination_factor", C.c_float), ("inclination_summand", C.c_float), ("padding", C.c_float * 2)]


class LtcTable(C.Structure):
	_fields_ = [("roughness_count", C.c_uint32), ("inclination_count", C.c_uint32), ("fresnel_count", C.c_uint32),
		("d_table0", C.c_void_p), ("d_table1", C.c_void_p), ("h_table0", C.POINTER(C.c_uint16)), ("h_table1", C.POINTER(C.c_uint16)),
		("constants", LtcConstants)]


class NoiseTable(C.Structure):
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("layers", C.c_uint32), ("d_noise", C.c_void_p), ("h_noise", C.POINTER(C.c_uint16)), ("random_seed", C.c_uint32)]


class Camera(C.Structure):
	_fields_ = [("position_world_space", C.c_float * 3), ("rotation_z", C.c_float), ("rotation_x", C.c_float), ("vertical_fov", C.c_float),
		("near_plane", C.c_float), ("far_plane", C.c_float), ("speed", C.c_float), ("rotate_camera", C.c_int), ("rotation_x_0", C.c_float), ("rotation_z_0", C.c_float)]


class PolygonalLight(C.Structure):
	_fields_ = [("rotation_angles", C.c_float * 3), ("scaling_x", C.c_float), ("translation", C.c_float * 3), ("scaling_y", C.c_float),
		("radiant_flux", C.c_float * 3), ("inv_scaling_x", C.c_float), ("surface_radiance", C.c_float * 3), ("inv_scaling_y", C.c_float),
		("plane", C.c_float * 4), ("vertex_count", C.c_uint32), ("texturing_technique", C.c_uint32), ("texture_index", C.c_uint32), ("padding_0", C.c_uint32),
		("rotation", (C.c_float * 4) * 3), ("area", C.c_float), ("rcp_area", C.c_float), ("padding_1", C.c_float * 2),
		("texture_file_path", C.c_void_p), ("vertices_plane_space", C.POINTER(C.c_float)), ("vertices_world_space", C.POINTER(C.c_float)), ("fan_areas", C.POINTER(C.c_float))]


class SceneSpecification(C.Structure):
	_fields_ = [("camera", Camera), ("polygonal_light_count", C.c_uint32), ("polygonal_lights", C.POINTER(PolygonalLight))]


class RenderSettings(C.Structure):
	_fields_ = [("exposure_factor", C.c_float), ("roughness_factor", C.c_float), ("sample_count", C.c_uint32), ("sampling_strategies", C.c_int), ("mis_heuristic", C.c_int),
		("mis_visibility_estimate", C.c_float), ("polygon_sampling_technique", C.c_int), ("error_min_exponent", C.c_float),
		("animate_noise", C.c_int), ("trace_shadow_rays", C.c_int), ("show_polygonal_lights", C.c_int)]


class Texture(C.Structure):
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("mip_count", C.c_uint32), ("vk_format", C.c_uint32), ("h_texels", C.POINTER(C.c_float)),
		("texel_float_count", C.c_uint64), ("is_constant", C.c_int)]


class RenderTargets(C.Structure):
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("d_visibility", C.c_void_p), ("d_gbuffer", C.c_void_p), ("d_frame", C.c_void_p)]


class LightTextures(C.Structure):
	_fields_ = [("texture_count", C.c_uint32), ("textures", C.POINTER(Texture)), ("d_texels", C.c_void_p), ("d_dims", C.c_void_p), ("d_offsets", C.c_void_p), ("texel_count", C.c_uint64)]


class ShadingPassDesc(C.Structure):
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("polygonal_light_count", C.c_uint32),
		("min_polygonal_light_vertex_count", C.c_uint32), ("max_polygonal_light_vertex_count", C.c_uint32), ("sample_count", C.c_uint32),
		("sampling_strategies", C.c_int), ("mis_heuristic", C.c_int), ("polygon_sampling_technique", C.c_int),
		("trace_shadow_rays", C.c_int), ("show_polygonal_lights", C.c_int), ("stripe_index", C.c_uint32), ("stripe_count", C.c_uint32),
		("scene", C.POINTER(Scene)), ("ltc_table", C.POINTER(LtcTable)), ("noise_table", C.POINTER(NoiseTable)), ("output_srgb", C.c_int), ("error_display", C.c_int),
		("light_textures", C.POINTER(LightTextures))]


class ShadingPass(C.Structure):
	_fields_ = [("desc", ShadingPassDesc), ("constants_size", C.c_size_t), ("d_constants", C.c_void_p), ("h_constants_pinned", C.c_void_p),
		("d_gbuffer_staging", C.c_void_p), ("d_out_staging", C.c_void_p), ("kernel_launches", C.c_uint64), ("last_kernel_ms", C.c_float),
		("event_begin", C.c_void_p), ("event_end", C.c_void_p), ("timing_enabled", C.c_int),
		("event_constants", C.c_void_p), ("tile_count", C.c_uint32), ("d_tile_list", C.c_void_p), ("h_tile_list", C.c_void_p),
		("d_tile_cost", C.c_void_p), ("h_tile_cost", C.c_void_p), ("event_costs", C.c_void_p), ("costs_pending", C.c_int), ("reorder_tiles", C.c_int),
		("d_subset_tiles", C.c_void_p), ("h_subset_tiles", C.c_void_p), ("event_subset", C.c_void_p)]


MAX_GPUS = 8   # VKR_MAX_GPUS


class FrameExchange(C.Structure):
	"""vkr_frame_exchange_t: one frame on several GPUs, pixels stored into every GPU's frame from the kernel epilogue (include/vkr_b200.h)."""
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("rank", C.c_uint32), ("world", C.c_uint32), ("d_block", C.c_void_p),
		("d_peer_blocks", C.c_void_p * MAX_GPUS), ("peer_is_ipc", C.c_int * MAX_GPUS), ("frames_exchanged", C.c_uint64), ("h_status", C.POINTER(C.c_int)), ("timeout_ns", C.c_uint64)]


class Accumulator(C.Structure):
	"""vkr_accumulator_t: running mean and sum of squared deviations of frames, float64 (include/vkr_b200.h)."""
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("frame_count", C.c_uint64), ("d_state", C.c_void_p), ("d_partials", C.c_void_p), ("h_partials", C.c_void_p)]


class Rasterizer(C.Structure):
	"""vkr_rasterizer_t: the rasterised visibility buffer (DESIGN.md §5 "Rasterised visibility")"""
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("triangle_capacity", C.c_uint64), ("d_keys", C.c_void_p), ("d_scratch", C.c_void_p),
		("d_constants", C.c_void_p), ("scratch_bytes", C.c_uint64), ("scan_temp_bytes", C.c_uint64), ("large_ctas", C.c_uint32)]


class AdaptiveAccumulator(C.Structure):
	"""vkr_adaptive_accumulator_t: the accumulator's state per 16x8 screen tile, with a frame count and an active flag per tile (include/vkr_b200.h)."""
	_fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("tiles_x", C.c_uint32), ("tiles_y", C.c_uint32), ("frame_count", C.c_uint64), ("active_tile_count", C.c_uint32),
		("d_state", C.c_void_p), ("d_tile_frames", C.c_void_p), ("d_tile_active", C.c_void_p), ("d_partials", C.c_void_p), ("h_partials", C.c_void_p)]


class FrameError(C.Structure):
	"""vkr_frame_error_t: a frame against a reference over the pixels with finite inputs."""
	_fields_ = [("mse", C.c_double * 3), ("rel_mse", C.c_double * 3), ("mae", C.c_double * 3), ("max_abs_error", C.c_double),
		("pixel_count", C.c_uint64), ("nonfinite_pixels", C.c_uint64)]


class LtcFitDesc(C.Structure):
	"""vkr_ltc_fit_desc_t: the size of an LTC table to fit and the fit's quadrature and iteration limit (include/vkr_b200.h)."""
	_fields_ = [("resolution", C.c_uint32), ("fresnel_count", C.c_uint32), ("quadrature_size", C.c_uint32), ("iteration_limit", C.c_uint32)]


class LtcFitStats(C.Structure):
	"""vkr_ltc_fit_stats_t: what a fit cost and how well its cells fit; cell_errors is set by the caller (NULL or F * N * N doubles)."""
	_fields_ = [("cell_count", C.c_uint64), ("objective_evaluations", C.c_uint64), ("iteration_limit_hits", C.c_uint64),
		("max_error", C.c_double), ("median_error", C.c_double), ("mean_error", C.c_double), ("fit_ms", C.c_float), ("cell_errors", C.POINTER(C.c_double))]


class NoiseGenDesc(C.Structure):
	"""vkr_noise_gen_desc_t: the type, size and seed of a noise table to generate (include/vkr_b200.h)."""
	_fields_ = [("type", C.c_int), ("width", C.c_uint32), ("height", C.c_uint32), ("layers", C.c_uint32), ("seed", C.c_uint32)]


class NoiseGenStats(C.Structure):
	"""vkr_noise_gen_stats_t: the generating kernel's time and, for dither arrays, the relaxations stopped at the iteration limit."""
	_fields_ = [("kernel_ms", C.c_float), ("relaxation_limit_hits", C.c_uint32)]


TRACE_COUNTER_NAMES = ["rays", "occluded", "cache_hits", "node_visits", "leaf_visits", "triangle_tests", "warp_rounds", "warp_node_steps", "known_occluded", "idle_polls",
	"entries", "resolve_polls", "candidates"]   # vkr_trace_counter_t
TRACE_COUNTER_COUNT = 16

_lib = None


def load_library():
	"""Loads libvkr_b200.so. Raises (never falls back) when the CUDA library is missing."""
	global _lib
	if _lib is not None:
		return _lib
	if not os.path.exists(LIB_PATH):
		raise RuntimeError("%s is missing: run `python __graft_entry__.py` (build()) first. There is no CPU fallback." % LIB_PATH)
	lib = C.CDLL(LIB_PATH)
	missing = [s for s in EXPORTED_SYMBOLS if not hasattr(lib, s)]
	if missing:
		raise RuntimeError("libvkr_b200.so lacks symbols declared in include/vkr_b200.h: %s" % missing)
	P = C.POINTER
	lib.vkr_abi_version.restype = C.c_uint32
	lib.vkr_create_device.argtypes = [P(Device), C.c_int, C.c_void_p]
	lib.vkr_destroy_device.argtypes = [P(Device)]; lib.vkr_destroy_device.restype = None
	lib.vkr_device_wait_idle.argtypes = [P(Device)]
	lib.vkr_load_scene.argtypes = [P(Scene), P(Device), C.c_char_p, C.c_char_p, C.c_int]
	lib.vkr_destroy_scene.argtypes = [P(Scene), P(Device)]; lib.vkr_destroy_scene.restype = None
	lib.vkr_load_ltc_table.argtypes = [P(LtcTable), P(Device), C.c_char_p, C.c_uint32]
	lib.vkr_destroy_ltc_table.argtypes = [P(LtcTable), P(Device)]; lib.vkr_destroy_ltc_table.restype = None
	lib.vkr_load_noise_table.argtypes = [P(NoiseTable), P(Device), C.c_uint32, C.c_uint32, C.c_uint32, C.c_int]
	lib.vkr_destroy_noise_table.argtypes = [P(NoiseTable), P(Device)]; lib.vkr_destroy_noise_table.restype = None
	lib.vkr_set_noise_constants.argtypes = [P(C.c_uint32), P(C.c_uint32), P(C.c_uint32), P(NoiseTable), C.c_int]; lib.vkr_set_noise_constants.restype = None
	lib.vkr_update_polygonal_light.argtypes = [P(PolygonalLight)]; lib.vkr_update_polygonal_light.restype = None
	lib.vkr_set_polygonal_light_vertex_count.argtypes = [P(PolygonalLight), C.c_uint32]; lib.vkr_set_polygonal_light_vertex_count.restype = None
	lib.vkr_destroy_polygonal_light.argtypes = [P(PolygonalLight)]; lib.vkr_destroy_polygonal_light.restype = None
	lib.vkr_get_world_to_projection_space.argtypes = [C.c_void_p, P(Camera), C.c_float]; lib.vkr_get_world_to_projection_space.restype = None
	lib.vkr_quick_load.argtypes = [P(SceneSpecification), C.c_char_p]
	lib.vkr_quick_save.argtypes = [P(SceneSpecification), C.c_char_p]
	lib.vkr_destroy_scene_specification.argtypes = [P(SceneSpecification)]; lib.vkr_destroy_scene_specification.restype = None
	lib.vkr_specify_default_render_settings.argtypes = [P(RenderSettings)]; lib.vkr_specify_default_render_settings.restype = None
	lib.vkr_get_constants_size.argtypes = [P(SceneSpecification)]; lib.vkr_get_constants_size.restype = C.c_size_t
	lib.vkr_write_constants.argtypes = [C.c_void_p, P(SceneSpecification), P(RenderSettings), P(Scene), P(LtcTable), P(NoiseTable), C.c_uint32, C.c_uint32]
	lib.vkr_write_constants.restype = C.c_size_t
	lib.vkr_set_frame_bits.argtypes = [C.c_void_p, C.c_uint32]; lib.vkr_set_frame_bits.restype = None
	lib.vkr_gbuffer_size.argtypes = [C.c_uint32, C.c_uint32]; lib.vkr_gbuffer_size.restype = C.c_size_t
	lib.vkr_run_visibility_pass.argtypes = [P(Device), P(Scene), C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
	lib.vkr_run_gbuffer_pass.argtypes = [P(Device), P(Scene), C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
	lib.vkr_create_shading_pass.argtypes = [P(ShadingPass), P(Device), P(ShadingPassDesc)]
	lib.vkr_destroy_shading_pass.argtypes = [P(ShadingPass), P(Device)]; lib.vkr_destroy_shading_pass.restype = None
	lib.vkr_shading_pass_run.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
	lib.vkr_shading_pass_run_host.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
	lib.vkr_shading_pass_wait.argtypes = [P(ShadingPass), P(Device)]
	lib.vkr_shading_pass_run_tiles.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
	lib.vkr_shading_pass_run_with_counters.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, P(C.c_uint64)]
	lib.vkr_create_frame_exchange.argtypes = [P(FrameExchange), P(Device), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
	lib.vkr_destroy_frame_exchange.argtypes = [P(FrameExchange), P(Device)]; lib.vkr_destroy_frame_exchange.restype = None
	lib.vkr_frame_exchange_get_handle.argtypes = [P(FrameExchange), P(Device), C.c_void_p]
	lib.vkr_frame_exchange_connect.argtypes = [P(FrameExchange), P(Device), C.c_void_p]
	lib.vkr_frame_exchange_connect_local.argtypes = [P(FrameExchange), P(Device), P(C.c_void_p)]
	lib.vkr_frame_exchange_frame.argtypes = [P(FrameExchange)]; lib.vkr_frame_exchange_frame.restype = C.c_void_p
	lib.vkr_shading_pass_run_exchange.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, P(FrameExchange)]
	lib.vkr_shading_pass_run_host_exchange.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, P(FrameExchange), C.c_void_p]
	lib.vkr_frame_exchange_wait.argtypes = [P(FrameExchange), P(Device)]
	lib.vkr_frame_exchange_download.argtypes = [P(FrameExchange), P(Device), C.c_void_p]
	lib.vkr_trace_shadow_rays.argtypes = [P(Device), P(Scene), C.c_uint32, C.c_void_p, C.c_void_p]
	lib.vkr_sample_polygon_batch.argtypes = [P(Device), C.c_uint32, C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
	lib.vkr_sample_related_work_batch.argtypes = [P(Device), C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, P(C.c_float), P(C.c_int32)]
	lib.vkr_probe_rsqrt_exhaustive.argtypes = [P(Device), P(C.c_uint64), P(C.c_uint32)]
	lib.vkr_bvh_build_probe.argtypes = [C.c_void_p, C.c_uint64, P(P(C.c_float)), P(C.c_uint64), P(P(C.c_float)), P(P(C.c_uint32)), P(C.c_uint32)]
	lib.vkr_bvh_build_probe_with.argtypes = [C.c_int, C.c_void_p, C.c_uint64, P(P(C.c_float)), P(C.c_uint64), P(P(C.c_float)), P(P(C.c_uint32)), P(C.c_uint32)]
	lib.vkr_bvh_build_probe_device.argtypes = [P(Device), C.c_void_p, C.c_uint64, P(P(C.c_float)), P(C.c_uint64), P(P(C.c_float)), P(P(C.c_uint32)), P(C.c_uint32)]
	lib.vkr_bvh4_build_probe.argtypes = [C.c_void_p, C.c_uint64, P(P(C.c_float)), P(C.c_uint64), P(P(C.c_float)), P(P(C.c_uint32)), P(C.c_uint32), P(C.c_uint64), P(C.c_uint32)]
	lib.vkr_bvh_free_probe.argtypes = [P(C.c_float), P(C.c_float), P(C.c_uint32)]; lib.vkr_bvh_free_probe.restype = None
	lib.vkr_load_texture.argtypes = [P(Texture), C.c_char_p]
	lib.vkr_create_and_assign_light_textures.argtypes = [P(LightTextures), P(Device), P(SceneSpecification)]
	lib.vkr_destroy_light_textures.argtypes = [P(LightTextures), P(Device)]; lib.vkr_destroy_light_textures.restype = None
	lib.vkr_destroy_texture.argtypes = [P(Texture)]; lib.vkr_destroy_texture.restype = None
	lib.vkr_create_render_targets.argtypes = [P(RenderTargets), P(Device), C.c_uint32, C.c_uint32]
	lib.vkr_destroy_render_targets.argtypes = [P(RenderTargets), P(Device)]; lib.vkr_destroy_render_targets.restype = None
	lib.vkr_download_frame.argtypes = [P(RenderTargets), P(Device), C.c_void_p]
	lib.vkr_download_gbuffer.argtypes = [P(RenderTargets), P(Device), C.c_void_p, C.c_void_p]
	lib.vkr_upload_gbuffer.argtypes = [P(RenderTargets), P(Device), C.c_void_p]
	lib.vkr_quantize_unorm8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]; lib.vkr_quantize_unorm8.restype = None
	lib.vkr_combine_ldr_screenshots_into_hdr.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]; lib.vkr_combine_ldr_screenshots_into_hdr.restype = None
	lib.vkr_write_png.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p]
	lib.vkr_write_hdr.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p]
	lib.vkr_take_screenshot.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_char_p]
	lib.vkr_take_screenshot_formats.argtypes = [P(ShadingPass), P(Device), C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p]
	lib.vkr_quantize_unorm8_device.argtypes = [P(Device), C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
	lib.vkr_encode_jpg.argtypes = [P(Device), C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, P(C.c_size_t)]
	lib.vkr_write_jpg.argtypes = [P(Device), C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int]
	lib.vkr_record_frame_time.argtypes = [C.c_double]; lib.vkr_record_frame_time.restype = None
	lib.vkr_get_frame_time.argtypes = []; lib.vkr_get_frame_time.restype = C.c_float
	lib.vkr_reset_frame_times.argtypes = []; lib.vkr_reset_frame_times.restype = None
	lib.vkr_create_rasterizer.argtypes = [P(Rasterizer), P(Device), C.c_uint32, C.c_uint32, C.c_uint64]
	lib.vkr_destroy_rasterizer.argtypes = [P(Rasterizer), P(Device)]; lib.vkr_destroy_rasterizer.restype = None
	lib.vkr_rasterize_visibility.argtypes = [P(Rasterizer), P(Device), P(Scene), C.c_void_p, C.c_void_p, C.c_void_p]
	lib.vkr_create_accumulator.argtypes = [P(Accumulator), P(Device), C.c_uint32, C.c_uint32]
	lib.vkr_destroy_accumulator.argtypes = [P(Accumulator), P(Device)]; lib.vkr_destroy_accumulator.restype = None
	lib.vkr_accumulator_reset.argtypes = [P(Accumulator), P(Device)]
	lib.vkr_accumulate_frame.argtypes = [P(Accumulator), P(Device), C.c_void_p]
	lib.vkr_accumulator_resolve.argtypes = [P(Accumulator), P(Device), C.c_void_p, C.c_void_p]
	lib.vkr_accumulator_mean_variance.argtypes = [P(Accumulator), P(Device), P(C.c_double)]
	lib.vkr_compare_frames.argtypes = [P(Device), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, P(FrameError)]
	lib.vkr_create_adaptive_accumulator.argtypes = [P(AdaptiveAccumulator), P(Device), C.c_uint32, C.c_uint32]
	lib.vkr_destroy_adaptive_accumulator.argtypes = [P(AdaptiveAccumulator), P(Device)]; lib.vkr_destroy_adaptive_accumulator.restype = None
	lib.vkr_adaptive_accumulator_reset.argtypes = [P(AdaptiveAccumulator), P(Device)]
	lib.vkr_adaptive_accumulate_frame.argtypes = [P(AdaptiveAccumulator), P(Device), C.c_void_p]
	lib.vkr_adaptive_update_tiles.argtypes = [P(AdaptiveAccumulator), P(Device), C.c_double, C.c_uint32, C.c_uint32, C.c_void_p, P(C.c_uint32)]
	lib.vkr_adaptive_tile_frames.argtypes = [P(AdaptiveAccumulator), P(Device), C.c_void_p]
	lib.vkr_adaptive_resolve.argtypes = [P(AdaptiveAccumulator), P(Device), C.c_void_p, C.c_void_p]
	lib.vkr_adaptive_estimated_rel_mse.argtypes = [P(AdaptiveAccumulator), P(Device), P(C.c_double)]
	lib.vkr_ltc_fit_default_desc.argtypes = [P(LtcFitDesc)]; lib.vkr_ltc_fit_default_desc.restype = None
	lib.vkr_fit_ltc_table.argtypes = [P(Device), P(LtcFitDesc), C.c_void_p, P(LtcFitStats)]
	lib.vkr_write_ltc_fits.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p]
	lib.vkr_noise_table_from_image.argtypes = [P(NoiseTable), P(Device), C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32]
	lib.vkr_noise_gen_default_desc.argtypes = [C.c_int, P(NoiseGenDesc)]; lib.vkr_noise_gen_default_desc.restype = None
	lib.vkr_generate_noise_table.argtypes = [P(Device), P(NoiseGenDesc), C.c_void_p, P(NoiseGenStats)]
	lib.vkr_write_noise_table.argtypes = [C.c_char_p, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
	_lib = lib
	return lib
