"""Convenience wrapper: one scene + camera + lights + settings -> device resources and passes.

Everything here goes through the C-ABI (include/vkr_b200.h); no computation happens in Python.
"""
import ctypes as C

import numpy as np

from . import api


class Frame:
	"""Owns device, scene, LTC table, noise table and the scene specification of one dataset."""

	def __init__(self, vks, textures, save, ltc_dir, cuda_device=0, stream=None, noise=(256, 256, 64), fresnel_count=51, request_acceleration_structure=True,
		noise_type=api.NOISE_WHITE, noise_root=None):
		"""noise = (width, height, layers) of the noise table. noise_type api.NOISE_BLUE or api.NOISE_AHMED reads the table from
		<noise_root>/data/noise/<the loader's file name> (e.g. written by tools/make_noise_tables.py) and uploads it with the loader's initial seed."""
		self.lib = api.load_library()
		self.device = api.Device(); self.scene = api.Scene(); self.ltc = api.LtcTable(); self.noise = api.NoiseTable()
		self.spec = api.SceneSpecification(); self.settings = api.RenderSettings()
		self._passes = []
		self._check(self.lib.vkr_create_device(C.byref(self.device), cuda_device, stream), "vkr_create_device")
		self._check(self.lib.vkr_load_scene(C.byref(self.scene), C.byref(self.device), vks.encode(), textures.encode(), int(request_acceleration_structure)), "vkr_load_scene")
		self._check(self.lib.vkr_load_ltc_table(C.byref(self.ltc), C.byref(self.device), ltc_dir.encode(), fresnel_count), "vkr_load_ltc_table")
		if noise_type == api.NOISE_WHITE:
			self._check(self.lib.vkr_load_noise_table(C.byref(self.noise), C.byref(self.device), noise[0], noise[1], noise[2], api.NOISE_WHITE), "vkr_load_noise_table")
		else:
			from .noise_gen import LOADER_SEED, read_noise_table
			if noise_root is None:
				raise ValueError("noise type %d is read from a file: pass noise_root" % noise_type)
			texels = read_noise_table(noise_root, noise_type, *noise)
			self._check(self.lib.vkr_noise_table_from_image(C.byref(self.noise), C.byref(self.device), noise[0], noise[1], noise[2], texels.ctypes.data, LOADER_SEED), "vkr_noise_table_from_image")
		self._check(self.lib.vkr_quick_load(C.byref(self.spec), save.encode()), "vkr_quick_load")
		# create_and_assign_light_textures (src/main.c:371): texture indices for all lights; the textures go to the device only if a light is textured
		self.light_textures = api.LightTextures()
		if any(self.spec.polygonal_lights[i].texturing_technique != 0 for i in range(self.spec.polygonal_light_count)):
			self._check(self.lib.vkr_create_and_assign_light_textures(C.byref(self.light_textures), C.byref(self.device), C.byref(self.spec)), "vkr_create_and_assign_light_textures")
		else:
			self._check(self.lib.vkr_create_and_assign_light_textures(None, None, C.byref(self.spec)), "vkr_create_and_assign_light_textures")
		self.lib.vkr_specify_default_render_settings(C.byref(self.settings))
		self.settings.animate_noise = 0
		self.settings.exposure_factor = 1.0

	@staticmethod
	def _check(code, what):
		if code != 0:
			raise RuntimeError("%s failed with code %d" % (what, code))

	# ---- settings
	def configure(self, sample_count=None, strategy=None, heuristic=None, technique=None, trace_shadow_rays=None, show_lights=None, light_count=None, output_srgb=None, frame_bits=None, error_display=None):
		s = self.settings
		if error_display is not None: self.error_display = int(error_display)   # render_settings_t::error_display (src/main.h:150)
		if output_srgb is not None: self.output_srgb = int(output_srgb)     # !OUTPUT_LINEAR_RGB (src/main.c:790)
		if frame_bits is not None: self.frame_bits = int(frame_bits)         # screenshot.frame_bits (src/main.c:2132)
		if sample_count is not None: s.sample_count = sample_count
		if strategy is not None: s.sampling_strategies = strategy
		if heuristic is not None: s.mis_heuristic = heuristic
		if technique is not None: s.polygon_sampling_technique = technique
		if trace_shadow_rays is not None: s.trace_shadow_rays = int(trace_shadow_rays)
		if show_lights is not None: s.show_polygonal_lights = int(show_lights)
		if light_count is not None:
			if light_count > self.spec.polygonal_light_count:
				raise ValueError("the quicksave holds only %d lights" % self.spec.polygonal_light_count)
			self._light_count_override = light_count
		return self

	@property
	def light_count(self):
		return getattr(self, "_light_count_override", self.spec.polygonal_light_count)

	def light_vertex_counts(self):
		return [self.spec.polygonal_lights[i].vertex_count for i in range(self.light_count)]

	def constants(self, width, height):
		"""The constant block exactly as the reference's write_constants() lays it out (bytes)."""
		spec = self.spec
		saved = spec.polygonal_light_count
		spec.polygonal_light_count = self.light_count
		try:
			size = self.lib.vkr_get_constants_size(C.byref(spec))
			buf = (C.c_uint8 * size)()
			written = self.lib.vkr_write_constants(buf, C.byref(spec), C.byref(self.settings), C.byref(self.scene), C.byref(self.ltc), C.byref(self.noise), width, height)
			assert written == size, (written, size)
			if getattr(self, "frame_bits", 0):
				self.lib.vkr_set_frame_bits(buf, self.frame_bits)
		finally:
			spec.polygonal_light_count = saved
		return bytes(buf)

	def pass_desc(self, width, height, stripe_index=0, stripe_count=1):
		s = self.settings
		counts = self.light_vertex_counts() or [3]
		d = api.ShadingPassDesc()
		d.width, d.height = width, height
		d.polygonal_light_count = self.light_count
		d.min_polygonal_light_vertex_count = min(counts); d.max_polygonal_light_vertex_count = max(max(counts), 3)
		d.sample_count = s.sample_count
		d.sampling_strategies = s.sampling_strategies; d.mis_heuristic = s.mis_heuristic; d.polygon_sampling_technique = s.polygon_sampling_technique
		d.trace_shadow_rays = s.trace_shadow_rays; d.show_polygonal_lights = s.show_polygonal_lights
		d.stripe_index, d.stripe_count = stripe_index, stripe_count
		d.scene = C.pointer(self.scene); d.ltc_table = C.pointer(self.ltc); d.noise_table = C.pointer(self.noise)
		d.output_srgb = getattr(self, "output_srgb", 0)
		d.error_display = getattr(self, "error_display", 0)
		d.light_textures = C.pointer(self.light_textures) if self.light_textures.texture_count else None
		return d

	def create_pass(self, width, height, stripe_index=0, stripe_count=1, timing=False):
		p = api.ShadingPass()
		desc = self.pass_desc(width, height, stripe_index, stripe_count)
		self._check(self.lib.vkr_create_shading_pass(C.byref(p), C.byref(self.device), C.byref(desc)), "vkr_create_shading_pass")
		p.timing_enabled = int(timing)
		self._passes.append(p)
		return p

	def destroy_pass(self, p):
		self.lib.vkr_destroy_shading_pass(C.byref(p), C.byref(self.device))
		self._passes = [q for q in self._passes if q is not p]

	# ---- host-buffer conveniences built on cudaMalloc'ed scratch inside the library (tests, smoke)
	def gbuffer_host(self, width, height, visibility="ray"):
		"""Runs the visibility + G-buffer producer on the device and returns (visibility, gbuffer) as numpy arrays. visibility = "ray": the primary-ray
		cast (vkr_run_visibility_pass, needs the acceleration structure); "raster": the reference's subpass 0, culled and clipped (vkr_rasterize_visibility)."""
		import torch
		if visibility not in ("ray", "raster"):
			raise ValueError("visibility must be 'ray' or 'raster', not %r" % (visibility,))
		dev = torch.device("cuda", self.device.cuda_device)
		with torch.cuda.device(dev):
			vis = torch.empty((height, width), dtype=torch.int32, device=dev)
			gb = torch.empty((4, height, width, 4), dtype=torch.float32, device=dev)
			constants = self.constants(width, height)
			torch.cuda.synchronize()
			if visibility == "ray":
				self._check(self.lib.vkr_run_visibility_pass(C.byref(self.device), C.byref(self.scene), constants, width, height, vis.data_ptr()), "vkr_run_visibility_pass")
			else:
				r = api.Rasterizer()
				self._check(self.lib.vkr_create_rasterizer(C.byref(r), C.byref(self.device), width, height, max(self.scene.triangle_count, 1)), "vkr_create_rasterizer")
				try:
					self._check(self.lib.vkr_rasterize_visibility(C.byref(r), C.byref(self.device), C.byref(self.scene), constants, vis.data_ptr(), None), "vkr_rasterize_visibility")
				finally:
					self.lib.vkr_destroy_rasterizer(C.byref(r), C.byref(self.device))
			self._check(self.lib.vkr_run_gbuffer_pass(C.byref(self.device), C.byref(self.scene), constants, width, height, vis.data_ptr(), gb.data_ptr()), "vkr_run_gbuffer_pass")
			self._check(self.lib.vkr_device_wait_idle(C.byref(self.device)), "vkr_device_wait_idle")
			return vis.cpu().numpy().view(np.uint32), gb.cpu().numpy()

	def shade_host(self, width, height, gbuffer, stripe_index=0, stripe_count=1, out=None):
		"""End-to-end call with host buffers (vkr_shading_pass_run_host). Returns float32 [H, W, 4]."""
		p = self.create_pass(width, height, stripe_index, stripe_count)
		try:
			constants = self.constants(width, height)
			gb = np.ascontiguousarray(gbuffer, dtype=np.float32)
			if out is None:
				out = np.zeros((height, width, 4), dtype=np.float32)
			self._check(self.lib.vkr_shading_pass_run_host(C.byref(p), C.byref(self.device), constants, len(constants), gb.ctypes.data, out.ctypes.data), "vkr_shading_pass_run_host")
		finally:
			self.destroy_pass(p)
		return out

	def close(self):
		for p in list(self._passes):
			self.destroy_pass(p)
		dev = C.byref(self.device)
		self.lib.vkr_destroy_light_textures(C.byref(self.light_textures), dev)
		self.lib.vkr_destroy_scene_specification(C.byref(self.spec))
		self.lib.vkr_destroy_noise_table(C.byref(self.noise), dev)
		self.lib.vkr_destroy_ltc_table(C.byref(self.ltc), dev)
		self.lib.vkr_destroy_scene(C.byref(self.scene), dev)
		self.lib.vkr_destroy_device(dev)
