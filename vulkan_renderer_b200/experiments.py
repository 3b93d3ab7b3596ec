"""The reference's experiment list as a batch driver (SURVEY 8 row f3).

The reference defines its own benchmark in src/experiment_list.c: a table of (scene, quicksave, resolution, render settings,
screenshot path) that the application cycles through, writing the median frame time in milliseconds into each screenshot's
file name (advance_experiments, src/main.c:1948-2016; get_frame_time, src/frame_timer.c:43-75). This module rebuilds

  * the run-time measurements of the polygon sampling techniques (src/experiment_list.c:366-409): 3 to 7 light vertices x
    central / decentral configuration x (128 lights, 1 sample | 1 light, 128 samples) x the 13 sampling techniques,
    1920x1080, diffuse shading only, shadow rays and light display off,
  * the figure experiments that need no light textures: attic strategies and sampling error (:66-128), small distant lights (:130-168), the MIS
    heuristics on a shadowed plane (:170-220), the Cornell box with every technique (:222-266), the bias test (:268-292), the roughness planes (:316-339),

on the synthetic stand-ins of the scenes (vulkan_renderer_b200.synth; the reference's assets are not in its repository) and
runs them through the C-ABI: one shading pass per experiment, frame time = the median of the recorded frame times, kernel
times from CUDA events. Output: one JSON record per experiment and, optionally, the screenshot (*.png or *.hdr). convergence_groups() and
run_convergence() measure the figures' error against converged references and their noise (vulkan_renderer_b200.convergence).
Everything that computes goes through libvkr_b200.so; there is no CPU fallback.
"""
import ctypes as C
import json
import os
import time

from . import api, synth

# names used in the screenshot paths (src/experiment_list.c:37-50), index = sample_polygon_technique_t
SAMPLE_POLYGON_NAME = ["baseline", "area_turk", "rectangle_solid_angle_urena", "solid_angle_arvo", "solid_angle_ours", "clipped_solid_angle_ours",
	"bilinear_cosine_warp_hart", "bilinear_cosine_warp_clipping_hart", "biquadratic_cosine_warp_hart", "biquadratic_cosine_warp_clipping_hart",
	"projected_solid_angle_arvo", "projected_solid_angle_ours", "projected_solid_angle_biased_ours"]


def _settings(**kw):
	"""render_settings_t of one experiment; the defaults are those every block of the reference's list starts from."""
	s = dict(exposure_factor=8.0, roughness_factor=1.0, sample_count=1, sampling_strategies=api.STRATEGY_DIFFUSE_ONLY, mis_heuristic=api.MIS_BALANCE,
		mis_visibility_estimate=0.5, error_min_exponent=-7.0, polygon_sampling_technique=api.TECHNIQUE_PSA, animate_noise=0, trace_shadow_rays=1, show_polygonal_lights=1)
	s.update(kw)
	return s


def timing_experiments():
	"""src/experiment_list.c:366-409: 5 vertex counts x 2 configurations x 2 light/sample splits x 13 techniques = 260 experiments."""
	out = []
	for vertex_count in range(3, 8):
		for central in (True, False):
			for many_lights in (True, False):
				for technique in range(len(SAMPLE_POLYGON_NAME)):
					configuration = "central_" if central else "decentral_"
					light_count = 128 if many_lights else 1
					suffix = "_128" if many_lights else ""
					out.append(dict(
						name="timings_%s%d%s_%s" % (configuration, vertex_count, suffix, SAMPLE_POLYGON_NAME[technique]),
						screenshot_path="data/experiments/timings_%s%d%s_%s_%%.3f.png" % (configuration, vertex_count, suffix, SAMPLE_POLYGON_NAME[technique]),
						quick_save_path="data/quicksaves/roughness_planes_%s%d%s.save" % (configuration, vertex_count, suffix),
						scene="roughness_planes", scene_parameters=dict(vertices=vertex_count, central=int(central), lights=light_count),
						width=1920, height=1080, light_count=light_count,
						settings=_settings(polygon_sampling_technique=technique, sample_count=1 if many_lights else 128,
							exposure_factor=8.0 / float(light_count), trace_shadow_rays=0, show_polygonal_lights=0)))
	return out


def _figure(name, scene, width, height, scene_parameters=None, quick_save_path=None, **settings):
	return dict(name=name, screenshot_path="data/experiments/%s_%%.3f.png" % name, scene=scene, scene_parameters=scene_parameters or {}, quick_save_path=quick_save_path,
		width=width, height=height, light_count=None, settings=_settings(**settings))


def attic_experiments():
	"""src/experiment_list.c:66-110: the attic with different sampling strategies (2 samples per pixel in total each) and a reference."""
	make = lambda name, **kw: _figure(name, "room", 1440, 1440, **kw)
	return [
		make("attic_solid_angle_and_ggx_mis_2spp", sampling_strategies=api.STRATEGY_DIFFUSE_GGX_MIS, polygon_sampling_technique=api.TECHNIQUE_SOLID_ANGLE),
		make("attic_projected_solid_angle_ours_and_ggx_mis_2spp", sampling_strategies=api.STRATEGY_DIFFUSE_GGX_MIS),
		make("attic_projected_solid_angle_ours_2spp", sampling_strategies=api.STRATEGY_DIFFUSE_ONLY, sample_count=2),
		make("attic_diffuse_and_specular_ours_clamped_optimal_mis_ours_2spp", sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_MIS, mis_heuristic=api.MIS_OPTIMAL_CLAMPED),
		make("attic_reference_128spp", sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_MIS, sample_count=64),
	]


def error_experiments():
	"""src/experiment_list.c:112-128: the sampling error in the attic, colour coded (error_display_t)."""
	base = dict(trace_shadow_rays=0, show_polygonal_lights=0, mis_heuristic=api.MIS_BALANCE)
	return [
		_figure("error_attic_backward", "room", 1440, 1440, error_display=api.ERROR_DISPLAY_DIFFUSE_BACKWARD, **base),
		_figure("error_attic_backward_times_psa", "room", 1440, 1440, error_display=api.ERROR_DISPLAY_DIFFUSE_BACKWARD_SCALED, **base),
	]


def small_light_experiments():
	"""src/experiment_list.c:130-168: a small and a tiny distant light in the Bistro, every diffuse technique except Hart's clipping variants."""
	out = []
	for size in ("small", "tiny"):
		save = "data/quicksaves/Bistro_outside_%s_light.save" % size
		for technique, label in enumerate(SAMPLE_POLYGON_NAME):
			if technique in (api.TECHNIQUE_BILINEAR_COSINE_WARP_CLIPPING_HART, api.TECHNIQUE_BIQUADRATIC_COSINE_WARP_CLIPPING_HART):
				continue
			out.append(_figure("bistro_%s_polygon_%s_1spp" % (size, label), "city", 1920, 1080, dict(light_size=size), save, exposure_factor=14.0, polygon_sampling_technique=technique))
		out.append(_figure("bistro_%s_polygon_reference_128spp" % size, "city", 1920, 1080, dict(light_size=size), save, exposure_factor=14.0,
			polygon_sampling_technique=api.TECHNIQUE_AREA_TURK, sample_count=128))
	return out


def mis_plane_experiments():
	"""src/experiment_list.c:170-220: a shadowed plane with every MIS heuristic, GGX MIS, the one-sample estimator and a reference."""
	names = ["balance_veach", "power_veach", "weighted_ours", "clamped_optimal_ours", "optimal_ours"]
	base = dict(sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_MIS)
	out = [_figure("mis_plane_%s_2spp" % label, "shadowed_plane", 1024, 1024, mis_heuristic=heuristic, **base) for heuristic, label in enumerate(names)]
	out.append(_figure("mis_plane_solid_angle_and_ggx_balance_veach_2spp", "shadowed_plane", 1024, 1024, sampling_strategies=api.STRATEGY_DIFFUSE_GGX_MIS, mis_heuristic=api.MIS_BALANCE))
	out.append(_figure("mis_plane_diffuse_and_specular_random_ours_1spp", "shadowed_plane", 1024, 1024, sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_RANDOM))
	out.append(_figure("mis_plane_reference_128spp", "shadowed_plane", 1024, 1024, mis_heuristic=api.MIS_BALANCE, sample_count=64, **base))
	return out


def cornell_box_experiments():
	"""src/experiment_list.c:222-266: the Cornell box with every diffuse technique, Arvo's with a tilted light, references."""
	out = [_figure("cornell_box_%s_1spp" % label, "cornell", 1024, 1024, polygon_sampling_technique=technique) for technique, label in enumerate(SAMPLE_POLYGON_NAME)]
	tilted = dict(scene_parameters=dict(tilted=1), quick_save_path="data/quicksaves/cornell_box_tilted_light.save")
	out.append(_figure("cornell_box_projected_solid_angle_arvo_tilted_1spp", "cornell", 1024, 1024, polygon_sampling_technique=api.TECHNIQUE_PROJECTED_SOLID_ANGLE_ARVO, **tilted))
	out.append(_figure("cornell_box_reference_tilted_128spp", "cornell", 1024, 1024, polygon_sampling_technique=api.TECHNIQUE_SOLID_ANGLE, sample_count=128, **tilted))
	out.append(_figure("cornell_box_reference_128spp", "cornell", 1024, 1024, polygon_sampling_technique=api.TECHNIQUE_SOLID_ANGLE, sample_count=128))
	return out


def shadowed_plane_experiments():
	"""src/experiment_list.c:268-292: 2048 samples per technique with the unbiased and the biased sampler (the view provokes the bias)."""
	base = dict(exposure_factor=10.0, sample_count=2048, sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_MIS, mis_heuristic=api.MIS_OPTIMAL_CLAMPED)
	return [_figure("shadowed_plane_reference_4096spp", "shadowed_plane", 1024, 1024, **base),
		_figure("shadowed_plane_biased_4096spp", "shadowed_plane", 1024, 1024, polygon_sampling_technique=api.TECHNIQUE_PSA_BIASED, **base)]


def ies_profile_experiments():
	"""src/experiment_list.c:294-314: the attic under a rectangular light with an IES profile (polygon_texturing_ies_profile)."""
	return [_figure("ies_profile_attic_2spp", "room", 1280, 1024, dict(ies_profile=1), "data/quicksaves/attic_ies_profile.save", exposure_factor=8.0,
		sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_MIS, mis_heuristic=api.MIS_OPTIMAL_CLAMPED)]


def roughness_planes_experiments():
	"""src/experiment_list.c:316-362: three planes of different roughness under a Lambertian emitter, then under a textured one (polygon_texturing_area)."""
	base = dict(exposure_factor=8.0, sampling_strategies=api.STRATEGY_DIFFUSE_SPECULAR_MIS, mis_heuristic=api.MIS_WEIGHTED)
	parameters = dict(vertices=4, central=1, lights=1)
	return [_figure("roughness_planes_lambertian_2spp", "roughness_planes", 2048 + 256, 1024, parameters, **base),
		_figure("roughness_planes_lambertian_diffuse_only_1spp", "roughness_planes", 2048 + 256, 1024, parameters, **dict(base, sampling_strategies=api.STRATEGY_DIFFUSE_ONLY)),
		_figure("roughness_planes_screen_2spp", "roughness_planes", 1280, 1024, dict(screen=1), "data/quicksaves/roughness_planes_screen.save", **dict(base, mis_heuristic=api.MIS_OPTIMAL_CLAMPED))]


def experiment_list(all_figs=True, all_timings=True):
	"""create_experiment_list (src/experiment_list.c:25-555) in its order; the figures for the HTML viewer are left out (html_figs = VK_FALSE in the reference)."""
	figures = (attic_experiments() + error_experiments() + small_light_experiments() + mis_plane_experiments() + cornell_box_experiments() + shadowed_plane_experiments()
		+ ies_profile_experiments() + roughness_planes_experiments())
	return (figures if all_figs else []) + (timing_experiments() if all_timings else [])


def prepare_data(experiment, data_root, ltc_dir=None, noise_root=None):
	"""Writes the synthetic scene + quicksave an experiment names (once) and returns the dataset description. ltc_dir: a directory of fit<i>.dat
	files (e.g. from tools/fit_ltc.py) that replaces the dataset's synthetic LTC table; None keeps it. noise_root: a directory holding
	data/noise/ahmed_2d_rgba_256x256_64.blob (e.g. from tools/make_noise_tables.py) to shade with the Ahmed-Wonka table the reference's experiment
	list names (src/experiment_list.c) instead of white noise; None keeps white noise."""
	tag = experiment["scene"] + "".join("_%s%s" % kv for kv in sorted(experiment["scene_parameters"].items()))
	info = synth.build_dataset(os.path.join(data_root, tag), experiment["scene"], **experiment["scene_parameters"])
	if ltc_dir is not None:
		info = dict(info, ltc=ltc_dir)
	if noise_root is not None:
		info = dict(info, noise_root=noise_root)
	return info


def open_dataset_frame(info, cuda_device=0):
	"""A Frame over a dataset of prepare_data, with the noise table it names."""
	from .frame import Frame
	noise_root = info.get("noise_root")
	return Frame(info["vks"], info["textures"], info["save"], info["ltc"], cuda_device=cuda_device,
		noise_type=api.NOISE_AHMED if noise_root is not None else api.NOISE_WHITE, noise_root=noise_root)


def _configure(frame, experiment):
	"""Applies an experiment's render settings and light count to a Frame."""
	for key, value in experiment["settings"].items():
		if key == "error_display":
			frame.configure(error_display=value)   # a pass setting (-D defines), not part of the constant block
		else:
			setattr(frame.settings, key, value)
	if experiment.get("light_count"):
		frame.configure(light_count=experiment["light_count"])


def run_experiment(experiment, data_root, out_dir=None, frames=12, warmup=3, width=None, height=None, cuda_device=0, screenshot=True, ltc_dir=None, noise_root=None):
	"""Runs one experiment like the application does: set up scene, lights and settings, render `warmup` + `frames` frames, take the
	median frame time, store the screenshot under its path with the time in milliseconds filled in. Returns the JSON record.
	ltc_dir: LTC table to shade with instead of the synthetic one; noise_root: Ahmed-Wonka table instead of white noise (prepare_data)."""
	info = prepare_data(experiment, data_root, ltc_dir, noise_root)
	width = width or experiment["width"]; height = height or experiment["height"]
	frame = open_dataset_frame(info, cuda_device)
	lib = frame.lib
	lib.vkr_get_frame_time.restype = C.c_float
	lib.vkr_record_frame_time.argtypes = [C.c_double]
	targets = api.RenderTargets()
	try:
		s = experiment["settings"]
		_configure(frame, experiment)
		constants = frame.constants(width, height)
		frame._check(lib.vkr_create_render_targets(C.byref(targets), C.byref(frame.device), width, height), "vkr_create_render_targets")
		frame._check(lib.vkr_run_visibility_pass(C.byref(frame.device), C.byref(frame.scene), constants, width, height, targets.d_visibility), "vkr_run_visibility_pass")
		frame._check(lib.vkr_run_gbuffer_pass(C.byref(frame.device), C.byref(frame.scene), constants, width, height, targets.d_visibility, targets.d_gbuffer), "vkr_run_gbuffer_pass")
		p = frame.create_pass(width, height, timing=True)
		lib.vkr_reset_frame_times()
		clock = 1.0   # the frame timer takes time stamps; kernel times from CUDA events are accumulated into one
		kernel_ms = []
		for i in range(warmup + frames):
			frame._check(lib.vkr_shading_pass_run(C.byref(p), C.byref(frame.device), constants, len(constants), targets.d_gbuffer, targets.d_frame), "vkr_shading_pass_run")
			frame._check(lib.vkr_shading_pass_wait(C.byref(p), C.byref(frame.device)), "vkr_shading_pass_wait")
			if i == warmup:
				lib.vkr_record_frame_time(clock)
			if i >= warmup:
				clock += 1.0e-3 * p.last_kernel_ms; lib.vkr_record_frame_time(clock); kernel_ms.append(float(p.last_kernel_ms))
		frame_time_ms = 1.0e3 * float(lib.vkr_get_frame_time())
		record = dict(name=experiment["name"], scene=experiment["scene"], quick_save_path=experiment["quick_save_path"], width=width, height=height,
			light_count=frame.light_count, light_vertex_counts=sorted(set(frame.light_vertex_counts())), settings=dict(s),
			frame_time_ms=round(frame_time_ms, 4), frames=frames, kernel_ms_min=round(min(kernel_ms), 4), kernel_ms_max=round(max(kernel_ms), 4),
			msamples_per_s=round(width * height * s["sample_count"] / frame_time_ms / 1.0e3, 3) if frame_time_ms > 0 else None,
			timed="shading kernel, CUDA events (the reference's number is the whole frame, src/main.c:2006)")
		if noise_root is not None:
			record["noise_root"] = noise_root
		if screenshot and out_dir is not None:
			path = os.path.join(out_dir, experiment["screenshot_path"] % frame_time_ms)
			os.makedirs(os.path.dirname(path), exist_ok=True)
			hdr = path.endswith(".hdr")
			frame._check(lib.vkr_take_screenshot(C.byref(p), C.byref(frame.device), constants, len(constants), targets.d_gbuffer, None if hdr else path.encode(), path.encode() if hdr else None), "vkr_take_screenshot")
			record["screenshot"] = path
		return record
	finally:
		lib.vkr_destroy_render_targets(C.byref(targets), C.byref(frame.device))
		frame.close()


def run(experiments, data_root, out_dir, json_path=None, **kw):
	"""Runs the experiments in order and writes the timing matrix as JSON (a list of records, see run_experiment)."""
	records = []
	for e in experiments:
		records.append(run_experiment(e, data_root, out_dir, **kw))
		print("%-70s %9.3f ms" % (records[-1]["name"], records[-1]["frame_time_ms"]), flush=True)
	if json_path:
		os.makedirs(os.path.dirname(os.path.abspath(json_path)), exist_ok=True)
		with open(json_path, "w") as f:
			json.dump(records, f, indent=1)
	return records


def convergence_groups():
	"""The figure experiments whose error can be measured, each with the experiment of the list that serves as its reference: same scene, scene
	parameters, quicksave, resolution, exposure and light display. Left out: the error displays (they show no radiance) and the figures without a
	reference of their own view (the IES profile attic, the textured screen)."""
	names = [e["name"] for e in experiment_list(all_timings=False)]
	def members(prefix, reference, exclude=()):
		return [n for n in names if n.startswith(prefix) and n != reference and n not in exclude]
	cornell_tilted = "cornell_box_projected_solid_angle_arvo_tilted_1spp"
	return [
		dict(name="attic", reference="attic_reference_128spp", members=members("attic_", "attic_reference_128spp")),
		dict(name="bistro_small", reference="bistro_small_polygon_reference_128spp", members=members("bistro_small_", "bistro_small_polygon_reference_128spp")),
		dict(name="bistro_tiny", reference="bistro_tiny_polygon_reference_128spp", members=members("bistro_tiny_", "bistro_tiny_polygon_reference_128spp")),
		dict(name="mis_plane", reference="mis_plane_reference_128spp", members=members("mis_plane_", "mis_plane_reference_128spp")),
		dict(name="cornell_box", reference="cornell_box_reference_128spp", members=members("cornell_box_", "cornell_box_reference_128spp", (cornell_tilted, "cornell_box_reference_tilted_128spp"))),
		dict(name="cornell_box_tilted", reference="cornell_box_reference_tilted_128spp", members=[cornell_tilted]),
		dict(name="shadowed_plane", reference="shadowed_plane_reference_4096spp", members=["shadowed_plane_biased_4096spp"]),   # the bias test
		dict(name="roughness_planes", reference="roughness_planes_lambertian_2spp", members=["roughness_planes_lambertian_diffuse_only_1spp"]),
	]


def run_convergence(group, data_root, out_dir, reference_frames, variance_frames, width=None, height=None, cuda_device=0, ltc_dir=None, noise_root=None, adaptive=None):
	"""Measures the members of one convergence group (convergence_groups()) against a converged reference: the reference experiment's settings
	averaged over `reference_frames` animated frames. Per member: its screenshot frame (animate_noise = 0, the frame run_experiment shades, in linear
	radiance) against that reference, and the mean per-frame variance over `variance_frames` animated frames. The record also holds the error of the
	reference experiment's own screenshot frame (reference_frame_error). With out_dir, the reference is stored as out_dir/convergence/<group>_reference.hdr.
	ltc_dir: LTC table for the reference and the members instead of the synthetic one; noise_root: Ahmed-Wonka table for the reference and the
	members instead of white noise (prepare_data). adaptive: a target relMSE; the reference is then built by convergence.accumulate_adaptive with
	max_frames = reference_frames, and the record's "adaptive" entry says what it shaded, what it cost and its estimated relMSE (its
	reference_mean_variance is None: the pixels average different frame counts). Returns the JSON record."""
	from . import convergence
	by_name = {e["name"]: e for e in experiment_list(all_timings=False)}

	def open_frame(experiment):
		frame = open_dataset_frame(prepare_data(experiment, data_root, ltc_dir, noise_root), cuda_device)
		_configure(frame, experiment)
		return frame

	ref_experiment = by_name[group["reference"]]
	w = width or ref_experiment["width"]; h = height or ref_experiment["height"]
	frame = open_frame(ref_experiment)
	try:
		if adaptive is None:
			reference = convergence.accumulate(frame, w, h, reference_frames, animate=True)
		else:
			start = time.perf_counter()
			reference = convergence.accumulate_adaptive(frame, w, h, reference_frames, adaptive)
			wall_s = time.perf_counter() - start
		# the reference experiment's own screenshot frame against the converged image: the error of one frame of these settings (for the bias test: unbiased)
		reference_frame_error = convergence.frame_error(frame, convergence.accumulate(frame, w, h, 1, animate=False).mean, reference.mean)
		if out_dir is not None:
			path = os.path.join(out_dir, "convergence", "%s_reference.hdr" % group["name"])
			os.makedirs(os.path.dirname(path), exist_ok=True)
			rgb = reference.mean[..., :3].copy()
			frame._check(frame.lib.vkr_write_hdr(path.encode(), w, h, rgb.ctypes.data), "vkr_write_hdr")
	finally:
		frame.close()
	record = dict(group=group["name"], reference=group["reference"], width=w, height=h, ltc=ltc_dir or "synthetic", reference_frames=reference_frames,
		reference_samples_per_pixel=ref_experiment["settings"]["sample_count"] * reference_frames,
		reference_mean_variance=list(reference.mean_variance) if adaptive is None and reference.mean_variance is not None else None,
		reference_frame_error=reference_frame_error, accumulate_ms_per_frame=round(reference.accumulate_ms_per_frame if adaptive is None else reference.accumulate_ms / reference.frames, 5),
		variance_frames=variance_frames, timed="accumulate kernel per frame at %dx%d, CUDA events" % (w, h), members=[])
	if adaptive is not None:
		record["adaptive"] = dict(target_rel_mse=adaptive, frames=reference.frames, estimated_rel_mse=list(reference.estimated_rel_mse),
			tile_frames_shaded=reference.tile_frames_shaded, tile_frames_full=reference.tile_frames_full,
			shaded_fraction=round(reference.tile_frames_shaded / reference.tile_frames_full, 5),
			tile_frames_min=int(reference.tile_frames.min()), tile_frames_max=int(reference.tile_frames.max()),
			shade_ms=round(reference.shade_ms, 3), accumulate_ms=round(reference.accumulate_ms, 3), wall_s=round(wall_s, 3),
			timed="shading and accumulate launches of the reference, CUDA events; wall_s: the whole adaptive reference, host clock")
	if noise_root is not None:
		record["noise_root"] = noise_root
	for name in group["members"]:
		experiment = by_name[name]
		frame = open_frame(experiment)
		try:
			screenshot = convergence.accumulate(frame, w, h, 1, animate=False).mean
			error = convergence.frame_error(frame, screenshot, reference.mean)
			noise = convergence.accumulate(frame, w, h, variance_frames, animate=True) if variance_frames >= 2 else None
		finally:
			frame.close()
		member = dict(name=name, settings=dict(experiment["settings"]), samples_per_pixel=experiment["settings"]["sample_count"],
			mse=error["mse"], rel_mse=error["rel_mse"], mae=error["mae"], max_abs_error=error["max_abs_error"], nonfinite_pixels=error["nonfinite_pixels"],
			mean_variance=list(noise.mean_variance) if noise is not None else None)
		record["members"].append(member)
	return record


def run_convergences(groups, data_root, out_dir, json_path, reference_frames, variance_frames, **kw):
	"""Runs the groups in order and writes their records as JSON (a list, see run_convergence)."""
	records = []
	for group in groups:
		record = run_convergence(group, data_root, out_dir, reference_frames, variance_frames, **kw)
		records.append(record)
		print("%s against %s (%d frames, %dx%d; accumulate %.4f ms per frame)" % (group["name"], group["reference"], reference_frames, record["width"], record["height"],
			record["accumulate_ms_per_frame"]), flush=True)
		if "adaptive" in record:
			a = record["adaptive"]
			print("  adaptive reference, target relMSE %g: %d of %d tile-frames shaded (%.3f), estimated relMSE %.4e, shading %.1f ms, %.2f s" % (a["target_rel_mse"],
				a["tile_frames_shaded"], a["tile_frames_full"], a["shaded_fraction"], sum(a["estimated_rel_mse"]) / 3.0, a["shade_ms"], a["wall_s"]), flush=True)
		e = record["reference_frame_error"]
		print("  %-70s relMSE %.4e  MSE %.4e" % ("(one frame of the reference's settings)", sum(e["rel_mse"]) / 3.0, sum(e["mse"]) / 3.0), flush=True)
		for m in sorted(record["members"], key=lambda m: sum(m["rel_mse"])):
			print("  %-70s relMSE %.4e  MSE %.4e  mean variance %s" % (m["name"], sum(m["rel_mse"]) / 3.0, sum(m["mse"]) / 3.0,
				"%.4e" % (sum(m["mean_variance"]) / 3.0) if m["mean_variance"] else "-"), flush=True)
	os.makedirs(os.path.dirname(os.path.abspath(json_path)), exist_ok=True)
	with open(json_path, "w") as f:
		json.dump(records, f, indent=1)
	return records
