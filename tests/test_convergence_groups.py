"""The convergence groups of the experiment list (experiments.convergence_groups): every member is measured against a reference that renders the
same picture -- same scene, scene parameters, quicksave, resolution, exposure and light display -- and no error display is a member. Host side only;
the measurement itself needs a GPU (tests/test_gpu_zzzzzz_convergence.py)."""
from vulkan_renderer_b200 import experiments as E

SAME_PICTURE = ("scene", "scene_parameters", "quick_save_path", "width", "height", "light_count")


def test_every_member_shares_the_view_of_its_reference():
	by_name = {e["name"]: e for e in E.experiment_list()}
	groups = E.convergence_groups()
	assert len({g["name"] for g in groups}) == len(groups)
	members = [m for g in groups for m in g["members"]]
	assert len(set(members)) == len(members)
	for g in groups:
		ref = by_name[g["reference"]]
		assert g["members"] and g["reference"] not in g["members"]
		for name in g["members"]:
			e = by_name[name]
			for key in SAME_PICTURE:
				assert e[key] == ref[key], (name, key)
			for key in ("exposure_factor", "show_polygonal_lights"):
				assert e["settings"][key] == ref["settings"][key], (name, key)
			assert "error_display" not in e["settings"] and not name.startswith("error_")


def test_the_groups_the_figures_need():
	groups = {g["name"]: g for g in E.convergence_groups()}
	assert groups["shadowed_plane"] == dict(name="shadowed_plane", reference="shadowed_plane_reference_4096spp", members=["shadowed_plane_biased_4096spp"])
	assert groups["roughness_planes"]["members"] == ["roughness_planes_lambertian_diffuse_only_1spp"] and groups["roughness_planes"]["reference"] == "roughness_planes_lambertian_2spp"
	assert groups["cornell_box_tilted"]["members"] == ["cornell_box_projected_solid_angle_arvo_tilted_1spp"]
	assert groups["cornell_box"]["members"] == ["cornell_box_%s_1spp" % label for label in E.SAMPLE_POLYGON_NAME]
	assert len(groups["attic"]["members"]) == 4 and all(m.endswith("_2spp") for m in groups["attic"]["members"])
	assert len(groups["bistro_small"]["members"]) == len(groups["bistro_tiny"]["members"]) == 11
	assert len(groups["mis_plane"]["members"]) == 7 and groups["mis_plane"]["reference"] == "mis_plane_reference_128spp"
	grouped = {g["reference"] for g in groups.values()} | {m for g in groups.values() for m in g["members"]}
	left_out = [e["name"] for e in E.experiment_list(all_timings=False) if e["name"] not in grouped]
	assert sorted(left_out) == ["error_attic_backward", "error_attic_backward_times_psa", "ies_profile_attic_2spp", "roughness_planes_screen_2spp"]
