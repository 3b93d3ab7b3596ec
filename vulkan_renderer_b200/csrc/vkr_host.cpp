// vkr_host.cpp -- host side of libvkr_b200.so above the CUDA kernels: device, loaders for the
// reference's file formats (*.vks, *.vkt, fit*.dat, noise, *.save), camera / light math and the
// per-frame constant block. Each function names the reference code whose observable behaviour it
// reproduces; the code itself is written from the file formats and the maths, not from that source.
#include "../../include/vkr_b200.h"
#include "vkr_bvh.h"
#include "vkr_internal.h"
#include <cuda_runtime.h>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

using namespace vkr;

#define VKR_CUDA_OK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { printf("%s: %s\n", what, cudaGetErrorString(e_)); return 1; } } while (0)

extern "C" uint32_t vkr_abi_version(void) { return VKR_B200_ABI_VERSION; }

// ------------------------------------------------------------------------------------------------
// device
// ------------------------------------------------------------------------------------------------
extern "C" int vkr_create_device(vkr_device_t* device, int cuda_device, void* stream) {
	memset(device, 0, sizeof(*device));
	int count = 0;
	if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
		printf("Failed to create a device: no CUDA device is visible. This library has no CPU fallback.\n");
		return 1;
	}
	if (cuda_device < 0 || cuda_device >= count) {
		printf("Failed to create a device: CUDA device %d does not exist (%d visible).\n", cuda_device, count);
		return 1;
	}
	VKR_CUDA_OK(cudaSetDevice(cuda_device), "Failed to select the CUDA device");
	cudaDeviceProp prop;
	VKR_CUDA_OK(cudaGetDeviceProperties(&prop, cuda_device), "Failed to query device properties");
	device->cuda_device = cuda_device;
	device->sm_count = prop.multiProcessorCount;
	device->ray_tracing_supported = 1;
	snprintf(device->name, sizeof(device->name), "%s", prop.name);
	if (stream) { device->stream = stream; device->owns_stream = 0; }
	else {
		cudaStream_t s;
		if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) {
			printf("Failed to create a CUDA stream.\n");
			memset(device, 0, sizeof(*device));
			return 1;
		}
		device->stream = (void*) s; device->owns_stream = 1;
	}
	return 0;
}

extern "C" void vkr_destroy_device(vkr_device_t* device) {
	if (device->owns_stream && device->stream) cudaStreamDestroy((cudaStream_t) device->stream);
	memset(device, 0, sizeof(*device));
}

extern "C" int vkr_device_wait_idle(const vkr_device_t* device) {
	VKR_CUDA_OK(cudaStreamSynchronize((cudaStream_t) device->stream), "Failed to wait for the device");
	return 0;
}

namespace vkr {
int upload(void** d_ptr, const void* src, size_t bytes, const vkr_device_t* device) {
	*d_ptr = nullptr;
	if (!device) return 0; // host-only load (parity tests of the loaders on machines without a GPU)
	if (cudaSetDevice(device->cuda_device) != cudaSuccess) return 1;
	if (cudaMalloc(d_ptr, bytes ? bytes : 16) != cudaSuccess) { *d_ptr = nullptr; return 1; }
	if (bytes && cudaMemcpy(*d_ptr, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(*d_ptr); *d_ptr = nullptr; return 1; }
	return 0;
}
}

// ------------------------------------------------------------------------------------------------
// scene (*.vks reader: src/scene.c:419-483; acceleration structure input: src/scene.c:175-187)
// ------------------------------------------------------------------------------------------------
extern "C" void vkr_destroy_scene(vkr_scene_t* scene, const vkr_device_t* device) {
	(void) device;
	if (scene->material_names) {
		for (uint64_t i = 0; i != scene->material_count; ++i) free(scene->material_names[i]);
		free(scene->material_names);
	}
	free(scene->material_params);
	void* dev_ptrs[] = { scene->d_quantized_positions, scene->d_normals_and_tex_coords, scene->d_material_indices, scene->d_material_params,
		scene->d_shadow_nodes, scene->d_shadow_tris, scene->d_primary_nodes, scene->d_primary_tris, scene->d_primary_tri_ids,
		scene->d_texture_data, scene->d_texture_dims, scene->d_texture_offsets, scene->d_shadow_nodes_interleaved };
	for (void* p : dev_ptrs) if (p) cudaFree(p);
	memset(scene, 0, sizeof(*scene));
}

static void unpack_position(const uint32_t q[2], float p[3]) { // bit layout: src/scene.h:56-62
	p[0] = (float) (q[0] & 0x1FFFFFu);
	p[1] = (float) (((q[0] & 0xFFE00000u) >> 21) | ((q[1] & 0x3FFu) << 11));
	p[2] = (float) ((q[1] & 0x7FFFFC00u) >> 10);
}

// Everything of load_scene() that follows the file: device copies of the three mesh buffers, acceleration structures, materials. Shared by vkr_load_scene
// (the library's own *.vks reader) and vkr_scene_from_buffers (boundary B1: the reference's unchanged load_scene() ran against shim/ and hands its buffers over).
// as_vertices: the triangle soup of the acceleration structure build (scene.c:175-209) or NULL (dequantised here the same way); given_textures: 3 per
// material, decoded (vkr_texture_t), or NULL to read <texture_path>/<material>_{BaseColor,Specular,Normal}.vkt.
static int scene_from_arrays(vkr_scene_t* scene, const vkr_device_t* device, const uint32_t* positions, const uint16_t* normals_uvs, const uint8_t* material_indices,
	const float* as_vertices, const vkr_texture_t* given_textures, const char* file_path, const char* texture_path, int request_acceleration_structure)
{
	const uint64_t n = scene->triangle_count;
	if (upload(&scene->d_quantized_positions, positions, (size_t) n * 3 * 2 * 4, device)
		|| upload(&scene->d_normals_and_tex_coords, normals_uvs, (size_t) n * 3 * 4 * 2, device)
		|| upload(&scene->d_material_indices, material_indices, (size_t) n, device))
	{
		printf("Failed to create device buffers and allocate memory for meshes of the scene file at path %s. It has %llu triangles.\n", file_path, (unsigned long long) n);
		vkr_destroy_scene(scene, device); return 1;
	}
	// Acceleration structures
	const auto t0 = std::chrono::steady_clock::now();
	if (request_acceleration_structure && device && device->ray_tracing_supported) {
		std::vector<float> soup(9 * n);
		host_bvh bvh;
		// (a) shadow rays: the float soup of scene.c:175-187 (multiply, then add)
		if (as_vertices) memcpy(soup.data(), as_vertices, sizeof(float) * 9 * n); // what the reference hands to vkCmdBuildAccelerationStructuresKHR
		else for (uint64_t i = 0; i != 3 * n; ++i) {
			float p[3]; unpack_position(&positions[2 * i], p);
			for (int j = 0; j != 3; ++j) soup[3 * i + j] = p[j] * scene->dequantization_factor[j] + scene->dequantization_summand[j];
		}
		// Builder: binned SAH on the host by default; VKR_BVH_BUILDER=lbvh / lbvh_gpu select the linear BVH (host reference / GPU). Whatever the
		// linear builders cannot deliver (too deep a tree for the traversal stack, fewer than five triangles, a CUDA error) is built by the default one.
		const bvh_builder which = bvh_builder_from_environment();
		bool built_on_device = false;
		if (which == bvh_builder_lbvh_gpu && cudaSetDevice(device->cuda_device) == cudaSuccess) {
			void* d_ids = nullptr; uint64_t pairs = 0; uint32_t depth = 0;
			if (build_lbvh_device(soup.data(), n, device->stream, &scene->d_shadow_nodes, &scene->d_shadow_tris, &d_ids, &pairs, &depth) == 0) {
				cudaFree(d_ids);
				if (depth < 62) { built_on_device = true; scene->shadow_node_count = pairs; scene->shadow_max_depth = depth; scene->shadow_bvh_width = 2; }
				else { cudaFree(scene->d_shadow_nodes); cudaFree(scene->d_shadow_tris); scene->d_shadow_nodes = scene->d_shadow_tris = nullptr; }
			}
			if (!built_on_device) printf("The GPU BVH builder did not produce a usable tree for %s; building on the host instead.\n", file_path);
		}
		if (!built_on_device) {
			scene->shadow_bvh_width = 2;
			if (which == bvh_builder_lbvh) build_lbvh(bvh, soup.data(), n);
			if (which != bvh_builder_lbvh || bvh.max_depth >= 62) build_bvh(bvh, soup.data(), n);
			scene->shadow_node_count = bvh.node_count; scene->shadow_max_depth = bvh.max_depth;
			if (bvh.max_depth >= 62 || upload(&scene->d_shadow_nodes, bvh.nodes.data(), bvh.nodes.size() * 4, device) || upload(&scene->d_shadow_tris, bvh.tris.data(), bvh.tris.size() * 4, device)) {
				printf("Failed to construct an acceleration structure for the scene file at path %s.\n", file_path);
				vkr_destroy_scene(scene, device); return 1;
			}
		}
		// the form the trace warps walk: the two children's numbers side by side (vkr_trace.cuh)
		if (interleave_node_pairs_device(scene->d_shadow_nodes, scene->shadow_node_count, &scene->d_shadow_nodes_interleaved, device->stream)) {
			printf("Failed to interleave the acceleration structure for the scene file at path %s.\n", file_path);
			vkr_destroy_scene(scene, device); return 1;
		}
		// (b) primary rays: vertices as the shaders decode them (fma, mesh_quantization.glsl:38-45)
		for (uint64_t i = 0; i != 3 * n; ++i) {
			float p[3]; unpack_position(&positions[2 * i], p);
			for (int j = 0; j != 3; ++j) soup[3 * i + j] = fmaf(p[j], scene->dequantization_factor[j], scene->dequantization_summand[j]);
		}
		build_bvh(bvh, soup.data(), n);
		scene->primary_node_count = bvh.node_count; scene->primary_max_depth = bvh.max_depth;
		if (bvh.max_depth >= 62 || upload(&scene->d_primary_nodes, bvh.nodes.data(), bvh.nodes.size() * 4, device) || upload(&scene->d_primary_tris, bvh.tris.data(), bvh.tris.size() * 4, device)
			|| upload(&scene->d_primary_tri_ids, bvh.tri_ids.data(), bvh.tri_ids.size() * 4, device)) {
			printf("Failed to construct an acceleration structure for the scene file at path %s.\n", file_path);
			vkr_destroy_scene(scene, device); return 1;
		}
	}
	scene->build_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
	// Materials: <texture_path>/<material>_{BaseColor,Specular,Normal}.vkt (scene.c:24-31, 529-533), every mip level decoded to RGBA32F (vkr_textures.cpp).
	// material_params holds the first texel of the smallest mip level (the texture average): all there is to a constant texture. If any texture is
	// not constant, the chains go to the device and the G-buffer producer filters them (vkr_texture.cuh).
	scene->material_params = (float*) calloc(8 * (scene->material_count ? scene->material_count : 1), sizeof(float));
	static const char* suffixes[3] = { "BaseColor", "Specular", "Normal" };
	std::vector<vkr_texture_t> textures(3 * (size_t) scene->material_count);
	bool failed = false, any_pattern = false;
	const bool own_textures = given_textures == nullptr;
	for (uint64_t i = 0; i != scene->material_count && !failed; ++i) {
		float tex[3][4];
		for (int j = 0; j != 3 && !failed; ++j) {
			vkr_texture_t& t = textures[3 * i + j];
			if (own_textures) {
				const std::string path = std::string(texture_path) + "/" + scene->material_names[i] + "_" + suffixes[j] + ".vkt";
				failed = vkr_load_texture(&t, path.c_str()) != 0;
			}
			else { t = given_textures[3 * i + j]; failed = !t.h_texels || !t.mip_count; }
			if (failed) break;
			any_pattern = any_pattern || !t.is_constant;
			const uint32_t last = t.mip_count - 1;
			const uint64_t last_texels = (uint64_t) ((t.width >> last) ? (t.width >> last) : 1) * ((t.height >> last) ? (t.height >> last) : 1);
			memcpy(tex[j], t.h_texels + (t.texel_float_count - 4 * last_texels), sizeof(tex[j]));
		}
		if (failed) break;
		float* mp = scene->material_params + 8 * i;
		mp[0] = tex[0][0]; mp[1] = tex[0][1]; mp[2] = tex[0][2];
		mp[3] = tex[1][1]; mp[4] = tex[1][2];
		mp[5] = tex[2][0]; mp[6] = tex[2][1]; mp[7] = 0.0f;
	}
	if (!failed) failed = upload(&scene->d_material_params, scene->material_params, sizeof(float) * 8 * scene->material_count, device) != 0;
	if (!failed && device && any_pattern) {
		std::vector<uint32_t> dims(4 * textures.size()); std::vector<uint64_t> offsets(textures.size());
		uint64_t texel_count = 0;
		for (size_t k = 0; k != textures.size(); ++k) {
			dims[4 * k] = textures[k].width; dims[4 * k + 1] = textures[k].height; dims[4 * k + 2] = textures[k].mip_count; dims[4 * k + 3] = 0;
			offsets[k] = texel_count; texel_count += textures[k].texel_float_count / 4;
		}
		std::vector<float> data(4 * (size_t) texel_count);
		for (size_t k = 0; k != textures.size(); ++k) memcpy(&data[4 * (size_t) offsets[k]], textures[k].h_texels, sizeof(float) * (size_t) textures[k].texel_float_count);
		failed = upload(&scene->d_texture_data, data.data(), data.size() * 4, device) || upload(&scene->d_texture_dims, dims.data(), dims.size() * 4, device)
			|| upload(&scene->d_texture_offsets, offsets.data(), offsets.size() * 8, device);
		scene->textured = 1; scene->texture_texel_count = texel_count;
	}
	if (own_textures) for (vkr_texture_t& t : textures) vkr_destroy_texture(&t);
	if (failed) {
		printf("Failed to load material textures for the scene file at path %s using texture path %s.\n", file_path, texture_path ? texture_path : "(textures handed over)");
		vkr_destroy_scene(scene, device); return 1;
	}
	return 0;
}


extern "C" int vkr_scene_from_buffers(vkr_scene_t* scene, const vkr_device_t* device, const vkr_scene_buffers_t* b, int request_acceleration_structure) {
	memset(scene, 0, sizeof(*scene));
	if (!b->triangle_count || b->triangle_count >= (1ull << 27) || b->material_count > 256 || !b->quantized_positions || !b->normals_and_tex_coords || !b->material_indices
		|| (!b->material_textures && !b->texture_path) || (!b->material_names && !b->material_textures))
	{
		printf("Failed to take over a scene: %llu triangles, %llu materials, or buffers are missing.\n", (unsigned long long) b->triangle_count, (unsigned long long) b->material_count);
		return 1;
	}
	scene->triangle_count = b->triangle_count; scene->material_count = b->material_count;
	memcpy(scene->dequantization_factor, b->dequantization_factor, 12); memcpy(scene->dequantization_summand, b->dequantization_summand, 12);
	scene->material_names = (char**) calloc(scene->material_count ? scene->material_count : 1, sizeof(char*));
	for (uint64_t i = 0; i != scene->material_count; ++i) {
		const char* name = (b->material_names && b->material_names[i]) ? b->material_names[i] : "";
		scene->material_names[i] = (char*) malloc(strlen(name) + 1);
		strcpy(scene->material_names[i], name);
	}
	for (uint64_t i = 0; i != b->triangle_count; ++i)
		if (b->material_indices[i] >= scene->material_count) {
			printf("The scene refers to material %u but has %llu materials only.\n", (unsigned) b->material_indices[i], (unsigned long long) scene->material_count);
			vkr_destroy_scene(scene, device); return 1;
		}
	return scene_from_arrays(scene, device, b->quantized_positions, b->normals_and_tex_coords, b->material_indices, b->acceleration_structure_vertices, b->material_textures,
		"(buffers handed over)", b->texture_path, request_acceleration_structure);
}

extern "C" int vkr_load_scene(vkr_scene_t* scene, const vkr_device_t* device, const char* file_path, const char* texture_path, int request_acceleration_structure) {
	memset(scene, 0, sizeof(*scene));
	FILE* file = fopen(file_path, "rb");
	if (!file) { printf("Failed to open the scene file at %s.\n", file_path); return 1; }
	uint32_t file_marker = 0, version = 0;
	fread(&file_marker, 4, 1, file); fread(&version, 4, 1, file);
	if (file_marker != 0xabcabc || version != 1) {
		printf("The scene file at path %s is invalid or unsupported. The format marker is 0x%x, the version is %d.\n", file_path, file_marker, version);
		fclose(file); return 1;
	}
	fread(&scene->material_count, 8, 1, file);
	fread(&scene->triangle_count, 8, 1, file);
	fread(scene->dequantization_factor, 4, 3, file);
	fread(scene->dequantization_summand, 4, 3, file);
	printf("Triangle count: %llu\n", (unsigned long long) scene->triangle_count);
	if (scene->triangle_count == 0) {
		printf("The scene file at path %s is completely empty, i.e. it holds 0 triangles.\n", file_path);
		fclose(file); memset(scene, 0, sizeof(*scene)); return 1;
	}
	if (scene->triangle_count >= (1ull << 27) || scene->material_count > 256) {
		printf("The scene file at path %s is too large for this library (%llu triangles, %llu materials).\n", file_path, (unsigned long long) scene->triangle_count, (unsigned long long) scene->material_count);
		fclose(file); memset(scene, 0, sizeof(*scene)); return 1;
	}
	scene->material_names = (char**) calloc(scene->material_count ? scene->material_count : 1, sizeof(char*));
	for (uint64_t i = 0; i != scene->material_count; ++i) {
		uint64_t name_length = 0;
		fread(&name_length, 8, 1, file);
		if (name_length > 4096) { printf("The scene file at path %s has a corrupt material table.\n", file_path); fclose(file); vkr_destroy_scene(scene, device); return 1; }
		scene->material_names[i] = (char*) malloc(name_length + 1);
		fread(scene->material_names[i], 1, name_length + 1, file);
		scene->material_names[i][name_length] = 0;
	}
	const uint64_t n = scene->triangle_count;
	std::vector<uint32_t> positions(2 * 3 * n);
	std::vector<uint16_t> normals_uvs(4 * 3 * n);
	std::vector<uint8_t> material_indices(n);
	fread(positions.data(), 4, positions.size(), file);
	fread(normals_uvs.data(), 2, normals_uvs.size(), file);
	fread(material_indices.data(), 1, material_indices.size(), file);
	uint32_t eof_marker = 0;
	fread(&eof_marker, 4, 1, file);
	fclose(file);
	if (eof_marker != 0xE0FE0F) {
		printf("The scene file at path %s seems to be invalid. The geometry data is not followed by the expected end of file marker.\n", file_path);
		vkr_destroy_scene(scene, device); return 1;
	}
	for (uint64_t i = 0; i != n; ++i) // the G-buffer pass indexes the material table with these on the device
		if (material_indices[i] >= scene->material_count) {
			printf("The scene file at path %s refers to material %u but has %llu materials only.\n", file_path, (unsigned) material_indices[i], (unsigned long long) scene->material_count);
			vkr_destroy_scene(scene, device); return 1;
		}
	return scene_from_arrays(scene, device, positions.data(), normals_uvs.data(), material_indices.data(), nullptr, nullptr, file_path, texture_path, request_acceleration_structure);
}

// ------------------------------------------------------------------------------------------------
// LTC table (fit<i>.dat reader + quantisation: src/ltc_table.c:23-116; constants :184-191)
// ------------------------------------------------------------------------------------------------
extern "C" void vkr_destroy_ltc_table(vkr_ltc_table_t* table, const vkr_device_t* device) {
	(void) device;
	if (table->d_table0) cudaFree(table->d_table0);
	if (table->d_table1) cudaFree(table->d_table1);
	free(table->h_table0); free(table->h_table1);
	memset(table, 0, sizeof(*table));
}

extern "C" int vkr_load_ltc_table(vkr_ltc_table_t* table, const vkr_device_t* device, const char* directory, uint32_t fresnel_count) {
	memset(table, 0, sizeof(*table));
	table->fresnel_count = fresnel_count;
	size_t slice0 = 0, slice1 = 0;
	for (uint32_t i = 0; i != fresnel_count; ++i) {
		const std::string path = std::string(directory) + "/fit" + std::to_string(i) + ".dat";
		FILE* file = fopen(path.c_str(), "rb");
		if (!file) { printf("Failed to open the linearly transformed cosine table at %s.\n", path.c_str()); vkr_destroy_ltc_table(table, device); return 1; }
		uint64_t resolution = 0;
		fread(&resolution, 8, 1, file);
		if (table->roughness_count == 0) {
			if (resolution == 0 || resolution > 4096) { printf("The linearly transformed cosine table at %s has an invalid resolution.\n", path.c_str()); fclose(file); vkr_destroy_ltc_table(table, device); return 1; }
			table->roughness_count = table->inclination_count = (uint32_t) resolution;
			slice0 = (size_t) resolution * resolution * 4; slice1 = (size_t) resolution * resolution * 2;
			table->h_table0 = (uint16_t*) calloc(slice0 * fresnel_count, 2);
			table->h_table1 = (uint16_t*) calloc(slice1 * fresnel_count, 2);
		}
		else if (resolution != table->roughness_count) {
			printf("The linearly transformed cosine tables in directory %s have inconsistent resolutions.\n", directory);
			fclose(file); vkr_destroy_ltc_table(table, device); return 1;
		}
		for (uint64_t j = 0; j != resolution * resolution; ++j) {
			float m[5] = {0, 0, 0, 0, 0};
			fread(m, 4, 5, file);
			// m = {m00, m02, m11, m20, albedo} of [[m00,0,m02],[0,m11,0],[m20,0,1]]; adjugate up to a factor:
			float inv[5] = { m[2], -m[1] * m[2], m[0] - m[1] * m[3], -m[2] * m[3], m[0] * m[2] }; // inv00, inv02, inv11, inv20, inv22
			float max_magnitude = fabsf(inv[0]);
			for (int k = 1; k != 5; ++k) if (max_magnitude < fabsf(inv[k])) max_magnitude = fabsf(inv[k]);
			for (int k = 0; k != 5; ++k) inv[k] /= max_magnitude;
			const float entries[6] = { inv[0], -inv[1], inv[2], inv[3], inv[4], m[4] };
			for (int k = 0; k != 6; ++k) {
				float e = entries[k];
				if (e < 0.0f) e = 0.0f;
				if (e > 1.0f) e = 1.0f;
				const uint16_t q = (uint16_t) (e * 65535.0f + 0.5f);
				if (k < 4) table->h_table0[slice0 * i + 4 * j + k] = q;
				else table->h_table1[slice1 * i + 2 * j + (k - 4)] = q;
			}
		}
		fclose(file);
	}
	if (upload(&table->d_table0, table->h_table0, slice0 * fresnel_count * 2, device) || upload(&table->d_table1, table->h_table1, slice1 * fresnel_count * 2, device)) {
		printf("Failed to create device local textures for LTC tables.");
		vkr_destroy_ltc_table(table, device); return 1;
	}
	const float pi = 3.1415926535897932384626433832795f;
	table->constants.fresnel_index_factor = (float) (table->fresnel_count - 1);
	table->constants.fresnel_index_summand = 0.0f;
	table->constants.roughness_factor = (float) (table->roughness_count - 1) / (float) table->roughness_count;
	table->constants.roughness_summand = 0.5f / (float) table->roughness_count;
	table->constants.inclination_factor = (float) (table->inclination_count - 1) / (0.5f * pi * table->inclination_count);
	table->constants.inclination_summand = 0.5f / (float) table->inclination_count;
	return 0;
}

// Boundary B1: the two texture arrays as the reference's load_ltc_table() uploads them (ltc_table.c:86-141: RGBA16_UNORM and RG16_UNORM, fresnel-major)
extern "C" int vkr_ltc_table_from_images(vkr_ltc_table_t* table, const vkr_device_t* device, uint32_t roughness_count, uint32_t inclination_count, uint32_t fresnel_count,
	const uint16_t* table0_rgba16, const uint16_t* table1_rg16, const vkr_ltc_constants_t* constants)
{
	memset(table, 0, sizeof(*table));
	if (!roughness_count || roughness_count != inclination_count || !fresnel_count || !table0_rgba16 || !table1_rg16 || !constants) {
		printf("Failed to take over a linearly transformed cosine table of resolution %ux%u with %u slices.\n", roughness_count, inclination_count, fresnel_count);
		return 1;
	}
	table->roughness_count = roughness_count; table->inclination_count = inclination_count; table->fresnel_count = fresnel_count;
	const size_t n0 = (size_t) roughness_count * inclination_count * 4 * fresnel_count, n1 = n0 / 2;
	table->h_table0 = (uint16_t*) malloc(2 * n0); table->h_table1 = (uint16_t*) malloc(2 * n1);
	memcpy(table->h_table0, table0_rgba16, 2 * n0); memcpy(table->h_table1, table1_rg16, 2 * n1);
	table->constants = *constants;
	if (upload(&table->d_table0, table->h_table0, 2 * n0, device) || upload(&table->d_table1, table->h_table1, 2 * n1, device)) {
		printf("Failed to create device local textures for LTC tables.");
		vkr_destroy_ltc_table(table, device); return 1;
	}
	return 0;
}

// ------------------------------------------------------------------------------------------------
// noise table (src/noise_table.c:46-168)
// ------------------------------------------------------------------------------------------------
static uint32_t wang_hash(uint32_t seed) { // Wang's integer hash, as used by the reference (math_utilities.h:50-57)
	seed = (seed ^ 61u) ^ (seed >> 16);
	seed *= 9u;
	seed ^= seed >> 4;
	seed *= 0x27d4eb2du;
	seed ^= seed >> 15;
	return seed;
}

extern "C" void vkr_destroy_noise_table(vkr_noise_table_t* noise, const vkr_device_t* device) {
	(void) device;
	if (noise->d_noise) cudaFree(noise->d_noise);
	free(noise->h_noise);
	memset(noise, 0, sizeof(*noise));
}

extern "C" int vkr_load_noise_table(vkr_noise_table_t* noise, const vkr_device_t* device, uint32_t width, uint32_t height, uint32_t layers, vkr_noise_type_t noise_type) {
	memset(noise, 0, sizeof(*noise));
	noise->random_seed = 3124705;
	if (width > 9999 || height > 9999 || layers > 9999 || !width || !height || !layers || (width & (width - 1)) || (height & (height - 1)) || (layers & (layers - 1))) {
		printf("Invalid noise resolution or slice count.\n");
		return 1;
	}
	const uint32_t cell_count = width * height * layers * 4;
	noise->h_noise = (uint16_t*) malloc(sizeof(uint16_t) * cell_count);
	if (noise_type == vkr_noise_type_white) {
		for (uint32_t i = 0; i != cell_count; ++i) noise->h_noise[i] = (uint16_t) (wang_hash(i + 243708u) & 0xFFFFu);
	}
	else {
		const char* pattern = (noise_type == vkr_noise_type_blue) ? "data/noise/blue_noise_rgba_%02dx%02d_%02d.blob" : (noise_type == vkr_noise_type_ahmed) ? "data/noise/ahmed_2d_rgba_%02dx%02d_%02d.blob" : nullptr;
		if (!pattern) { printf("Failed to load a noise table. The given type is unknown.\n"); vkr_destroy_noise_table(noise, device); return 1; }
		char path[256];
		snprintf(path, sizeof(path), pattern, width, height, layers);
		FILE* file = fopen(path, "rb");
		if (!file) { printf("Failed to open the noise file at path %s. Please check path and permissions?\n", path); vkr_destroy_noise_table(noise, device); return 1; }
		fread(noise->h_noise, 2, cell_count, file);
		fclose(file);
	}
	noise->width = width; noise->height = height; noise->layers = layers;
	if (upload(&noise->d_noise, noise->h_noise, sizeof(uint16_t) * cell_count, device)) {
		printf("Failed to create a noise texture of resolution %ux%u with %u layers.\n", width, height, layers);
		vkr_destroy_noise_table(noise, device); return 1;
	}
	return 0;
}

// Boundary B1: the texture array as the reference's load_noise_table() uploads it (noise_table.c:105-160: RGBA16_UNORM, layer-major)
extern "C" int vkr_noise_table_from_image(vkr_noise_table_t* noise, const vkr_device_t* device, uint32_t width, uint32_t height, uint32_t layers, const uint16_t* texels_rgba16, uint32_t random_seed) {
	memset(noise, 0, sizeof(*noise));
	if (!width || !height || !layers || (width & (width - 1)) || (height & (height - 1)) || (layers & (layers - 1)) || !texels_rgba16) {
		printf("Invalid noise resolution or slice count.\n");
		return 1;
	}
	const size_t cell_count = (size_t) width * height * layers * 4;
	noise->h_noise = (uint16_t*) malloc(sizeof(uint16_t) * cell_count);
	memcpy(noise->h_noise, texels_rgba16, sizeof(uint16_t) * cell_count);
	noise->width = width; noise->height = height; noise->layers = layers; noise->random_seed = random_seed;
	if (upload(&noise->d_noise, noise->h_noise, sizeof(uint16_t) * cell_count, device)) {
		printf("Failed to create a noise texture of resolution %ux%u with %u layers.\n", width, height, layers);
		vkr_destroy_noise_table(noise, device); return 1;
	}
	return 0;
}

extern "C" void vkr_set_noise_constants(uint32_t resolution_mask[2], uint32_t* texture_index_mask, uint32_t random_numbers[4], vkr_noise_table_t* noise, int animate_noise) {
	resolution_mask[0] = noise->width - 1;
	resolution_mask[1] = noise->height - 1;
	*texture_index_mask = noise->layers - 1;
	for (uint32_t i = 0; i != 4; ++i) random_numbers[i] = animate_noise ? wang_hash(noise->random_seed * 4 + i) : (i * 0x123456u);
	if (animate_noise) ++noise->random_seed;
}

// ------------------------------------------------------------------------------------------------
// lights (src/polygonal_light.c:24-126) and camera (src/camera.c:24-83).
// Host floating point is compiled with -ffp-contract=off and without -mfma: products and sums
// round separately, like the reference's plain C on x86-64.
// ------------------------------------------------------------------------------------------------
extern "C" void vkr_set_polygonal_light_vertex_count(vkr_polygonal_light_t* light, uint32_t n) {
	if (n == light->vertex_count && light->vertices_plane_space && light->vertices_world_space && light->fan_areas) return;
	float* plane = (float*) calloc(4 * (size_t) n, sizeof(float));
	if (light->vertices_plane_space) memcpy(plane, light->vertices_plane_space, sizeof(float) * 4 * (n < light->vertex_count ? n : light->vertex_count));
	free(light->vertices_plane_space); light->vertices_plane_space = plane;
	free(light->vertices_world_space); light->vertices_world_space = (float*) calloc(4 * (size_t) n, sizeof(float));
	free(light->fan_areas); light->fan_areas = (float*) calloc(4 * (size_t) (n > 2 ? n - 2 : 1), sizeof(float));
	light->vertex_count = n;
}

extern "C" void vkr_destroy_polygonal_light(vkr_polygonal_light_t* light) {
	free(light->vertices_plane_space); free(light->vertices_world_space); free(light->fan_areas); free(light->texture_file_path);
	memset(light, 0, sizeof(*light));
}

extern "C" void vkr_update_polygonal_light(vkr_polygonal_light_t* light) {
	const float pi = 3.1415926535897932384626433832795f;
	light->inv_scaling_x = 1.0f / light->scaling_x;
	light->inv_scaling_y = 1.0f / light->scaling_y;
	// Rotation from Euler angles, R = Rx * Ry * Rz in the reference's convention
	const float cx = cosf(light->rotation_angles[0]), sx = sinf(light->rotation_angles[0]);
	const float cy = cosf(light->rotation_angles[1]), sy = sinf(light->rotation_angles[1]);
	const float cz = cosf(light->rotation_angles[2]), sz = sinf(light->rotation_angles[2]);
	const float cxsy = cx * sy, sxsy = sx * sy;
	const float rotation[3][4] = {
		{ cy * cz, -cy * sz, -sy, 0.0f },
		{ -sxsy * cz + cx * sz, sxsy * sz + cx * cz, -sx * cy, 0.0f },
		{ cxsy * cz + sx * sz, -cxsy * sz + sx * cz, cx * cy, 0.0f },
	};
	memcpy(light->rotation, rotation, sizeof(rotation));
	const float scalings[2] = { light->scaling_x, light->scaling_y };
	for (uint32_t i = 0; i != light->vertex_count; ++i)
		for (uint32_t j = 0; j != 3; ++j) {
			float w = light->translation[j];
			for (uint32_t k = 0; k != 2; ++k) w += scalings[k] * rotation[j][k] * light->vertices_plane_space[i * 4 + k];
			light->vertices_world_space[i * 4 + j] = w;
		}
	light->plane[0] = rotation[0][2]; light->plane[1] = rotation[1][2]; light->plane[2] = rotation[2][2];
	light->plane[3] = -(rotation[0][2] * light->translation[0] + rotation[1][2] * light->translation[1] + rotation[2][2] * light->translation[2]);
	float signed_area = 0.0f;
	const float* vp = light->vertices_plane_space;
	for (uint32_t i = 0; i + 2 < light->vertex_count; ++i) {
		const float m00 = vp[(i + 2) * 4 + 0] - vp[0], m01 = vp[(i + 1) * 4 + 0] - vp[0];
		const float m10 = vp[(i + 2) * 4 + 1] - vp[1], m11 = vp[(i + 1) * 4 + 1] - vp[1];
		const float triangle_area = 0.5f * (m00 * m11 - m01 * m10);
		signed_area += triangle_area;
		const float flip = (triangle_area < 0.0f) ? -1.0f : 1.0f;
		light->fan_areas[4 * i + 0] = scalings[0] * scalings[1] * triangle_area * flip;
		light->fan_areas[4 * i + 1] = scalings[0] * scalings[1] * signed_area * flip;
	}
	signed_area *= scalings[0] * scalings[1];
	const float abs_area = (signed_area < 0.0f) ? -signed_area : signed_area;
	light->area = abs_area;
	light->rcp_area = 1.0f / abs_area;
	const float flux_factor = 1.0f / (abs_area * pi);
	for (uint32_t i = 0; i != 3; ++i) light->surface_radiance[i] = light->radiant_flux[i] * flux_factor;
	for (uint32_t i = 0; i != 4; ++i) light->plane[i] = (signed_area > 0.0f) ? light->plane[i] : (-light->plane[i]);
}

static void world_to_view_space(float out[4][4], const vkr_first_person_camera_t* camera) {
	const float cos_x = cosf(camera->rotation_x), sin_x = sinf(camera->rotation_x);
	const float cos_z = cosf(camera->rotation_z), sin_z = sinf(camera->rotation_z);
	const float rx[3][3] = { {1.0f, 0.0f, 0.0f}, {0.0f, cos_x, sin_x}, {0.0f, -sin_x, cos_x} };
	const float rz[3][3] = { {cos_z, sin_z, 0.0f}, {-sin_z, cos_z, 0.0f}, {0.0f, 0.0f, 1.0f} };
	float rotation[3][3] = {{0.0f}};
	for (int i = 0; i != 3; ++i) for (int j = 0; j != 3; ++j) for (int l = 0; l != 3; ++l) rotation[i][j] += rz[i][l] * rx[l][j];
	float origin[3] = {0.0f, 0.0f, 0.0f};
	for (int i = 0; i != 3; ++i) for (int j = 0; j != 3; ++j) origin[i] -= rotation[j][i] * camera->position_world_space[j];
	const float result[4][4] = {
		{ rotation[0][0], rotation[1][0], rotation[2][0], origin[0] },
		{ rotation[0][1], rotation[1][1], rotation[2][1], origin[1] },
		{ rotation[0][2], rotation[1][2], rotation[2][2], origin[2] },
		{ 0.0f, 0.0f, 0.0f, 1.0f } };
	memcpy(out, result, sizeof(result));
}

extern "C" void vkr_get_world_to_projection_space(float world_to_projection_space[4][4], const vkr_first_person_camera_t* camera, float aspect_ratio) {
	float w2v[4][4];
	world_to_view_space(w2v, camera);
	const float near_plane = camera->near_plane, far_plane = camera->far_plane;
	const float top = tanf(0.5f * camera->vertical_fov);
	const float right = aspect_ratio * top;
	const float v2p[4][4] = {
		{ -1.0f / right, 0.0f, 0.0f, 0.0f },
		{ 0.0f, 1.0f / top, 0.0f, 0.0f },
		{ 0.0f, 0.0f, -(far_plane + near_plane) / (far_plane - near_plane), -2.0f * far_plane * near_plane / (far_plane - near_plane) },
		{ 0.0f, 0.0f, -1.0f, 0.0f } };
	memset(world_to_projection_space, 0, sizeof(float) * 16);
	for (int i = 0; i != 4; ++i) for (int j = 0; j != 4; ++j) for (int l = 0; l != 4; ++l) world_to_projection_space[i][j] += v2p[i][l] * w2v[l][j];
}

// ------------------------------------------------------------------------------------------------
// quicksaves (layout: src/main.c:49-130) -- 64-bit size_t and pointers, like the reference
// ------------------------------------------------------------------------------------------------
static const size_t kQuicksaveLightBytes = sizeof(float) * 20 + sizeof(uint32_t) * 2; // POLYGONAL_LIGHT_QUICKSAVE_SIZE
static const size_t kLightFixedBytes = kQuicksaveLightBytes + sizeof(uint32_t) * 2 + sizeof(float) * 16; // POLYGONAL_LIGHT_FIXED_CONSTANT_BUFFER_SIZE

extern "C" void vkr_destroy_scene_specification(vkr_scene_specification_t* spec) {
	for (uint32_t i = 0; i != spec->polygonal_light_count; ++i) vkr_destroy_polygonal_light(&spec->polygonal_lights[i]);
	free(spec->polygonal_lights);
	memset(spec, 0, sizeof(*spec));
}

// ------------------------------------------------------------------------------------------------
// light textures (src/main.c:364-418)
// ------------------------------------------------------------------------------------------------
extern "C" void vkr_destroy_light_textures(vkr_light_textures_t* lt, const vkr_device_t* device) {
	(void) device;
	for (uint32_t i = 0; i != lt->texture_count && lt->textures; ++i) vkr_destroy_texture(&lt->textures[i]);
	free(lt->textures);
	void* dev_ptrs[] = { lt->d_texels, lt->d_dims, lt->d_offsets };
	for (void* p : dev_ptrs) if (p) cudaFree(p);
	memset(lt, 0, sizeof(*lt));
}

extern "C" int vkr_create_and_assign_light_textures(vkr_light_textures_t* lt, const vkr_device_t* device, vkr_scene_specification_t* spec) {
	if (lt) memset(lt, 0, sizeof(*lt));
	// unique paths in the order of first use; the empty string stands for the white default
	std::vector<std::string> unique_paths;
	for (uint32_t i = 0; i != spec->polygonal_light_count; ++i) {
		std::string path = spec->polygonal_lights[i].texture_file_path ? spec->polygonal_lights[i].texture_file_path : "";
		if (!path.empty()) {
			FILE* file = fopen(path.c_str(), "rb");
			if (file) fclose(file);
			else {
				printf("The light texture at path %s does not exist. Using a white texture instead.\n", path.c_str());
				path.clear();
			}
		}
		uint32_t index = (uint32_t) unique_paths.size();
		for (uint32_t j = 0; j != unique_paths.size(); ++j) if (unique_paths[j] == path) index = j;
		if (index == unique_paths.size()) unique_paths.push_back(path);
		spec->polygonal_lights[i].texture_index = index;
	}
	if (!lt) return 0;
	if (unique_paths.empty()) unique_paths.push_back(""); // the reference avoids empty descriptor arrays the same way
	lt->texture_count = (uint32_t) unique_paths.size();
	lt->textures = (vkr_texture_t*) calloc(lt->texture_count, sizeof(vkr_texture_t));
	bool failed = false;
	for (uint32_t i = 0; i != lt->texture_count && !failed; ++i) {
		vkr_texture_t& t = lt->textures[i];
		if (unique_paths[i].empty()) { // white, 1x1
			t.width = t.height = t.mip_count = 1; t.vk_format = 109; t.texel_float_count = 4; t.is_constant = 1;
			t.h_texels = (float*) malloc(4 * sizeof(float));
			for (int c = 0; c != 4; ++c) t.h_texels[c] = 1.0f;
		}
		else failed = vkr_load_texture(&t, unique_paths[i].c_str()) != 0;
	}
	if (!failed) {
		std::vector<uint32_t> dims(4 * (size_t) lt->texture_count); std::vector<uint64_t> offsets(lt->texture_count);
		uint64_t texel_count = 0;
		for (uint32_t k = 0; k != lt->texture_count; ++k) {
			dims[4 * k] = lt->textures[k].width; dims[4 * k + 1] = lt->textures[k].height; dims[4 * k + 2] = lt->textures[k].mip_count; dims[4 * k + 3] = 0;
			offsets[k] = texel_count; texel_count += lt->textures[k].texel_float_count / 4;
		}
		lt->texel_count = texel_count;
		if (device) {
			std::vector<float> data(4 * (size_t) texel_count);
			for (uint32_t k = 0; k != lt->texture_count; ++k) memcpy(&data[4 * (size_t) offsets[k]], lt->textures[k].h_texels, sizeof(float) * (size_t) lt->textures[k].texel_float_count);
			failed = upload(&lt->d_texels, data.data(), data.size() * 4, device) || upload(&lt->d_dims, dims.data(), dims.size() * 4, device) || upload(&lt->d_offsets, offsets.data(), offsets.size() * 8, device);
		}
	}
	if (failed) {
		printf("Failed to load the textures of the polygonal lights.\n");
		vkr_destroy_light_textures(lt, device); return 1;
	}
	return 0;
}

extern "C" int vkr_quick_load(vkr_scene_specification_t* spec, const char* quick_save_path) {
	FILE* file = fopen(quick_save_path, "rb");
	if (!file) { printf("Failed to load a quick save. Please check path and permissions: %s\n", quick_save_path); return 1; }
	vkr_scene_specification_t loaded; memset(&loaded, 0, sizeof(loaded));
	uint32_t legacy_count = 0;
	if (fread(&loaded.camera, sizeof(loaded.camera), 1, file) != 1 || fread(&legacy_count, 4, 1, file) != 1 || fread(&loaded.polygonal_light_count, 4, 1, file) != 1 || loaded.polygonal_light_count > 65536) {
		printf("The quick save at %s is truncated or corrupt.\n", quick_save_path);
		fclose(file); return 1;
	}
	loaded.polygonal_lights = (vkr_polygonal_light_t*) calloc(loaded.polygonal_light_count ? loaded.polygonal_light_count : 1, sizeof(vkr_polygonal_light_t));
	for (uint32_t i = 0; i != loaded.polygonal_light_count; ++i) {
		vkr_polygonal_light_t* light = &loaded.polygonal_lights[i];
		fread(light, kQuicksaveLightBytes, 1, file);
		if (light->scaling_y <= 0.0f) light->scaling_y = light->scaling_x; // legacy files
		uint64_t path_size = 0;
		fread(&path_size, 8, 1, file);
		if (path_size > 65536 || light->vertex_count < 3 || light->vertex_count > 4096) {
			printf("The quick save at %s is truncated or corrupt.\n", quick_save_path);
			loaded.polygonal_light_count = i; vkr_destroy_scene_specification(&loaded); fclose(file); return 1;
		}
		if (path_size) { light->texture_file_path = (char*) malloc(path_size); fread(light->texture_file_path, 1, path_size, file); light->texture_file_path[path_size - 1] = 0; }
		uint64_t legacy_pointers[2];
		fread(legacy_pointers, 8, 2, file);
		const uint32_t n = light->vertex_count;
		light->vertex_count = 0;
		vkr_set_polygonal_light_vertex_count(light, n);
		fread(light->vertices_plane_space, sizeof(float), 4 * (size_t) n, file);
	}
	fclose(file);
	vkr_destroy_scene_specification(spec);
	*spec = loaded;
	return 0;
}

extern "C" int vkr_quick_save(const vkr_scene_specification_t* spec, const char* quick_save_path) {
	FILE* file = fopen(quick_save_path, "wb");
	if (!file) { printf("Quick save failed. Please check path and permissions: %s\n", quick_save_path); return 1; }
	fwrite(&spec->camera, sizeof(spec->camera), 1, file);
	const uint32_t legacy_count = 0;
	fwrite(&legacy_count, 4, 1, file);
	fwrite(&spec->polygonal_light_count, 4, 1, file);
	for (uint32_t i = 0; i != spec->polygonal_light_count; ++i) {
		const vkr_polygonal_light_t* light = &spec->polygonal_lights[i];
		fwrite(light, kQuicksaveLightBytes, 1, file);
		uint64_t path_size = light->texture_file_path ? strlen(light->texture_file_path) + 1 : 0;
		fwrite(&path_size, 8, 1, file);
		if (path_size) fwrite(light->texture_file_path, 1, path_size, file);
		const uint64_t null_pointers[2] = {0, 0};
		fwrite(null_pointers, 8, 2, file);
		fwrite(light->vertices_plane_space, sizeof(float), 4 * (size_t) light->vertex_count, file);
	}
	fclose(file);
	return 0;
}

// ------------------------------------------------------------------------------------------------
// render settings and per-frame constants (src/main.c:232-249, 2114-2188; src/main.h:488-505)
// ------------------------------------------------------------------------------------------------
extern "C" void vkr_specify_default_render_settings(vkr_render_settings_t* settings) {
	memset(settings, 0, sizeof(*settings));
	settings->exposure_factor = 8.0f;
	settings->roughness_factor = 1.0f;
	settings->sample_count = 1;
	settings->sampling_strategies = vkr_sampling_strategies_diffuse_specular_mis;
	settings->mis_heuristic = vkr_mis_heuristic_optimal_clamped;
	settings->mis_visibility_estimate = 0.5f;
	settings->polygon_sampling_technique = vkr_sample_polygon_projected_solid_angle;
	settings->error_min_exponent = -7.0f;
	settings->trace_shadow_rays = 1;
	settings->show_polygonal_lights = 1;
	settings->animate_noise = 1;
}

static uint32_t max_light_vertex_count(const vkr_scene_specification_t* spec) {
	uint32_t m = 3;
	for (uint32_t i = 0; i != spec->polygonal_light_count; ++i) if (m < spec->polygonal_lights[i].vertex_count) m = spec->polygonal_lights[i].vertex_count;
	return m;
}

extern "C" size_t vkr_get_constants_size(const vkr_scene_specification_t* spec) {
	const uint32_t v = max_light_vertex_count(spec);
	return 256 + (size_t) spec->polygonal_light_count * (kLightFixedBytes + 16 * (size_t) v * 2 + 16 * (size_t) (v - 2));
}

namespace {
struct frame_constants { // = per_frame_constants_t, src/main.h:488-505
	float mesh_dequantization_factor[3], padding_0, mesh_dequantization_summand[3];
	float error_factor;
	float world_to_projection_space[4][4];
	float pixel_to_ray_direction_world_space[3][4];
	float camera_position_world_space[3];
	float mis_visibility_estimate;
	uint32_t viewport_size[2];
	int32_t cursor_position[2];
	float exposure_factor, roughness_factor;
	uint32_t noise_resolution_mask[2];
	uint32_t noise_texture_index_mask;
	uint32_t frame_bits;
	uint32_t padding_3[2];
	uint32_t noise_random_numbers[4];
	vkr_ltc_constants_t ltc_constants;
};
static_assert(sizeof(frame_constants) == 256, "constant block layout");

// General 4x4 inverse by cofactors in the reference's term order (math_utilities.h:24-46 semantics)
void invert_4x4(float inverse[4][4], const float matrix[4][4]) {
	const float* m = &matrix[0][0];
	float* inv = &inverse[0][0];
	// Cofactor expansion, every cofactor as six triple products added left to right (the term order
	// decides the rounding; it follows the reference so that pixel_to_ray_direction agrees bit for bit).
#define T3(a, b, c) (m[a] * m[b] * m[c])
	inv[0] = T3(5, 10, 15) - T3(5, 11, 14) - T3(9, 6, 15) + T3(9, 7, 14) + T3(13, 6, 11) - T3(13, 7, 10);
	inv[4] = -T3(4, 10, 15) + T3(4, 11, 14) + T3(8, 6, 15) - T3(8, 7, 14) - T3(12, 6, 11) + T3(12, 7, 10);
	inv[8] = T3(4, 9, 15) - T3(4, 11, 13) - T3(8, 5, 15) + T3(8, 7, 13) + T3(12, 5, 11) - T3(12, 7, 9);
	inv[12] = -T3(4, 9, 14) + T3(4, 10, 13) + T3(8, 5, 14) - T3(8, 6, 13) - T3(12, 5, 10) + T3(12, 6, 9);
	inv[1] = -T3(1, 10, 15) + T3(1, 11, 14) + T3(9, 2, 15) - T3(9, 3, 14) - T3(13, 2, 11) + T3(13, 3, 10);
	inv[5] = T3(0, 10, 15) - T3(0, 11, 14) - T3(8, 2, 15) + T3(8, 3, 14) + T3(12, 2, 11) - T3(12, 3, 10);
	inv[9] = -T3(0, 9, 15) + T3(0, 11, 13) + T3(8, 1, 15) - T3(8, 3, 13) - T3(12, 1, 11) + T3(12, 3, 9);
	inv[13] = T3(0, 9, 14) - T3(0, 10, 13) - T3(8, 1, 14) + T3(8, 2, 13) + T3(12, 1, 10) - T3(12, 2, 9);
	inv[2] = T3(1, 6, 15) - T3(1, 7, 14) - T3(5, 2, 15) + T3(5, 3, 14) + T3(13, 2, 7) - T3(13, 3, 6);
	inv[6] = -T3(0, 6, 15) + T3(0, 7, 14) + T3(4, 2, 15) - T3(4, 3, 14) - T3(12, 2, 7) + T3(12, 3, 6);
	inv[10] = T3(0, 5, 15) - T3(0, 7, 13) - T3(4, 1, 15) + T3(4, 3, 13) + T3(12, 1, 7) - T3(12, 3, 5);
	inv[14] = -T3(0, 5, 14) + T3(0, 6, 13) + T3(4, 1, 14) - T3(4, 2, 13) - T3(12, 1, 6) + T3(12, 2, 5);
	inv[3] = -T3(1, 6, 11) + T3(1, 7, 10) + T3(5, 2, 11) - T3(5, 3, 10) - T3(9, 2, 7) + T3(9, 3, 6);
	inv[7] = T3(0, 6, 11) - T3(0, 7, 10) - T3(4, 2, 11) + T3(4, 3, 10) + T3(8, 2, 7) - T3(8, 3, 6);
	inv[11] = -T3(0, 5, 11) + T3(0, 7, 9) + T3(4, 1, 11) - T3(4, 3, 9) - T3(8, 1, 7) + T3(8, 3, 5);
	inv[15] = T3(0, 5, 10) - T3(0, 6, 9) - T3(4, 1, 10) + T3(4, 2, 9) + T3(8, 1, 6) - T3(8, 2, 5);
#undef T3
	const float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
	const float rcp_det = 1.0f / det;
	for (int i = 0; i != 16; ++i) inv[i] = inv[i] * rcp_det;
}
}

extern "C" void vkr_set_frame_bits(void* constants, uint32_t frame_bits) {
	memcpy((char*) constants + 196, &frame_bits, sizeof(frame_bits)); // per_frame_constants_t::frame_bits (main.h:499)
}

extern "C" size_t vkr_write_constants(void* data, const vkr_scene_specification_t* spec, const vkr_render_settings_t* settings,
	const vkr_scene_t* scene, const vkr_ltc_table_t* ltc, vkr_noise_table_t* noise, uint32_t width, uint32_t height)
{
	frame_constants c; memset(&c, 0, sizeof(c));
	for (int i = 0; i != 3; ++i) {
		c.mesh_dequantization_factor[i] = scene->dequantization_factor[i];
		c.mesh_dequantization_summand[i] = scene->dequantization_summand[i];
		c.camera_position_world_space[i] = spec->camera.position_world_space[i];
	}
	c.mis_visibility_estimate = settings->mis_visibility_estimate;
	c.viewport_size[0] = width; c.viewport_size[1] = height;
	c.ltc_constants = ltc->constants;
	c.error_factor = powf(10.0f, -settings->error_min_exponent);
	c.exposure_factor = settings->exposure_factor;
	c.roughness_factor = settings->roughness_factor;
	c.frame_bits = 0;
	vkr_set_noise_constants(c.noise_resolution_mask, &c.noise_texture_index_mask, c.noise_random_numbers, noise, settings->animate_noise);
	const float aspect_ratio = ((float) width) / ((float) height);
	vkr_get_world_to_projection_space(c.world_to_projection_space, &spec->camera, aspect_ratio);
	float viewport_transform[4];
	viewport_transform[0] = 2.0f / width;
	viewport_transform[1] = 2.0f / height;
	viewport_transform[2] = 0.5f * viewport_transform[0] - 1.0f;
	viewport_transform[3] = 0.5f * viewport_transform[1] - 1.0f;
	float w2p_no_translation[4][4], p2w_no_translation[4][4];
	memcpy(w2p_no_translation, c.world_to_projection_space, sizeof(w2p_no_translation));
	w2p_no_translation[0][3] = 0.0f; w2p_no_translation[1][3] = 0.0f; w2p_no_translation[2][3] = 0.0f;
	invert_4x4(p2w_no_translation, w2p_no_translation);
	const float pixel_to_projection[4][3] = {
		{ viewport_transform[0], 0.0f, viewport_transform[2] },
		{ 0.0f, viewport_transform[1], viewport_transform[3] },
		{ 0.0f, 0.0f, 1.0f },
		{ 0.0f, 0.0f, 1.0f } };
	for (int i = 0; i != 3; ++i) for (int j = 0; j != 3; ++j) for (int k = 0; k != 4; ++k)
		c.pixel_to_ray_direction_world_space[i][j] += p2w_no_translation[i][k] * pixel_to_projection[k][j];
	memcpy(data, &c, sizeof(c));
	size_t offset = sizeof(c);
	const uint32_t max_v = max_light_vertex_count(spec);
	char* out = (char*) data;
	for (uint32_t i = 0; i != spec->polygonal_light_count; ++i) {
		vkr_polygonal_light_t* light = &spec->polygonal_lights[i];
		vkr_update_polygonal_light(light);
		memcpy(out + offset, light, kLightFixedBytes);
		offset += kLightFixedBytes;
		const float* vertex_data[2] = { light->vertices_plane_space, light->vertices_world_space };
		for (int j = 0; j != 2; ++j) {
			memset(out + offset, 0, 16 * (size_t) max_v);
			memcpy(out + offset, vertex_data[j], 16 * (size_t) light->vertex_count);
			if (light->vertex_count < max_v) memcpy(out + offset + 16 * (size_t) light->vertex_count, vertex_data[j], 16);
			offset += 16 * (size_t) max_v;
		}
		// fan areas, the last entry repeated (the reference reads past the array here when vertex_count < max,
		// main.c:2184 -- only Turk sampling consumes these, so we repeat the last valid entry instead)
		memcpy(out + offset, light->fan_areas, 16 * (size_t) (light->vertex_count - 2));
		offset += 16 * (size_t) (light->vertex_count - 2);
		for (uint32_t k = light->vertex_count; k != max_v; ++k) {
			memcpy(out + offset, light->fan_areas + 4 * (size_t) (light->vertex_count - 3), 16);
			offset += 16;
		}
	}
	return offset;
}

// ------------------------------------------------------------------------------------------------
// host-side probe of the BVH builder (structural tests without a GPU)
// ------------------------------------------------------------------------------------------------
namespace vkr {
bvh_builder bvh_builder_from_environment() {
	const char* name = getenv("VKR_BVH_BUILDER");
	if (name && !strcmp(name, "lbvh")) return bvh_builder_lbvh;
	if (name && !strcmp(name, "lbvh_gpu")) return bvh_builder_lbvh_gpu;
	return bvh_builder_sah;
}
}

// builder: 0 = binned SAH (vkr_bvh.cpp, what scenes are loaded with by default), 1 = linear BVH (vkr_lbvh.cpp)
extern "C" int vkr_bvh_build_probe_with(int builder, const float* vertices, uint64_t triangle_count, float** out_nodes, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth) {
	host_bvh bvh;
	if (builder == 1) build_lbvh(bvh, vertices, triangle_count);
	else if (builder == 0) build_bvh(bvh, vertices, triangle_count);
	else { printf("The BVH builder probe knows the host builders 0 (SAH) and 1 (linear BVH), not %d.\n", builder); return 1; }
	*out_nodes = (float*) malloc(sizeof(float) * (bvh.nodes.size() ? bvh.nodes.size() : 1));
	*out_tris = (float*) malloc(sizeof(float) * (bvh.tris.size() ? bvh.tris.size() : 1));
	*out_tri_ids = (uint32_t*) malloc(sizeof(uint32_t) * (bvh.tri_ids.size() ? bvh.tri_ids.size() : 1));
	memcpy(*out_nodes, bvh.nodes.data(), sizeof(float) * bvh.nodes.size());
	memcpy(*out_tris, bvh.tris.data(), sizeof(float) * bvh.tris.size());
	memcpy(*out_tri_ids, bvh.tri_ids.data(), sizeof(uint32_t) * bvh.tri_ids.size());
	*out_node_count = bvh.node_count; *out_max_depth = bvh.max_depth;
	return 0;
}
// The GPU builder's output copied to the host in the format of the host probes (tests: array-for-array equality with builder 1)
extern "C" int vkr_bvh_build_probe_device(const vkr_device_t* device, const float* vertices, uint64_t triangle_count, float** out_nodes, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth) {
	*out_nodes = nullptr; *out_tris = nullptr; *out_tri_ids = nullptr; *out_node_count = 0; *out_max_depth = 0;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess) { printf("Failed to select the CUDA device for the BVH builder probe.\n"); return 1; }
	void *d_nodes = nullptr, *d_tris = nullptr, *d_ids = nullptr; uint64_t pairs = 0; uint32_t depth = 0;
	if (build_lbvh_device(vertices, triangle_count, device->stream, &d_nodes, &d_tris, &d_ids, &pairs, &depth)) {
		printf("The GPU BVH builder failed for %llu triangles.\n", (unsigned long long) triangle_count); return 1;
	}
	*out_nodes = (float*) malloc(sizeof(float) * 16 * (pairs ? pairs : 1));
	*out_tris = (float*) malloc(sizeof(float) * 12 * triangle_count);
	*out_tri_ids = (uint32_t*) malloc(sizeof(uint32_t) * triangle_count);
	const bool ok = cudaMemcpy(*out_nodes, d_nodes, sizeof(float) * 16 * pairs, cudaMemcpyDeviceToHost) == cudaSuccess
		&& cudaMemcpy(*out_tris, d_tris, sizeof(float) * 12 * triangle_count, cudaMemcpyDeviceToHost) == cudaSuccess
		&& cudaMemcpy(*out_tri_ids, d_ids, sizeof(uint32_t) * triangle_count, cudaMemcpyDeviceToHost) == cudaSuccess;
	cudaFree(d_nodes); cudaFree(d_tris); cudaFree(d_ids);
	if (!ok) { free(*out_nodes); free(*out_tris); free(*out_tri_ids); *out_nodes = nullptr; *out_tris = nullptr; *out_tri_ids = nullptr; printf("Failed to copy the BVH to the host.\n"); return 1; }
	*out_node_count = pairs; *out_max_depth = depth;
	return 0;
}

// The 4-wide collapse of builder 0's tree (vkr_bvh.h: host_bvh4): nodes4 = 32 floats per node, tris / tri_ids as in the other probes
extern "C" int vkr_bvh4_build_probe(const float* vertices, uint64_t triangle_count, float** out_nodes4, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth,
	uint64_t* out_bvh2_node_count, uint32_t* out_bvh2_max_depth)
{
	host_bvh bvh; host_bvh4 wide;
	build_bvh(bvh, vertices, triangle_count);
	build_bvh4_from_bvh2(wide, bvh);
	*out_nodes4 = (float*) malloc(sizeof(float) * wide.nodes.size());
	*out_tris = (float*) malloc(sizeof(float) * (bvh.tris.size() ? bvh.tris.size() : 1));
	*out_tri_ids = (uint32_t*) malloc(sizeof(uint32_t) * (bvh.tri_ids.size() ? bvh.tri_ids.size() : 1));
	memcpy(*out_nodes4, wide.nodes.data(), sizeof(float) * wide.nodes.size());
	memcpy(*out_tris, bvh.tris.data(), sizeof(float) * bvh.tris.size());
	memcpy(*out_tri_ids, bvh.tri_ids.data(), sizeof(uint32_t) * bvh.tri_ids.size());
	*out_node_count = wide.node_count; *out_max_depth = wide.max_depth;
	*out_bvh2_node_count = bvh.node_count; *out_bvh2_max_depth = bvh.max_depth;
	return 0;
}

extern "C" int vkr_bvh_build_probe(const float* vertices, uint64_t triangle_count, float** out_nodes, uint64_t* out_node_count, float** out_tris, uint32_t** out_tri_ids, uint32_t* out_max_depth) {
	return vkr_bvh_build_probe_with(0, vertices, triangle_count, out_nodes, out_node_count, out_tris, out_tri_ids, out_max_depth);
}
extern "C" void vkr_bvh_free_probe(float* nodes, float* tris, uint32_t* tri_ids) { free(nodes); free(tris); free(tri_ids); }
