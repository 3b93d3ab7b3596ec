// vkr_output.cpp -- what happens to a frame after the shading pass: screenshots and frame times (SURVEY 8 row f3).
//
// Replaces take_screenshot / implement_screenshot / combine_ldr_screenshots_into_hdr (src/main.c:1550-1770), the three
// stb_image_write entry points they call (*.png, *.hdr) and the frame timer (src/frame_timer.c:28-75). The reference reads the
// swapchain image back; here the frame is the float4 image the shading pass wrote, and the 8-bit quantisation the render
// target would have applied is done explicitly. File writers are written from the format specifications (PNG: stored deflate
// blocks, Radiance RGBE: run-length scanlines of literal packets) -- small and dependency-free, any reader opens the files.
// Host code: no contraction (-ffp-contract=off).
#include "vkr_b200.h"
#include "vkr_internal.h"
#include "vkr_jpeg.cuh"
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>

// ---------------------------------------------------------------------------------------------------------------------
// Render targets (create_render_targets / destroy_render_targets, src/main.c:253-315)
extern "C" void vkr_destroy_render_targets(vkr_render_targets_t* targets, const vkr_device_t* device) {
	(void) device;
	if (targets->d_visibility) cudaFree(targets->d_visibility);
	if (targets->d_gbuffer) cudaFree(targets->d_gbuffer);
	if (targets->d_frame) cudaFree(targets->d_frame);
	memset(targets, 0, sizeof(*targets));
}

extern "C" int vkr_create_render_targets(vkr_render_targets_t* targets, const vkr_device_t* device, uint32_t width, uint32_t height) {
	memset(targets, 0, sizeof(*targets));
	if (!width || !height) { printf("Failed to create render targets: the resolution is %ux%u.\n", width, height); return 1; }
	const size_t pixel_count = (size_t) width * height;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess || cudaMalloc(&targets->d_visibility, sizeof(uint32_t) * pixel_count) != cudaSuccess
		|| cudaMalloc(&targets->d_gbuffer, vkr_gbuffer_size(width, height)) != cudaSuccess || cudaMalloc(&targets->d_frame, sizeof(float) * 4 * pixel_count) != cudaSuccess)
	{
		printf("Failed to create render targets of resolution %ux%u.\n", width, height);
		vkr_destroy_render_targets(targets, device);
		return 1;
	}
	targets->width = width; targets->height = height;
	cudaMemsetAsync(targets->d_visibility, 0xFF, sizeof(uint32_t) * pixel_count, (cudaStream_t) device->stream);
	cudaMemsetAsync(targets->d_frame, 0, sizeof(float) * 4 * pixel_count, (cudaStream_t) device->stream);
	return 0;
}

static int copy_and_wait(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, const vkr_device_t* device, const char* what) {
	cudaStream_t stream = (cudaStream_t) device->stream;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess || cudaMemcpyAsync(dst, src, bytes, kind, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess) {
		printf("Failed to copy %s: %s\n", what, cudaGetErrorString(cudaGetLastError()));
		return 1;
	}
	return 0;
}

extern "C" int vkr_download_frame(const vkr_render_targets_t* targets, const vkr_device_t* device, float* out_rgba32f) {
	return copy_and_wait(out_rgba32f, targets->d_frame, sizeof(float) * 4 * (size_t) targets->width * targets->height, cudaMemcpyDeviceToHost, device, "the frame to the host");
}

extern "C" int vkr_download_gbuffer(const vkr_render_targets_t* targets, const vkr_device_t* device, uint32_t* out_visibility, float* out_gbuffer) {
	if (out_visibility && copy_and_wait(out_visibility, targets->d_visibility, sizeof(uint32_t) * (size_t) targets->width * targets->height, cudaMemcpyDeviceToHost, device, "the visibility buffer to the host")) return 1;
	if (out_gbuffer && copy_and_wait(out_gbuffer, targets->d_gbuffer, vkr_gbuffer_size(targets->width, targets->height), cudaMemcpyDeviceToHost, device, "the G-buffer to the host")) return 1;
	return 0;
}

extern "C" int vkr_upload_gbuffer(vkr_render_targets_t* targets, const vkr_device_t* device, const float* gbuffer) {
	return copy_and_wait(targets->d_gbuffer, gbuffer, vkr_gbuffer_size(targets->width, targets->height), cudaMemcpyHostToDevice, device, "the G-buffer to the device");
}

// ---------------------------------------------------------------------------------------------------------------------
// 8-bit render target: UNORM conversion as Vulkan specifies it (round to nearest of clamp(x, 0, 1) * 255); NaN -> 0
extern "C" void vkr_quantize_unorm8(const float* rgba32f, uint32_t width, uint32_t height, uint8_t* out_rgb8) {
	const size_t pixel_count = (size_t) width * height;
	for (size_t i = 0; i != pixel_count; ++i)
		for (int c = 0; c != 3; ++c) {
			out_rgb8[3 * i + c] = vkr_jpeg::unorm8(rgba32f[4 * i + c]);   // the device quantisation of JPEG screenshots shares it
		}
}

// half_to_float (src/math_utilities.h:70-84)
static float half_to_float(uint16_t half) {
	uint32_t u = ((uint32_t) half & 0x7fffu) << 13;
	float f; memcpy(&f, &u, 4);
	const uint32_t magic_bits = (254u - 15u) << 23, infnan_bits = (127u + 16u) << 23;
	float magic, was_infnan; memcpy(&magic, &magic_bits, 4); memcpy(&was_infnan, &infnan_bits, 4);
	f *= magic;
	memcpy(&u, &f, 4);
	if (f >= was_infnan) u |= 255u << 23;
	u |= ((uint32_t) half & 0x8000u) << 16;
	memcpy(&f, &u, 4);
	return f;
}

// combine_ldr_screenshots_into_hdr (src/main.c:1696-1707): entry i of the two LDR frames holds the low / high byte of a half
extern "C" void vkr_combine_ldr_screenshots_into_hdr(const uint8_t* low_bytes, const uint8_t* high_bytes, size_t entry_count, float* out_hdr) {
	for (size_t i = 0; i != entry_count; ++i)
		out_hdr[i] = half_to_float((uint16_t) ((uint16_t) low_bytes[i] | ((uint16_t) high_bytes[i] << 8)));
}

// ---------------------------------------------------------------------------------------------------------------------
// *.png (stbi_write_png at src/main.c:1734): 8-bit RGB, filter type 0, zlib stream of stored blocks
static uint32_t crc32_update(uint32_t crc, const uint8_t* data, size_t size) {
	static uint32_t table[256];
	static bool ready = false;
	if (!ready) {
		for (uint32_t n = 0; n != 256; ++n) {
			uint32_t c = n;
			for (int k = 0; k != 8; ++k) c = (c & 1u) ? (0xEDB88320u ^ (c >> 1)) : (c >> 1);
			table[n] = c;
		}
		ready = true;
	}
	for (size_t i = 0; i != size; ++i) crc = table[(crc ^ data[i]) & 0xFFu] ^ (crc >> 8);
	return crc;
}
static void put_u32_be(std::vector<uint8_t>& v, uint32_t x) { v.push_back((uint8_t) (x >> 24)); v.push_back((uint8_t) (x >> 16)); v.push_back((uint8_t) (x >> 8)); v.push_back((uint8_t) x); }
static void put_chunk(std::vector<uint8_t>& file, const char type[4], const std::vector<uint8_t>& payload) {
	put_u32_be(file, (uint32_t) payload.size());
	const size_t begin = file.size();
	file.insert(file.end(), type, type + 4);
	file.insert(file.end(), payload.begin(), payload.end());
	put_u32_be(file, crc32_update(0xFFFFFFFFu, file.data() + begin, file.size() - begin) ^ 0xFFFFFFFFu);
}

extern "C" int vkr_write_png(const char* file_path, uint32_t width, uint32_t height, const uint8_t* rgb8) {
	if (!width || !height || !rgb8) { printf("Failed to write %s: empty image.\n", file_path); return 1; }
	// scanlines with filter byte 0
	std::vector<uint8_t> raw((size_t) height * (3 * (size_t) width + 1));
	for (uint32_t y = 0; y != height; ++y) {
		raw[(size_t) y * (3 * (size_t) width + 1)] = 0;
		memcpy(&raw[(size_t) y * (3 * (size_t) width + 1) + 1], rgb8 + (size_t) y * 3 * width, 3 * (size_t) width);
	}
	// zlib: CMF/FLG, stored blocks of at most 65535 bytes, Adler-32
	std::vector<uint8_t> z;
	z.push_back(0x78); z.push_back(0x01);
	uint32_t a = 1, b = 0;
	for (size_t offset = 0; offset < raw.size(); offset += 65535) {
		const size_t n = std::min<size_t>(65535, raw.size() - offset);
		z.push_back((offset + n == raw.size()) ? 1 : 0);
		z.push_back((uint8_t) n); z.push_back((uint8_t) (n >> 8)); z.push_back((uint8_t) ~n); z.push_back((uint8_t) (~n >> 8));
		z.insert(z.end(), raw.begin() + offset, raw.begin() + offset + n);
		for (size_t i = 0; i != n; ++i) { a = (a + raw[offset + i]) % 65521u; b = (b + a) % 65521u; }
	}
	put_u32_be(z, (b << 16) | a);
	std::vector<uint8_t> file = { 0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A };
	std::vector<uint8_t> header;
	put_u32_be(header, width); put_u32_be(header, height);
	header.push_back(8); header.push_back(2); header.push_back(0); header.push_back(0); header.push_back(0); // 8 bit, RGB, deflate, adaptive filtering, no interlace
	put_chunk(file, "IHDR", header);
	put_chunk(file, "IDAT", z);
	put_chunk(file, "IEND", std::vector<uint8_t>());
	FILE* f = fopen(file_path, "wb");
	if (!f || fwrite(file.data(), 1, file.size(), f) != file.size()) {
		if (f) fclose(f);
		printf("Failed to store a screenshot to the *.png file at %s. Please check path and permissions.\n", file_path);
		return 1;
	}
	fclose(f);
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// *.hdr (stbi_write_hdr at src/main.c:1755): Radiance RGBE, shared exponent = exponent of the largest channel
static void float_to_rgbe(uint8_t rgbe[4], const float* rgb) {
	const float max_component = std::max(rgb[0], std::max(rgb[1], rgb[2]));
	if (!(max_component >= 1.0e-32f)) { rgbe[0] = rgbe[1] = rgbe[2] = rgbe[3] = 0; return; }
	int exponent;
	const float normalize = frexpf(max_component, &exponent) * 256.0f / max_component;
	for (int c = 0; c != 3; ++c) rgbe[c] = (uint8_t) (rgb[c] > 0.0f ? rgb[c] * normalize : 0.0f);
	rgbe[3] = (uint8_t) (exponent + 128);
}

extern "C" int vkr_write_hdr(const char* file_path, uint32_t width, uint32_t height, const float* rgb32f) {
	if (!width || !height || !rgb32f) { printf("Failed to write %s: empty image.\n", file_path); return 1; }
	FILE* f = fopen(file_path, "wb");
	if (!f) { printf("Failed to store a screenshot to the *.hdr file at %s. Please check path and permissions.\n", file_path); return 1; }
	fprintf(f, "#?RADIANCE\n# Written by vkr_b200\nFORMAT=32-bit_rle_rgbe\n\n-Y %u +X %u\n", height, width);
	std::vector<uint8_t> line((size_t) width * 4), out;
	const bool rle = width >= 8 && width < 32768; // the run-length format cannot express other widths
	for (uint32_t y = 0; y != height; ++y) {
		for (uint32_t x = 0; x != width; ++x) float_to_rgbe(&line[4 * (size_t) x], rgb32f + 3 * ((size_t) y * width + x));
		out.clear();
		if (!rle) out = line;
		else {
			out.push_back(2); out.push_back(2); out.push_back((uint8_t) (width >> 8)); out.push_back((uint8_t) width);
			for (int c = 0; c != 4; ++c) // one channel after the other, literal packets of at most 128 bytes
				for (uint32_t x = 0; x < width; x += 128) {
					const uint32_t n = std::min<uint32_t>(128, width - x);
					out.push_back((uint8_t) n);
					for (uint32_t i = 0; i != n; ++i) out.push_back(line[4 * (size_t) (x + i) + c]);
				}
		}
		if (fwrite(out.data(), 1, out.size(), f) != out.size()) {
			fclose(f);
			printf("Failed to store a screenshot to the *.hdr file at %s. Please check path and permissions.\n", file_path);
			return 1;
		}
	}
	fclose(f);
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Frame timer (src/frame_timer.c:28-75): the median of the differences of the last 100 recorded times. File-scope state
// like the reference's; one caller thread (SURVEY 8b).
enum { FRAME_TIME_COUNT = 100 };
static double g_recorded_times[FRAME_TIME_COUNT] = { 0.0 };
static uint32_t g_recorded_time_index = FRAME_TIME_COUNT - 1;

extern "C" void vkr_record_frame_time(double time_in_seconds) {
	++g_recorded_time_index;
	if (g_recorded_time_index >= FRAME_TIME_COUNT) g_recorded_time_index -= FRAME_TIME_COUNT;
	g_recorded_times[g_recorded_time_index] = time_in_seconds;
}

extern "C" void vkr_reset_frame_times(void) {
	memset(g_recorded_times, 0, sizeof(g_recorded_times));
	g_recorded_time_index = FRAME_TIME_COUNT - 1;
}

extern "C" float vkr_get_frame_time(void) {
	float frame_times[FRAME_TIME_COUNT];
	uint32_t recorded_count = 0;
	for (int32_t i = 0; i != FRAME_TIME_COUNT - 1; ++i) {
		const int32_t lhs = ((int32_t) g_recorded_time_index + FRAME_TIME_COUNT - i) % FRAME_TIME_COUNT;
		const int32_t rhs = ((int32_t) g_recorded_time_index + FRAME_TIME_COUNT - i - 1) % FRAME_TIME_COUNT;
		if (g_recorded_times[lhs] != 0.0 && g_recorded_times[rhs] != 0.0)
			frame_times[recorded_count++] = (float) (g_recorded_times[lhs] - g_recorded_times[rhs]);
	}
	if (recorded_count == 0) return 0.0f;
	std::sort(frame_times, frame_times + recorded_count);
	return frame_times[recorded_count / 2];
}

// ---------------------------------------------------------------------------------------------------------------------
// Screenshot of one frame (take_screenshot + implement_screenshot, src/main.c:1550-1770). LDR: the shader converts to sRGB, the
// 8-bit target quantises. HDR: two LDR frames carry the low and the high bytes of the half-precision colours (g_frame_bits = 1, 2;
// shading_pass.frag.glsl:871-887) and are combined on the host -- kept as the reference does it so that the files agree.
// *.jpg (stbi_write_jpg at quality 70, src/main.c:1745-1751): the frame is quantised and encoded on the device (vkr_jpeg.cu), so only the
// file comes back.
static const int kScreenshotJpegQuality = 70;

extern "C" int vkr_take_screenshot_formats(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer,
	const char* path_png, const char* path_jpg, const char* path_hdr)
{
	if ((path_png || path_jpg) && path_hdr) { printf("Cannot mix LDR and HDR screenshots.\n"); return 1; }
	if (!path_png && !path_jpg && !path_hdr) return 0;
	const uint32_t width = pass->desc.width, height = pass->desc.height;
	const size_t pixel_count = (size_t) width * height;
	if (constants_size != pass->constants_size || pass->desc.stripe_count > 1) { printf("Failed to take a screenshot: wrong constant block size or a striped pass.\n"); return 1; }
	const bool host_frame = path_png || path_hdr;   // *.png and *.hdr are written from the frame on the host
	std::vector<uint8_t> block((const uint8_t*) constants, (const uint8_t*) constants + constants_size);
	std::vector<float> frame(host_frame ? 4 * pixel_count : 0);
	std::vector<uint8_t> ldr(host_frame ? 3 * pixel_count * (path_hdr ? 2 : 1) : 0);
	void* d_frame = nullptr;
	void* d_rgb8 = nullptr;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess || cudaMalloc(&d_frame, sizeof(float) * 4 * pixel_count) != cudaSuccess
		|| (path_jpg && cudaMalloc(&d_rgb8, 3 * pixel_count) != cudaSuccess))
	{
		printf("Failed to create a staging image for taking a screenshot.\n");
		if (d_frame) cudaFree(d_frame);
		return 1;
	}
	const int saved_srgb = pass->desc.output_srgb;
	pass->desc.output_srgb = 1; // an UNORM render target: the shader itself converts to sRGB (OUTPUT_LINEAR_RGB=0)
	int failed = 0;
	for (uint32_t frame_bits = (path_hdr ? 1u : 0u); frame_bits <= (path_hdr ? 2u : 0u) && !failed; ++frame_bits) {
		vkr_set_frame_bits(block.data(), frame_bits);
		failed = vkr_shading_pass_run(pass, device, block.data(), constants_size, d_gbuffer, d_frame) || vkr_shading_pass_wait(pass, device);
		if (!failed && path_jpg) failed = vkr::jpeg_quantize(device, (const float*) d_frame, width, height, (uint8_t*) d_rgb8);
		if (!failed && host_frame) {
			failed = cudaMemcpy(frame.data(), d_frame, sizeof(float) * 4 * pixel_count, cudaMemcpyDeviceToHost) != cudaSuccess;
			if (!failed) vkr_quantize_unorm8(frame.data(), width, height, ldr.data() + (frame_bits == 2 ? 3 * pixel_count : 0));
		}
	}
	pass->desc.output_srgb = saved_srgb;
	if (failed) printf("Failed to render the frame for a screenshot.\n");
	else if (path_jpg) {
		failed = vkr::jpeg_write_device_image(device, path_jpg, (const uint8_t*) d_rgb8, width, height, kScreenshotJpegQuality);
		if (!failed) printf("Wrote screenshot to %s.\n", path_jpg);
	}
	cudaFree(d_frame);
	if (d_rgb8) cudaFree(d_rgb8);
	if (failed) return 1;
	if (path_png) {
		if (vkr_write_png(path_png, width, height, ldr.data())) return 1;
		printf("Wrote screenshot to %s.\n", path_png);
	}
	else if (path_hdr) {
		std::vector<float> hdr(3 * pixel_count);
		vkr_combine_ldr_screenshots_into_hdr(ldr.data(), ldr.data() + 3 * pixel_count, 3 * pixel_count, hdr.data());
		if (vkr_write_hdr(path_hdr, width, height, hdr.data())) return 1;
		printf("Wrote screenshot to %s.\n", path_hdr);
	}
	return 0;
}

extern "C" int vkr_take_screenshot(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer,
	const char* path_png, const char* path_hdr)
{
	return vkr_take_screenshot_formats(pass, device, constants, constants_size, d_gbuffer, path_png, nullptr, path_hdr);
}
