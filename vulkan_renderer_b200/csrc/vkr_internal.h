// vkr_internal.h -- helpers shared by the host translation units of libvkr_b200.so
#pragma once
#include "../../include/vkr_b200.h"
#include <stddef.h>
namespace vkr {
// cudaMalloc + synchronous copy; returns non-zero on failure and leaves *d_ptr NULL
int upload(void** d_ptr, const void* src, size_t bytes, const vkr_device_t* device);
// vkr_jpeg.cu: the UNORM8 quantisation of a DEVICE float4 frame into DEVICE RGB bytes (asynchronous on device->stream), and the *.jpg file of
// DEVICE RGB bytes (synchronous)
int jpeg_quantize(const vkr_device_t* device, const float* d_rgba32f, uint32_t width, uint32_t height, uint8_t* d_rgb8);
int jpeg_write_device_image(const vkr_device_t* device, const char* path, const uint8_t* d_rgb8, uint32_t width, uint32_t height, int quality);
}
