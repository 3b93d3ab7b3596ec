/* oracle/ref_jpeg.c -- TEST INFRASTRUCTURE: stbi_write_jpg of the reference's own stb_image_write.h, compiled where it lies by oracle/build_ref_jpeg.py
   into oracle/_ref/libref_jpeg.so, writing into a caller's buffer instead of a file. */
#include <stddef.h>
#include <string.h>

#define STB_IMAGE_WRITE_IMPLEMENTATION
#include "stb_image_write.h"

typedef struct { unsigned char* data; size_t capacity, size; } ref_jpeg_buffer_t;

static void append(void* context, void* data, int size) {
	ref_jpeg_buffer_t* b = (ref_jpeg_buffer_t*) context;
	if (b->size + (size_t) size <= b->capacity) memcpy(b->data + b->size, data, (size_t) size);
	b->size += (size_t) size;
}

/* 8-bit RGB; returns stb's result (1 = written); *out_size = the file's size, bytes beyond capacity are dropped */
int ref_write_jpg(const unsigned char* rgb8, int width, int height, int quality, unsigned char* out, size_t capacity, size_t* out_size) {
	ref_jpeg_buffer_t b = { out, capacity, 0 };
	const int ok = stbi_write_jpg_to_func(append, &b, width, height, 3, rgb8, quality);
	*out_size = b.size;
	return ok;
}
