// vkr_exchange.cu -- one frame on several GPUs of a box: the frame exchange (include/vkr_b200.h, vkr_frame_exchange_t).
//
// The reference renders on one GPU (render_frame, src/main.c:2197-2270); SURVEY 8e adds the split over the GPUs of an HGX box. Every GPU shades
// its share of the screen tiles and the shading kernel's epilogue stores each finished pixel into the frame of EVERY GPU -- its own and, through
// peer mappings over NVLink / NVSwitch, the others' (vkr_shading_tile.cuh, out_peers). What is left to do per frame is a barrier, made of two
// one-block kernels on the launching stream:
//   signal  release at system scope, then this GPU's arrival counter on every peer := frame number   (after the shading kernel in stream order)
//   wait    acquire: spin until the counters of all peers have reached the frame number              (bounded: a peer that died must not hang the GPU)
// Frames alternate between two buffers, so a fast GPU may write frame f + 1 while a slow one still reads frame f; it cannot reach frame f + 2 (the
// same buffer again) before the slow one has signalled f + 1, i.e. has left frame f behind in stream order.
//
// Processes exchange the 64-byte cudaIpcMemHandle_t of their blocks by their own means (bench.py: torch.distributed.all_gather_object; a C host: MPI
// or a socket); a single process driving all GPUs hands the pointers over directly. No collective library is involved.
#include "../../include/vkr_b200.h"
#include "vkr_internal.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>

#define VKR_CUDA_OK(call, what) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { printf("%s: %s\n", what, cudaGetErrorString(e_)); return 1; } } while (0)

int vkr_launch_shading(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, void* d_out, unsigned long long* d_stats,
	int peer_count, void* const* peer_outs);   // vkr_api.cu
int vkr_copy_tile_columns(const vkr_shading_pass_desc_t& d, void* dst, const void* src, size_t texel, cudaMemcpyKind kind, cudaStream_t stream);   // vkr_api.cu
extern "C" int vkr_frame_exchange_wait(vkr_frame_exchange_t* e, const vkr_device_t* device);

namespace {

struct peer_counters { unsigned long long* p[VKR_MAX_GPUS]; };

size_t frame_bytes(const vkr_frame_exchange_t* e) { return (size_t) e->width * e->height * 16; }
size_t block_bytes(const vkr_frame_exchange_t* e) { return 2 * frame_bytes(e) + sizeof(unsigned long long) * VKR_MAX_GPUS; }
// arrival counters of a block: counter[r] = number of the last frame rank r has finished writing into this block
unsigned long long* counters_of(const vkr_frame_exchange_t* e, void* block) { return (unsigned long long*) ((char*) block + 2 * frame_bytes(e)); }

__global__ void exchange_signal_kernel(peer_counters peers, int world, int rank, unsigned long long frame) {
	const int k = threadIdx.x;
	if (k < world && k != rank) {
		// everything this GPU wrote before (the shading kernel's peer stores precede this kernel in stream order) becomes visible before the counter does
		__threadfence_system();
		asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(peers.p[k] + rank), "l"(frame) : "memory");
	}
}

__global__ void exchange_wait_kernel(const unsigned long long* counters, int world, int rank, unsigned long long frame, unsigned long long timeout_ns, int* status) {
	const int k = threadIdx.x;
	if (k < world && k != rank) {
		unsigned long long begin, now;
		asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(begin));
		while (true) {
			unsigned long long seen;
			asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(counters + k) : "memory");
			if (seen >= frame) break;
			asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
			if (now - begin > timeout_ns) { *status = 1 + k; break; } // rank k never arrived: report instead of hanging the GPU
			__nanosleep(200);
		}
	}
	__syncthreads();
	__threadfence_system();
}

} // namespace

extern "C" void vkr_destroy_frame_exchange(vkr_frame_exchange_t* e, const vkr_device_t* device) {
	if (device && device->stream) { cudaSetDevice(device->cuda_device); cudaStreamSynchronize((cudaStream_t) device->stream); }
	for (uint32_t r = 0; r != VKR_MAX_GPUS; ++r)
		if (e->peer_is_ipc[r] && e->d_peer_blocks[r]) cudaIpcCloseMemHandle(e->d_peer_blocks[r]);
	if (e->d_block) cudaFree(e->d_block);
	if (e->h_status) cudaFreeHost(e->h_status);
	memset(e, 0, sizeof(*e));
}

extern "C" int vkr_create_frame_exchange(vkr_frame_exchange_t* e, const vkr_device_t* device, uint32_t width, uint32_t height, uint32_t rank, uint32_t world) {
	memset(e, 0, sizeof(*e));
	if (!width || !height || !world || world > VKR_MAX_GPUS || rank >= world) {
		printf("Failed to create a frame exchange: %ux%u pixels, rank %u of %u (at most %d GPUs).\n", width, height, rank, world, VKR_MAX_GPUS);
		return 1;
	}
	e->width = width; e->height = height; e->rank = rank; e->world = world; e->timeout_ns = 20ull * 1000000000ull;
	if (cudaSetDevice(device->cuda_device) != cudaSuccess || cudaMalloc(&e->d_block, block_bytes(e)) != cudaSuccess
		|| cudaMemset(e->d_block, 0, block_bytes(e)) != cudaSuccess || cudaHostAlloc((void**) &e->h_status, sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess)
	{
		printf("Failed to create a frame exchange: could not allocate %llu bytes on CUDA device %d.\n", (unsigned long long) block_bytes(e), device->cuda_device);
		vkr_destroy_frame_exchange(e, nullptr); return 1;
	}
	*e->h_status = 0;
	e->d_peer_blocks[rank] = e->d_block;
	return 0;
}

extern "C" int vkr_frame_exchange_get_handle(const vkr_frame_exchange_t* e, const vkr_device_t* device, unsigned char out_handle[64]) {
	static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the handle travels as 64 bytes");
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	cudaIpcMemHandle_t handle;
	VKR_CUDA_OK(cudaIpcGetMemHandle(&handle, e->d_block), "Failed to export the frame of this GPU to the other processes");
	memcpy(out_handle, &handle, 64);
	return 0;
}

extern "C" int vkr_frame_exchange_connect(vkr_frame_exchange_t* e, const vkr_device_t* device, const unsigned char* handles) {
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	for (uint32_t r = 0; r != e->world; ++r) {
		if (r == e->rank) continue;
		cudaIpcMemHandle_t handle; memcpy(&handle, handles + 64 * (size_t) r, 64);
		void* mapped = nullptr;
		cudaError_t err = cudaIpcOpenMemHandle(&mapped, handle, cudaIpcMemLazyEnablePeerAccess);
		if (err != cudaSuccess) {
			printf("Failed to map the frame of rank %u into the process of rank %u (no peer access between the GPUs?): %s\n", r, e->rank, cudaGetErrorString(err));
			return 1;
		}
		e->d_peer_blocks[r] = mapped; e->peer_is_ipc[r] = 1;
	}
	return 0;
}

extern "C" int vkr_frame_exchange_connect_local(vkr_frame_exchange_t* e, const vkr_device_t* device, void* const* d_blocks) {
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	for (uint32_t r = 0; r != e->world; ++r) {
		if (r == e->rank) continue;
		cudaPointerAttributes attributes;
		VKR_CUDA_OK(cudaPointerGetAttributes(&attributes, d_blocks[r]), "Failed to find the GPU of a peer frame");
		if (attributes.device != device->cuda_device) {
			int can = 0;
			cudaDeviceCanAccessPeer(&can, device->cuda_device, attributes.device);
			cudaError_t err = can ? cudaDeviceEnablePeerAccess(attributes.device, 0) : cudaErrorPeerAccessUnsupported;
			if (err == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); err = cudaSuccess; }
			if (err != cudaSuccess) { printf("CUDA device %d cannot write to the memory of CUDA device %d: %s\n", device->cuda_device, attributes.device, cudaGetErrorString(err)); return 1; }
		}
		e->d_peer_blocks[r] = d_blocks[r]; e->peer_is_ipc[r] = 0;
	}
	return 0;
}

extern "C" void* vkr_frame_exchange_frame(const vkr_frame_exchange_t* e) {
	if (!e->d_block) return nullptr;
	const uint64_t last = e->frames_exchanged ? e->frames_exchanged - 1 : 0;
	return (char*) e->d_block + frame_bytes(e) * (last & 1);
}

static int exchange_ready(const vkr_shading_pass_t* pass, const vkr_frame_exchange_t* e) {
	const vkr_shading_pass_desc_t& d = pass->desc;
	if (!e->d_block || d.width != e->width || d.height != e->height || d.stripe_index != e->rank || d.stripe_count != e->world) {
		printf("The frame exchange (%ux%u, rank %u of %u) does not match the shading pass (%ux%u, share %u of %u).\n", e->width, e->height, e->rank, e->world, d.width, d.height, d.stripe_index, d.stripe_count);
		return 0;
	}
	for (uint32_t r = 0; r != e->world; ++r)
		if (!e->d_peer_blocks[r]) { printf("The frame exchange of rank %u is not connected to rank %u.\n", e->rank, r); return 0; }
	return 1;
}

extern "C" int vkr_shading_pass_run_exchange(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const void* d_gbuffer, vkr_frame_exchange_t* e) {
	if (!exchange_ready(pass, e)) return 1;
	cudaStream_t stream = (cudaStream_t) device->stream;
	const uint64_t frame = e->frames_exchanged + 1;       // counters hold the number of the last frame written, starting at 1
	const size_t buffer = frame_bytes(e) * ((frame - 1) & 1);
	void* peers[VKR_MAX_GPUS]; int peer_count = 0;
	peer_counters counters; memset(&counters, 0, sizeof(counters));
	for (uint32_t r = 0; r != e->world; ++r) {
		counters.p[r] = counters_of(e, e->d_peer_blocks[r]);
		if (r != e->rank) peers[peer_count++] = (char*) e->d_peer_blocks[r] + buffer;
	}
	if (vkr_launch_shading(pass, device, constants, constants_size, d_gbuffer, (char*) e->d_block + buffer, nullptr, peer_count, peers)) return 1;
	if (e->world > 1) {
		exchange_signal_kernel<<<1, 32, 0, stream>>>(counters, (int) e->world, (int) e->rank, (unsigned long long) frame);
		int* d_status = nullptr;
		VKR_CUDA_OK(cudaHostGetDevicePointer((void**) &d_status, e->h_status, 0), "Failed to map the status word of the frame exchange");
		exchange_wait_kernel<<<1, 32, 0, stream>>>(counters_of(e, e->d_block), (int) e->world, (int) e->rank, (unsigned long long) frame, (unsigned long long) e->timeout_ns, d_status);
		VKR_CUDA_OK(cudaGetLastError(), "Failed to launch the barrier of the frame exchange");
	}
	e->frames_exchanged = frame;
	return 0;
}

extern "C" int vkr_frame_exchange_download(vkr_frame_exchange_t* e, const vkr_device_t* device, float* out_rgba32f) {
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	VKR_CUDA_OK(cudaMemcpyAsync(out_rgba32f, vkr_frame_exchange_frame(e), frame_bytes(e), cudaMemcpyDeviceToHost, (cudaStream_t) device->stream), "Failed to download the frame");
	return vkr_frame_exchange_wait(e, device);
}

extern "C" int vkr_frame_exchange_wait(vkr_frame_exchange_t* e, const vkr_device_t* device) {
	VKR_CUDA_OK(cudaStreamSynchronize((cudaStream_t) device->stream), "Failed to wait for the frame exchange");
	if (e->h_status && *e->h_status) { printf("Frame exchange: rank %d did not deliver frame %llu to rank %u in time.\n", *e->h_status - 1, (unsigned long long) e->frames_exchanged, e->rank); return 1; }
	return 0;
}

extern "C" int vkr_shading_pass_run_host_exchange(vkr_shading_pass_t* pass, const vkr_device_t* device, const void* constants, size_t constants_size, const float* gbuffer,
	vkr_frame_exchange_t* e, float* out_rgba32f)
{
	if (!exchange_ready(pass, e)) return 1;
	const vkr_shading_pass_desc_t& d = pass->desc;
	cudaStream_t stream = (cudaStream_t) device->stream;
	VKR_CUDA_OK(cudaSetDevice(device->cuda_device), "Failed to select the CUDA device");
	const size_t plane_bytes = frame_bytes(e);
	if (!pass->d_gbuffer_staging && cudaMalloc(&pass->d_gbuffer_staging, 4 * plane_bytes) != cudaSuccess) { printf("Failed to allocate the device staging buffer of the G-buffer.\n"); return 1; }
	for (int k = 0; k != 4; ++k)
		if (vkr_copy_tile_columns(d, (char*) pass->d_gbuffer_staging + k * plane_bytes, (const char*) gbuffer + k * plane_bytes, 16, cudaMemcpyHostToDevice, stream)) { printf("Failed to upload the G-buffer.\n"); return 1; }
	if (vkr_shading_pass_run_exchange(pass, device, constants, constants_size, pass->d_gbuffer_staging, e)) return 1;
	if (out_rgba32f) VKR_CUDA_OK(cudaMemcpyAsync(out_rgba32f, vkr_frame_exchange_frame(e), plane_bytes, cudaMemcpyDeviceToHost, stream), "Failed to download the frame");
	if (vkr_frame_exchange_wait(e, device)) return 1;
	return vkr_shading_pass_wait(pass, device);
}
