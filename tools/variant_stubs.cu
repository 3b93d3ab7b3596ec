// Developer tool (tools/build_variant.sh): tuning variants carry the quad-light benchmark kernels only; every other kernel family is a stub that refuses to launch,
// which keeps a variant library at a tenth of the size of the product library (they travel to the GPU box with every call).
#include "../vulkan_renderer_b200/csrc/vkr_kernels.h"
#define VKR_STUB(name) cudaError_t name(const vkr::shading_kernel_params&, cudaStream_t) { return cudaErrorNotSupported; }
VKR_STUB(vkr_launch_shading_kernel_v3) VKR_STUB(vkr_launch_shading_kernel_v5) VKR_STUB(vkr_launch_shading_kernel_v6) VKR_STUB(vkr_launch_shading_kernel_v7)
VKR_STUB(vkr_launch_textured_light_kernel_v3) VKR_STUB(vkr_launch_textured_light_kernel_v4) VKR_STUB(vkr_launch_textured_light_kernel_v5) VKR_STUB(vkr_launch_textured_light_kernel_v6) VKR_STUB(vkr_launch_textured_light_kernel_v7)
VKR_STUB(vkr_launch_textured_related_work_kernel_v3) VKR_STUB(vkr_launch_textured_related_work_kernel_v4) VKR_STUB(vkr_launch_textured_related_work_kernel_v5) VKR_STUB(vkr_launch_textured_related_work_kernel_v6) VKR_STUB(vkr_launch_textured_related_work_kernel_v7)
VKR_STUB(vkr_launch_related_work_kernel_v3) VKR_STUB(vkr_launch_related_work_kernel_v4) VKR_STUB(vkr_launch_related_work_kernel_v5) VKR_STUB(vkr_launch_related_work_kernel_v6) VKR_STUB(vkr_launch_related_work_kernel_v7)
