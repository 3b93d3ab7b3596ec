#!/bin/bash
# Developer tool for tuning experiments: builds the library with extra -D flags for the quad-light shading kernels (light vertex bound 4) only; the other
# kernel families are stubs (tools/variant_stubs.cu), everything else comes from the in-tree objects.
#   tools/build_variant.sh <name> "<nvcc flags>"   ->  vulkan_renderer_b200/variants/libvkr_<name>.so
# Select it with VKR_B200_LIB=<path> (tools/quick_time.py only; tests and bench always load the in-tree libvkr_b200.so).
set -e
cd "$(dirname "$0")/.."
name=$1; flags=$2
out=vulkan_renderer_b200/variants; mkdir -p $out
common="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -fmad=false -prec-div=true -prec-sqrt=true -ftz=false -ccbin /usr/bin/g++ -Xcompiler -fPIC -I include"
nvcc $common -DVKR_MAXV_TU=4 $flags -c vulkan_renderer_b200/csrc/vkr_shading_kernel.cu -o $out/$name.o
nvcc $common -DVKR_MAXV_TU=4 -DVKR_TRACE_STATS=1 $flags -c vulkan_renderer_b200/csrc/vkr_shading_kernel.cu -o $out/${name}_stats.o
[ $out/stubs.o -nt tools/variant_stubs.cu ] || nvcc $common -c tools/variant_stubs.cu -o $out/stubs.o
b=vulkan_renderer_b200/build
others=$(ls $b/*.o | grep -v "vkr_shading_kernel_\|vkr_textured_\|vkr_related_work_")
nvcc -shared -o $out/libvkr_$name.so $out/$name.o $out/${name}_stats.o $out/stubs.o $others -ccbin /usr/bin/g++ -Xcompiler -fopenmp -lgomp -cudart static
rm $out/$name.o $out/${name}_stats.o
echo built $out/libvkr_$name.so
