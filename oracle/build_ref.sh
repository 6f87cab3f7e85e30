#!/bin/bash
# Compiles the reference's own CUDA correlation kernels (Nets/Native/shift_corr.cu.cc) for sm_90a,
# unmodified and in place, into oracle/_ref/libref_shift_corr.so.  Two TensorFlow headers are stubbed:
# an empty Eigen Tensor header and cuda_kernel_helper.h providing only CUDA_1D_KERNEL_LOOP.
# No reference source is copied into the repository; outputs go to oracle/_ref/ only (git-ignored).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${REF:-/root/reference}
SRC="$REF/Nets/Native/shift_corr.cu.cc"
OUT="$HERE/_ref"
if [ ! -f "$SRC" ]; then echo "reference not present ($SRC); keeping any prebuilt $OUT"; exit 0; fi
mkdir -p "$OUT/stubs/third_party/eigen3/unsupported/Eigen/CXX11" "$OUT/stubs/tensorflow/core/util"
: > "$OUT/stubs/third_party/eigen3/unsupported/Eigen/CXX11/Tensor"
cat > "$OUT/stubs/tensorflow/core/util/cuda_kernel_helper.h" <<'H'
#pragma once
#define CUDA_1D_KERNEL_LOOP(i, n) \
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += blockDim.x * gridDim.x)
H
nvcc -std=c++14 -O2 -gencode arch=compute_90a,code=sm_90a -DGOOGLE_CUDA=1 -I "$OUT/stubs" -x cu \
     -Xcompiler -fPIC -c "$SRC" -o "$OUT/shift_corr.o"
nvcc -std=c++14 -O2 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -c "$HERE/ref_corr_wrapper.cu" -o "$OUT/wrapper.o"
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o "$OUT/libref_shift_corr.so" "$OUT/shift_corr.o" "$OUT/wrapper.o" -lcudart
echo "built $OUT/libref_shift_corr.so"
