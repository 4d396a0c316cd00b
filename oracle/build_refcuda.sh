#!/bin/bash
# Builds oracle/_ref/libmsda_refcuda.so: the reference's own MSDeformAttn CUDA kernels for sm_90a, compiled from the
# sources where they lie in a reference checkout ($UNINEXT_REFERENCE, default /root/reference; a GPU machine without one
# uses the prebuilt .so of a built tree, which is git-ignored).  Not the reference's build system: one nvcc command.
set -e
HERE=$(cd "$(dirname "$0")" && pwd)
REF=${UNINEXT_REFERENCE:-/root/reference}/projects/UNINEXT/uninext/models/deformable_detr/ops/src
[ -d "$REF" ] || { echo "no reference checkout here: keeping prebuilt oracle/_ref (if any)"; exit 0; }
TORCH_INC=$("${PYTHON:-python3}" -c "import torch.utils.cpp_extension as c; print(' '.join('-I'+p for p in c.include_paths()))")
mkdir -p "$HERE/_ref"
"${NVCC:-$(command -v nvcc || echo /usr/local/cuda/bin/nvcc)}" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo --shared -Xcompiler -fPIC \
     -I "$REF" $TORCH_INC -o "$HERE/_ref/libmsda_refcuda.so" "$HERE/refcuda_wrapper.cu"
echo "built $HERE/_ref/libmsda_refcuda.so"
