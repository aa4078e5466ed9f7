#!/usr/bin/env bash
# Build the C-ABI CUDA library for sm_90a (cross-compiles without a GPU).
set -euo pipefail
cd "$(dirname "$0")/.."
mkdir -p linetr_b200/lib
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
  -Xcompiler -fPIC,-Wall,-Wno-unused-function -shared ${LTR_NVCC_EXTRA:-} \
  -o linetr_b200/lib/liblinetr_b200.so.tmp linetr_b200/csrc/ltr_api.cu -lcudart
mv -f linetr_b200/lib/liblinetr_b200.so.tmp linetr_b200/lib/liblinetr_b200.so   # atomic: a snapshot never sees a half-written library
echo "built linetr_b200/lib/liblinetr_b200.so"
