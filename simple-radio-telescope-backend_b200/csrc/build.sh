#!/bin/bash
# Builds libsrtb_b200.so (sm_90a only) in-tree next to the sources.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo \
  -ccbin /usr/bin/g++ -Xcompiler -fPIC -Xcompiler -O2 --shared \
  ${SRTB_B200_PTXAS_V:+-Xptxas -v} \
  -o ${SRTB_B200_OUT:-libsrtb_b200.so} srtb_b200.cu -lcudart
echo "built $(pwd)/${SRTB_B200_OUT:-libsrtb_b200.so}"
