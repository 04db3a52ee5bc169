#!/bin/bash
# Builds variants/<name>.so with build-time knobs (they travel to the GPU box with gpurun; variants/ is git-ignored), so that one
# GPU call can A/B them: SSE_LIB=variants/<name>.so python bench.py ...
# usage: tools/build_variants.sh name1 "-DSSE_X=1 ..." name2 "..." ...
set -e
cd "$(dirname "$0")/.."
mkdir -p variants
while [ $# -ge 2 ]; do
  name=$1; defs=$2; shift 2
  ( cd inference_gateway_b200/csrc && nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O2 -shared -cudart static \
      $defs -o ../../variants/$name.so sse_fused.cu sse_kernel.cu sse_kernel2.cu sse_long.cu sse_host.cu sse_fold.cpp sse_gateway.cpp ) &
done
wait
ls -la variants/
