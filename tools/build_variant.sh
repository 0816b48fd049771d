#!/bin/bash
# Build a variant of the CUDA library for A/B runs (tools/dev_ab.py):  tools/build_variant.sh NAME [-DFLAG ...]
# -> tools/_timing/lib_NAME.so, always with -DBLANCE_SPEC_TIMING (leader cycle counters).
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p tools/_timing
${NVCC:-/usr/local/cuda/bin/nvcc} -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -fmad=false \
  -Xcompiler -fPIC -shared -cudart static -DBLANCE_SPEC_TIMING "$@" -Iinclude -Iblance_b200/csrc \
  blance_b200/csrc/c_abi.cu -o tools/_timing/lib_$name.so
