#!/bin/bash
# Rebuild dlrover_b200/csrc/libflashckpt.so for sm_90a (same flags as __graft_entry__.build()).
set -e
cd "$(dirname "$0")/../dlrover_b200/csrc"
${NVCC:-/usr/local/cuda/bin/nvcc} -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo \
  -Xcompiler -fPIC -shared "$@" -o libflashckpt.so flashckpt.cu -lpthread
