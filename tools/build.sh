#!/bin/bash
# Build libbffc.so in-tree for sm_90a (same command __graft_entry__.build() runs).
set -e
cd "$(dirname "$0")/../flash-fft-conv_b200/csrc"
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -shared -Xcompiler -fPIC \
  -I ../../include -o ../libbffc.so bffc.cu "$@"
