#!/bin/bash
# Builds libmagvit2_b200.so in-tree for sm_90a (H100; cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=../libmagvit2_b200.so
SRCS="simt_ops.cu"
SRCS="$SRCS tc_conv.cu tc_slab.cu"
$NVCC -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
  -Xcompiler -fPIC -shared -Xptxas -v \
  -o $OUT $SRCS 2> build.log || { grep -E "error|fatal" -A3 build.log | head -40; exit 1; }
grep -E "error|warning: v|spill" build.log | grep -v "0 bytes spill" | head -20 || true
echo "built $(realpath $OUT)"
