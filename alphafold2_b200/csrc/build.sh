#!/bin/bash
# Build libaf2b200.so for sm_90a (H100; cross-compiles without a GPU). Static cudart: no runtime dependency on torch's.
# usage: build.sh [output.so [extra nvcc flags...]]     (the extra form builds A/B variants with -D options)
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=${1:-libaf2b200.so}
shift || true
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xptxas -v \
  -Xcompiler -fPIC -shared -cudart static "$@" \
  -o "$OUT" api.cu 2> build.log || { cat build.log; exit 1; }
grep -E "error|warning: v|spill" build.log | grep -v " 0 bytes spill" | head -20 || true
echo "built $(pwd)/$OUT"
