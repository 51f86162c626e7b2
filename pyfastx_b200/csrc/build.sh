#!/usr/bin/env bash
# Build libfxg.so (C-ABI + sm_90a kernels) in-tree: pyfastx_b200/libfxg.so
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="${FXG_OUT:-$HERE/../libfxg.so}"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"$NVCC" -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
    -Xcompiler -fPIC,-O2,-Wall -Xptxas -v --shared ${FXG_DEFS:-} \
    "$HERE/fxg_api.cu" "$HERE/fxg_scan.cu" "$HERE/fxg_extract.cu" "$HERE/fxg_synth.cu" "$HERE/fxg_inflate.cu" "$HERE/fxg_comm.cu" "$HERE/fxg_stats.cu" "$HERE/fxg_search.cu" "$HERE/fxg_fxi.cpp" "$HERE/fxg_names.cpp" "$HERE/fxg_gzip.cpp" \
    -o "$OUT" -lcudart -ldl -lz 2> "$HERE/build.log" || { cat "$HERE/build.log"; exit 1; }
grep -E "error|warning: v|registers|spill" "$HERE/build.log" | grep -v "0 bytes spill" | head -40 || true
echo "built $OUT"
