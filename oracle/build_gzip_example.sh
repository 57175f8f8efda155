#!/bin/bash
# Compile the reference's examples/gzip_gpu_decompression.cu UNCHANGED (the source stays in the nvCOMP tree, nothing is
# copied) against this library's headers and libnvcomp.so -> oracle/_ref/bin/gzip_gpu_decompression: zlib compresses
# 64 KB chunks on the host, this library's batched Gzip decoder decodes them, the example checks the bytes.
# tests/test_inflate_gpu.py runs it.  Same conventions as build_reference_harness.sh:
#   oracle/build_gzip_example.sh [NVCOMP_TREE]
# The nvCOMP tree is the first argument, else $NVCOMP_REFERENCE_DIR, else /root/reference.  No-op when the tree is
# absent.  zlib's header and libz are installed, so no shim is needed.
set -u
R=${1:-${NVCOMP_REFERENCE_DIR:-/root/reference}}
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
SRC="$R/examples/gzip_gpu_decompression.cu"
[ -f "$SRC" ] || { echo "reference example not found at $SRC: skipping"; exit 0; }
mkdir -p "$ROOT/oracle/_ref/bin"
cd "$ROOT/oracle/_ref/bin"
LIB="$ROOT/nvcomp_b200/lib/libnvcomp.so"
EXE=gzip_gpu_decompression
if [ ! -x "$EXE" ] || [ "$SRC" -nt "$EXE" ] || [ "$LIB" -nt "$EXE" ]; then
  nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -O2 -w -DTHRUST_CUB_WRAPPED_NAMESPACE=nvcomp \
    -I"$ROOT/include" -I"$R/examples" -L"$ROOT/nvcomp_b200/lib" -lnvcomp -lz \
    -Xlinker '-rpath=$ORIGIN/../../../nvcomp_b200/lib' -x cu "$SRC" -o "$EXE" > "$EXE.log" 2>&1 ||
    { echo "FAILED: $EXE (see oracle/_ref/bin/$EXE.log)"; exit 1; }
fi
