#!/bin/bash
# Compile the reference's own benchmarks/examples UNCHANGED (sources stay in the nvCOMP tree, nothing is copied)
# against this library's headers and libnvcomp.so -> oracle/_ref/.  Acceptance harness for the drop-in boundary
# (SURVEY.md 2a: "must compile & link unchanged"); tests/test_reference_harness_gpu.py runs the binaries.
#   oracle/build_reference_harness.sh [NVCOMP_TREE]
# The nvCOMP tree is the first argument, else $NVCOMP_REFERENCE_DIR, else /root/reference (the documented default
# location, so that build() finds it without configuration).  No-op when the tree is absent.  Binaries find libnvcomp.so through an $ORIGIN-relative rpath, so the repository
# can be moved or copied after the build.
set -u
R=${1:-${NVCOMP_REFERENCE_DIR:-/root/reference}}
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
[ -d "$R/benchmarks" ] || { echo "reference tree not found at $R: skipping"; exit 0; }
OUT="$ROOT/oracle/_ref"
mkdir -p "$OUT/bin"
cd "$OUT/bin"
LIB="$ROOT/nvcomp_b200/lib/libnvcomp.so"
NV="nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -O2 -w -DTHRUST_CUB_WRAPPED_NAMESPACE=nvcomp \
  -I$ROOT/include -I$R/benchmarks -L$ROOT/nvcomp_b200/lib -lnvcomp"
build() { # name source
  if [ ! -x "$1" ] || [ "$2" -nt "$1" ] || [ "$LIB" -nt "$1" ]; then
    $NV -Xlinker '-rpath=$ORIGIN/../../../nvcomp_b200/lib' -x cu "$2" -o "$1" > "$1.log" 2>&1 || { echo "FAILED: $1 (see oracle/_ref/bin/$1.log)"; return 1; }
  fi
}
for f in lz4 snappy cascaded bitcomp ans gdeflate deflate zstd; do build benchmark_${f}_chunked $R/benchmarks/benchmark_${f}_chunked.cu & done
for f in benchmark_snappy_synth benchmark_lz4_synth benchmark_hlif; do build $f $R/benchmarks/$f.cpp & done
for f in low_level_quickstart_example high_level_quickstart_example; do build $f $R/examples/$f.cpp & done
# the LZ4 CPU-interop examples (known-answer tests of the wire format): liblz4.so.1 is installed, its header may not
# be -> prototype-only shim in tests/shim/
NV="$NV -I$ROOT/tests/shim -I$R/examples -l:liblz4.so.1"
for f in lz4_cpu_compression lz4_cpu_decompression; do build $f $R/examples/$f.cu & done
wait
# the reference's OWN CMake build against cmake/nvcomp-config.cmake (two of its targets are enough to prove it)
if command -v cmake > /dev/null; then
  cmake -S "$R" -B "$OUT/cmake" -Dnvcomp_DIR="$ROOT/cmake" -DBUILD_BENCHMARKS=ON -DCMAKE_CUDA_ARCHITECTURES=90a \
    -DCMAKE_BUILD_RPATH_USE_ORIGIN=ON -DCMAKE_BUILD_RPATH='$ORIGIN/../../../../nvcomp_b200/lib' \
    > "$OUT/cmake.log" 2>&1 &&
    cmake --build "$OUT/cmake" -j8 --target low_level_quickstart_example benchmark_snappy_synth >> "$OUT/cmake.log" 2>&1 ||
    echo "FAILED: reference CMake build (see oracle/_ref/cmake.log)"
fi
ls -1 | grep -v '\.log$' | wc -l
