#!/bin/bash
# Build A/B variants of the LZ and Cascaded decode kernels (compile-time switches, e.g. -DLZ_DEC_CTAS=6) for one GPU call:
#   bash tools/build_variants.sh "name1:-DX=1 -DY=2" "name2:..."   -> build/variants/<name>/libnvcomp.so
# tools/ab_bench.sh runs the per-dataset benchmark with each of them on the GPU box.
set -eu
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -Iinclude -Invcomp_b200/csrc"
make -s nvcomp_b200/lib/libnvcomp.so
for spec in "$@"; do
  name=${spec%%:*}; defs=${spec#*:}
  d=build/variants/$name; mkdir -p $d
  for f in lz4 snappy cascaded; do
    /usr/local/cuda/bin/nvcc $FLAGS $defs -Xptxas -v -c nvcomp_b200/csrc/$f.cu -o $d/$f.o 2> $d/$f.ptxas.log
  done
  others=$(ls build/*.o | grep -v -e /lz4.o -e /snappy.o -e /cascaded.o)
  /usr/local/cuda/bin/nvcc $ARCH -shared -o $d/libnvcomp.so $d/lz4.o $d/snappy.o $d/cascaded.o $others -cudart static
  for k in snappy_decompress_v2 snappy_decompress_light lz4_decompress_v2 lz4_decompress_light cascaded_decompress; do
    echo "$name $k: $(grep -h -A2 "${k}_kernel" $d/*.ptxas.log | grep -E "registers|spill" | tr -s ' ' | tr '\n' ' ')"
  done
done
