// device_headers_link.cu -- a link check of the eight warp-level device headers (nvcomp/device/*.cuh).  The Makefile
// compiles this file twice, with LINK_TU=1 and LINK_TU=2, and links both objects into one library: once as plain
// objects (build/tests/libdevice_headers_link.so) and once with relocatable device code (-rdc=true,
// build/tests/libdevice_headers_link_rdc.so).  A header that defines a function with external, non-inline linkage
// makes one of the two links fail with a multiple definition.  Each translation unit calls every function of the
// Deflate, Gzip and Zstd headers, so their out-of-line functions are emitted in both.  tests/test_device_headers_link.py
// loads both libraries.
#include <cuda_runtime.h>

#include "nvcomp/device/ans.cuh"
#include "nvcomp/device/bitcomp.cuh"
#include "nvcomp/device/cascaded.cuh"
#include "nvcomp/device/deflate.cuh"
#include "nvcomp/device/gzip.cuh"
#include "nvcomp/device/lz4.cuh"
#include "nvcomp/device/snappy.cuh"
#include "nvcomp/device/zstd.cuh"

#ifndef LINK_TU
#error "compile with -DLINK_TU=1 or -DLINK_TU=2"
#endif
#define LINK_CAT2(a, b) a##b
#define LINK_CAT(a, b) LINK_CAT2(a, b)

// a kernel name of its own in each translation unit
__global__ void LINK_CAT(use_all_tu, LINK_TU)(const void* comp, size_t comp_bytes, void* out, size_t cap, size_t* sizes,
                                               int algo) {
  extern __shared__ __align__(16) unsigned char smem[];
  nvcompBatchedDeflateOpts_t o;
  o.algo = algo;
  nvcomp::device::deflate::compress_warp(comp, comp_bytes, out, sizes, o, smem);
  nvcomp::device::deflate::decompress_warp(comp, comp_bytes, out, cap, sizes + 1, smem);
  nvcomp::device::gzip::decompress_warp(comp, comp_bytes, out, cap, sizes + 2, smem);
  nvcomp::device::zstd::decompress_warp(comp, comp_bytes, out, cap, sizes + 3, smem);
  const size_t a = nvcomp::device::deflate::decompressed_size_warp(comp, comp_bytes, smem);
  const size_t b = nvcomp::device::gzip::decompressed_size_warp(comp, comp_bytes, smem);
  const size_t c = nvcomp::device::zstd::decompressed_size_warp(comp, comp_bytes, smem);
  if (threadIdx.x == 0) sizes[4] = a + b + c;
}

// LINK_TU: which translation unit this symbol came from
extern "C" int LINK_CAT(device_headers_link_tu, LINK_TU)() { return LINK_TU; }
