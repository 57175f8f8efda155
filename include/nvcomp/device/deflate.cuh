// nvcomp/device/deflate.cuh -- warp-level Deflate (RFC 1951) compression and decompression inside a user's own kernels.
//
// This is this library's own interface.  The streams are the raw Deflate streams the batched C API (nvcomp/deflate.h)
// reads and writes: compress_warp writes byte for byte what nvcompBatchedDeflateCompressAsync writes for the chunk and
// opts.algo, and decompress_warp returns, for every chunk and capacity, the status, size and bytes that
// nvcompBatchedDeflateDecompressAsync returns.  Both run the batched kernels' own code (detail/deflate_compress.cuh,
// detail/inflate_decode.cuh).
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp, decompress_warp and decompressed_size_warp: as in nvcomp/device/lz4.cuh --
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - Compressed streams, inputs and outputs are global memory and must not overlap.  Any alignment is accepted, as
//     in the batched API.
//   - `smem` is this warp's own shared-memory region, aligned to kSmemAlignment: kDecompressSmemBytes for
//     decompress_warp and decompressed_size_warp, compress_smem_bytes(opts.algo) for compress_warp.  All are multiples
//     of kSmemAlignment, so warp w of a CTA can use smem_base + w * size.  The region holds nothing between calls
//     (the decoder's fixed-code tables are rebuilt by every call that needs them): the caller may use it for anything
//     else in between.  Every return passes a __syncwarp, so the warp can read what the call wrote right after it.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n)).  A successful decode writes exactly *actual bytes.
//   - A chunk that cannot be decoded (malformed, larger than capacity, or comp_bytes or capacity of 2^32 or more)
//     returns nvcompErrorCannotDecompress with *actual = 0; no input causes an out-of-bounds access.
//   - Several warps of one CTA may run any mix of Deflate, Gzip (nvcomp/device/gzip.cuh) and Zstd
//     (nvcomp/device/zstd.cuh) calls at once, each with its own region.  No call uses global scratch memory.
#pragma once

#include "nvcomp/deflate.h"
#include "nvcomp/device/detail/deflate_compress.cuh"
#include "nvcomp/device/detail/inflate_region.cuh"

namespace nvcomp {
namespace device {
namespace deflate {

// Largest chunk compress_warp accepts (64 KB).
constexpr size_t kMaxCompressChunkBytes = nvcompDeflateCompressionMaxAllowedChunkSize;

// Alignment of each warp's shared-memory region.
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decoding warp: the literal/length, distance and code-length decode tables, the fixed-code
// tables and the table builder's scratch (10 368 bytes).
constexpr size_t kDecompressSmemBytes = detail::kInfWarpSmem;

// Shared memory of one compressing warp for opts.algo = algo: the matcher's hash table, then the histograms, codes
// and output staging window -- 11 152 bytes for algos 0 and 2, 68 496 bytes for algo 1 (a 2^15-entry hash table).
// 0 for an algo compress_warp rejects.
__host__ __device__ constexpr size_t compress_smem_bytes(int algo) {
  return algo == 0 ? detail::kDeflateWarpSmem<0>
         : algo == 1 ? detail::kDeflateWarpSmem<1>
         : algo == 2 ? detail::kDeflateWarpSmem<2> : 0;
}

static_assert(kDecompressSmemBytes % kSmemAlignment == 0 && compress_smem_bytes(0) % kSmemAlignment == 0 &&
                  compress_smem_bytes(1) % kSmemAlignment == 0 && compress_smem_bytes(2) % kSmemAlignment == 0,
              "warp regions stay aligned");

// Upper bound of one compressed chunk of n bytes: the stored encoding, 5 header bytes per block of up to 65 535
// bytes; nvcompBatchedDeflateCompressGetMaxOutputChunkSize returns the same.  0 for n > kMaxCompressChunkBytes.
__host__ __device__ inline size_t max_compressed_bytes(size_t n) {
  return n > kMaxCompressChunkBytes ? 0 : n + 5 * (n / 65535 + 1);
}

// Decompressed size of the Deflate stream at `comp` -- what nvcompBatchedDeflateGetDecompressSizeAsync reports for
// the chunk: the stream carries no size header, so the warp walks it without writing.  0 for a malformed stream.
// `smem`: kDecompressSmemBytes bytes.  Warp-collective (see above).
__device__ inline size_t decompressed_size_warp(const void* comp, size_t comp_bytes, void* smem) {
  return detail::inflate_size_warp<false>(comp, comp_bytes, smem);
}

// Decode the comp_bytes-byte raw Deflate stream at `comp` into [out, out + capacity) with `smem`
// (kDecompressSmemBytes bytes).  Bytes after the end of the final block are not read.  Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem) {
  return detail::inflate_decompress_warp<false>(comp, comp_bytes, out, capacity, actual, smem);
}

// Compress the n_bytes bytes at `in` into one raw Deflate stream at `out` (max_compressed_bytes(n_bytes) bytes) and its
// size into *comp_bytes, with `smem` (compress_smem_bytes(opts.algo) bytes).  opts.algo selects the parse as in the
// batched call: 0 greedy, 1 greedy with a lazy step, 2 literals only.  Warp-collective (see above).  An algo outside
// 0-2 returns nvcompErrorInvalidValue, n_bytes > kMaxCompressChunkBytes returns nvcompErrorChunkSizeTooLarge; both
// with *comp_bytes = 0 and nothing else written.
__device__ inline nvcompStatus_t compress_warp(const void* in, size_t n_bytes, void* out, size_t* comp_bytes,
                                               nvcompBatchedDeflateOpts_t opts, void* smem) {
  using namespace detail;
  const int lane = lz::detail::lane_id();
  nvcompStatus_t st = nvcompSuccess;
  if (opts.algo < 0 || opts.algo > 2) st = nvcompErrorInvalidValue;
  else if (n_bytes > kMaxCompressChunkBytes) st = nvcompErrorChunkSizeTooLarge;
  uint32_t produced = 0;
  if (st == nvcompSuccess) {
    const uint8_t* i = (const uint8_t*)in;
    uint8_t* o = (uint8_t*)out;
    uint8_t* s = (uint8_t*)smem;
    const uint32_t n = (uint32_t)n_bytes;
    if (opts.algo == 0) produced = deflate_compress_chunk<0>(i, n, o, DeflateWarp::carve<0>(s), lane);
    else if (opts.algo == 1) produced = deflate_compress_chunk<1>(i, n, o, DeflateWarp::carve<1>(s), lane);
    else produced = deflate_compress_chunk<2>(i, n, o, DeflateWarp::carve<2>(s), lane);
  }
  if (lane == 0 && comp_bytes) *comp_bytes = produced;
  __syncwarp();
  return st;
}

}  // namespace deflate
}  // namespace device
}  // namespace nvcomp
