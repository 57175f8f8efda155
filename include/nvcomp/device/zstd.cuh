// nvcomp/device/zstd.cuh -- warp-level Zstandard (RFC 8878) compression and decompression inside a user's own kernels.
//
// This is this library's own interface.  decompress_warp returns, for every chunk and capacity, the status, size and
// bytes that nvcompBatchedZstdDecompressAsync (nvcomp/zstd.h) returns: a chunk is zero or more Zstandard and
// skippable frames, back to back, as libzstd's one-shot ZSTD_decompress reads it.  It runs the batched kernel's own
// code (detail/zstd_decode.cuh).  compress_warp writes one frame per chunk of up to 64 KB (detail/zstd_encode.cuh
// states its stream rules) that libzstd and decompress_warp read; the batched nvcompBatchedZstdCompress* entry points
// still return nvcompErrorNotSupported.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp, decompress_warp and decompressed_size_warp: as in nvcomp/device/lz4.cuh --
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - Compressed streams, inputs and outputs are global memory and must not overlap.  Any alignment is accepted.
//   - `smem` is this warp's own shared-memory region of kDecompressSmemBytes bytes, aligned to kSmemAlignment.  It
//     holds nothing between calls: every call builds the predefined FSE tables and the code info tables in the
//     region's tail (the batched kernel builds them once per CTA).  Every return passes a __syncwarp.
//   - compress_warp's region is kCompressSmemBytes bytes and also holds nothing between calls.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n)).  A successful decode writes exactly *actual bytes.
//   - A content checksum mismatch (or a truncated checksum) returns nvcompErrorBadChecksum, any other chunk that
//     cannot be decoded (malformed, larger than capacity, or comp_bytes or capacity of 2^32 or more)
//     nvcompErrorCannotDecompress; both with *actual = 0.  No input causes an out-of-bounds access.
//   - Several warps of one CTA may run any mix of Deflate, Gzip and Zstd calls at once, each with its own region.
//     No call uses global scratch memory.
#pragma once

#include "nvcomp/shared_types.h"
#include "nvcomp/zstd.h"
#include "nvcomp/device/detail/zstd_decode.cuh"
#include "nvcomp/device/detail/zstd_encode.cuh"

namespace nvcomp {
namespace device {
namespace zstd {

// Alignment of each warp's shared-memory region.
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decoding warp: the decoder's Huffman and FSE tables and scratch (15 872 bytes), then the
// predefined FSE tables and the literal-length / match-length code info (1 024 bytes).
constexpr size_t kDecompressSmemBytes = detail::kZsWarpSmem + detail::kZsPreSmem;

// Largest chunk compress_warp accepts (64 KB).
constexpr size_t kMaxCompressChunkBytes = nvcompZstdCompressionMaxAllowedChunkSize;

// Shared memory of one compressing warp: the matcher's hash table (8 KB), one block's literals and sequence records
// (24 KB), the Huffman and FSE workspace, the predefined tables and the staging window (47 376 bytes, so four
// compressing warps fit on an SM).
constexpr size_t kCompressSmemBytes = detail::kZstdEncWarpSmem;

static_assert(kDecompressSmemBytes % kSmemAlignment == 0 && kCompressSmemBytes % kSmemAlignment == 0,
              "warp regions stay aligned");
static_assert(kMaxCompressChunkBytes == detail::kZstdMaxCompressChunk, "one chunk limit");

// Upper bound of one compressed chunk of n bytes: the all-Raw frame, header (6 or 7 bytes) + n + 3 bytes per 16 KB
// block; never above libzstd's ZSTD_compressBound(n).  0 for n > kMaxCompressChunkBytes.
__host__ __device__ inline size_t max_compressed_bytes(size_t n) {
  return n > kMaxCompressChunkBytes ? 0 : (size_t)detail::zstd_enc_bound((uint32_t)n);
}

namespace detail {

// zstd_chunk<kCount> as the batched zstd_kernel calls it, with this warp's tables at the head of `smem` and the
// predefined tables, built by this call, in its tail.  A chunk or capacity of 2^32 bytes or more is rejected, as in the
// batched kernel.  Returns a ZstdResult and *produced; every lane is past the closing __syncwarp.
template <bool kCount>
__device__ __forceinline__ int zstd_in_region(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                              uint32_t* produced, void* smem) {
  const int lane = lz::detail::lane_id();
  const uint32_t base = lz::detail::smem_addr(smem);
  const ZstdWarp ws{base, base + kZsWarpSmem};
  zstd_build_predefined(ws.predef, ws.smem, lane);
  *produced = 0;
  int r = kZstdBad;
  if (comp_bytes <= 0xffffffffull && capacity <= 0xffffffffull)
    r = zstd_chunk<kCount>((const uint8_t*)comp, (uint32_t)comp_bytes, (uint8_t*)out, (uint32_t)capacity, produced,
                           ws, lane);
  __syncwarp();
  return r;
}

}  // namespace detail

// Decompressed size of the Zstd chunk at `comp` -- what nvcompBatchedZstdGetDecompressSizeAsync reports for the
// chunk: the warp walks every frame without writing (content checksums are not checked).  0 for a chunk it rejects.
// `smem`: kDecompressSmemBytes bytes.  Warp-collective (see above).
__device__ inline size_t decompressed_size_warp(const void* comp, size_t comp_bytes, void* smem) {
  uint32_t produced = 0;
  const int r = detail::zstd_in_region<true>(comp, comp_bytes, nullptr, 0xffffffffull, &produced, smem);
  return r == detail::kZstdOk ? (size_t)produced : 0;
}

// Decode the comp_bytes-byte Zstd chunk at `comp` into [out, out + capacity) with `smem` (kDecompressSmemBytes
// bytes).  Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem) {
  uint32_t produced = 0;
  const int r = detail::zstd_in_region<false>(comp, comp_bytes, out, capacity, &produced, smem);
  if (lz::detail::lane_id() == 0 && actual) *actual = r == detail::kZstdOk ? (size_t)produced : 0;
  __syncwarp();
  return r == detail::kZstdOk ? nvcompSuccess
         : r == detail::kZstdBadChecksum ? nvcompErrorBadChecksum : nvcompErrorCannotDecompress;
}

// Compress the n_bytes bytes at `in` into one Zstandard frame at `out` (max_compressed_bytes(n_bytes) bytes) and its
// size into *comp_bytes, with `smem` (kCompressSmemBytes bytes).  opts.algo must be 0 (the one parse); any other
// value returns nvcompErrorInvalidValue, n_bytes > kMaxCompressChunkBytes returns nvcompErrorChunkSizeTooLarge; both
// with *comp_bytes = 0 and nothing else written.  Warp-collective (see above).
__device__ inline nvcompStatus_t compress_warp(const void* in, size_t n_bytes, void* out, size_t* comp_bytes,
                                               nvcompBatchedZstdOpts_t opts, void* smem) {
  const int lane = lz::detail::lane_id();
  nvcompStatus_t st = nvcompSuccess;
  if (opts.algo != 0) st = nvcompErrorInvalidValue;
  else if (n_bytes > kMaxCompressChunkBytes) st = nvcompErrorChunkSizeTooLarge;
  uint32_t produced = 0;
  if (st == nvcompSuccess)
    produced = detail::zstd_compress_chunk((const uint8_t*)in, (uint32_t)n_bytes, (uint8_t*)out, (uint8_t*)smem, lane);
  if (lane == 0 && comp_bytes) *comp_bytes = produced;
  __syncwarp();
  return st;
}

}  // namespace zstd
}  // namespace device
}  // namespace nvcomp
