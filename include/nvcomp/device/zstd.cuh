// nvcomp/device/zstd.cuh -- warp-level Zstandard (RFC 8878) decompression inside a user's own kernels.
//
// This is this library's own interface.  decompress_warp returns, for every chunk and capacity, the status, size and
// bytes that nvcompBatchedZstdDecompressAsync (nvcomp/zstd.h) returns: a chunk is zero or more Zstandard and
// skippable frames, back to back, as libzstd's one-shot ZSTD_decompress reads it.  It runs the batched kernel's own
// code (detail/zstd_decode.cuh).  There is no Zstd compression.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of decompress_warp and decompressed_size_warp: as in nvcomp/device/lz4.cuh --
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual is written once (by lane 0; the pointer may be null).
//   - Compressed streams and outputs are global memory and must not overlap.  Any alignment is accepted.
//   - `smem` is this warp's own shared-memory region of kDecompressSmemBytes bytes, aligned to kSmemAlignment.  It
//     holds nothing between calls: every call builds the predefined FSE tables and the code info tables in the
//     region's tail (the batched kernel builds them once per CTA).  Every return passes a __syncwarp.
//   - decompress_warp writes only inside [out, out + capacity).  A successful decode writes exactly *actual bytes.
//   - A content checksum mismatch (or a truncated checksum) returns nvcompErrorBadChecksum, any other chunk that
//     cannot be decoded (malformed, larger than capacity, or comp_bytes or capacity of 2^32 or more)
//     nvcompErrorCannotDecompress; both with *actual = 0.  No input causes an out-of-bounds access.
//   - Several warps of one CTA may run any mix of Deflate, Gzip and Zstd calls at once, each with its own region.
//     No call uses global scratch memory.
#pragma once

#include "nvcomp/shared_types.h"
#include "nvcomp/zstd.h"
#include "nvcomp/device/detail/zstd_decode.cuh"

namespace nvcomp {
namespace device {
namespace zstd {

// Alignment of each warp's shared-memory region.
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decoding warp: the decoder's Huffman and FSE tables and scratch (15 872 bytes), then the
// predefined FSE tables and the literal-length / match-length code info (1 024 bytes).
constexpr size_t kDecompressSmemBytes = detail::kZsWarpSmem + detail::kZsPreSmem;

static_assert(kDecompressSmemBytes % kSmemAlignment == 0, "warp regions stay aligned");

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

}  // namespace zstd
}  // namespace device
}  // namespace nvcomp
