// nvcomp/device/lz4.cuh -- warp-level LZ4 compression and decompression inside a user's own kernels.
//
// This is this library's own interface.  The streams are the LZ4 blocks the batched C API (nvcomp/lz4.h) reads and
// writes: compress_warp writes byte for byte what nvcompBatchedLZ4CompressAsync writes for the chunk and data_type,
// and decompress_warp returns, for every chunk and capacity, the status, size and bytes that
// nvcompBatchedLZ4DecompressAsync returns.  Both run the batched kernels' own code (detail/lz77_compress.cuh,
// detail/lz4_encode.cuh, detail/lz4_decode.cuh): decompress_warp routes a chunk with the batched classifier's rule
// (lz_chunk_is_light) to the body the batched call would run for it, the direct sequence loop or the
// block-parallel decoder.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp, decompress_warp and decompressed_size_warp:
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - Compressed streams, inputs and outputs are global memory (the decoder stages compressed blocks with
//     cp.async.bulk from global memory).  Any alignment is accepted, as in the batched API, and the decoder reads
//     only what the batched decoder reads.
//   - `smem` is this warp's own shared-memory region, aligned to kSmemAlignment: kCompressSmemBytes for
//     compress_warp, kDecompressSmemBytes for decompress_warp.  Both are multiples of kSmemAlignment, so warp w of
//     a CTA can use smem_base + w * size.  The region holds nothing between calls: the caller may use it for
//     anything else in between.  decompress_warp initializes the region's mbarrier on entry, has no bulk copy in
//     flight on any return (failures included), invalidates the mbarrier (mbarrier.inval) before it returns, and
//     every return passes a __syncwarp.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n)).  A successful decode writes exactly *actual bytes.
//   - A chunk that cannot be decoded (malformed, or larger than capacity) returns nvcompErrorCannotDecompress with
//     *actual = 0; no input causes an out-of-bounds access.
//   - Several warps of one CTA may run any mix of LZ4 and Snappy (nvcomp/device/snappy.cuh) compression and
//     decompression at once, each with its own region.  No call uses global scratch memory.
#pragma once

#include "nvcomp/lz4.h"
#include "nvcomp/device/detail/lz4_decode.cuh"
#include "nvcomp/device/detail/lz4_encode.cuh"
#include "nvcomp/device/detail/lz_region.cuh"

namespace nvcomp {
namespace device {
namespace lz4 {

// Largest chunk compress_warp accepts (2^24 bytes).
constexpr size_t kMaxChunkBytes = nvcompLZ4CompressionMaxAllowedChunkSize;

// Alignment of each warp's shared-memory region (16-byte vector accesses and bulk-copy destinations).
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decompressing warp: the batched block decoder's per-warp region -- a 4 KB output ring, two
// 1 056-byte staging buffers, 1 KB of token records and a 16-byte mbarrier slot (7 248 bytes).
constexpr size_t kDecompressSmemBytes = lz::detail::kLzWarpSmem;

// Shared memory of one compressing warp: the matcher's hash table (4 096 16-bit entries, 8 KB).
constexpr size_t kCompressSmemBytes = lz::detail::kHashBytesPerWarp;

static_assert(kDecompressSmemBytes % kSmemAlignment == 0 && kCompressSmemBytes % kSmemAlignment == 0,
              "warp regions stay aligned");

// Upper bound of one compressed chunk of n bytes (LZ4_compressBound: n + n/255 + 16);
// nvcompBatchedLZ4CompressGetMaxOutputChunkSize returns the same.  0 for n > kMaxChunkBytes.
__host__ __device__ inline size_t max_compressed_bytes(size_t n) {
  return n > kMaxChunkBytes ? 0 : n + n / 255 + 16;
}

// Decompressed size of the LZ4 block at `comp` -- what nvcompBatchedLZ4GetDecompressSizeAsync reports for the chunk:
// the block carries no size header, so the warp walks its sequences without copying.  0 for a malformed block.
// Warp-collective (see above).
__device__ inline size_t decompressed_size_warp(const void* comp, size_t comp_bytes) {
  using namespace lz::detail;
  const int lane = lane_id();
  uint32_t produced = 0;
  bool ok = comp_bytes <= 0xffffffffull;
  if (ok) ok = lz4_walk_chunk((const uint8_t*)comp, (uint32_t)comp_bytes, &produced, lane);
  __syncwarp();
  return ok ? (size_t)produced : 0;
}

// Decode the comp_bytes-byte LZ4 block at `comp` into [out, out + capacity) with `smem` (kDecompressSmemBytes
// bytes).  Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem) {
  using namespace lz::detail;
  const int lane = lane_id();
  const uint8_t* in = (const uint8_t*)comp;
  uint8_t* o = (uint8_t*)out;
  const uint32_t n = (uint32_t)comp_bytes;   // lz_decompress_in_region calls these only for comp_bytes < 2^32
  return lz_decompress_in_region(
      comp_bytes, capacity, actual, smem,
      [&](uint32_t* produced) { return lz4_decode_chunk_direct(in, n, o, (uint64_t)capacity, produced, lane); },
      [&](uint32_t* produced, uint8_t* ring, uint32_t& parity) {
        return lz4_decode_chunk_v2(in, n, o, (uint64_t)capacity, produced, ring, parity, lane, false);
      });
}

// Compress the n_bytes bytes at `in` into the LZ4 block at `out` (max_compressed_bytes(n_bytes) bytes) and its size
// into *comp_bytes, with `smem` (kCompressSmemBytes bytes) as the hash table.  opts.data_type sets the matcher's
// candidate stride as in the batched call.  Warp-collective (see above).  A data_type the batched call rejects
// returns nvcompErrorInvalidValue, n_bytes > kMaxChunkBytes returns nvcompErrorChunkSizeTooLarge; both with
// *comp_bytes = 0 and nothing else written.
__device__ inline nvcompStatus_t compress_warp(const void* in, size_t n_bytes, void* out, size_t* comp_bytes,
                                               nvcompBatchedLZ4Opts_t opts, void* smem) {
  using namespace lz::detail;
  const int lane = lane_id();
  bool type_ok;
  const uint32_t step = lz4_step_for(opts.data_type, &type_ok);
  nvcompStatus_t st = nvcompSuccess;
  if (!type_ok) st = nvcompErrorInvalidValue;
  else if (n_bytes > kMaxChunkBytes) st = nvcompErrorChunkSizeTooLarge;
  if (st != nvcompSuccess) {
    if (lane == 0 && comp_bytes) *comp_bytes = 0;
    __syncwarp();
    return st;
  }
  Lz4Emitter em{(uint8_t*)out, 0};
  lz4_compress_chunk((const uint8_t*)in, (uint32_t)n_bytes, em, (uint16_t*)smem, step, lane);
  if (lane == 0 && comp_bytes) *comp_bytes = em.op;
  __syncwarp();
  return nvcompSuccess;
}

}  // namespace lz4
}  // namespace device
}  // namespace nvcomp
