// nvcomp/device/snappy.cuh -- warp-level Snappy compression and decompression inside a user's own kernels.
//
// This is this library's own interface.  The streams are the raw Snappy streams the batched C API (nvcomp/snappy.h)
// reads and writes: compress_warp writes byte for byte what nvcompBatchedSnappyCompressAsync writes for the chunk,
// and decompress_warp returns, for every chunk and capacity, the status, size and bytes that
// nvcompBatchedSnappyDecompressAsync returns.  Both run the batched kernels' own code (detail/lz77_compress.cuh,
// detail/snappy_encode.cuh, detail/snappy_decode.cuh): decompress_warp routes a chunk with the batched classifier's
// rule (lz_chunk_is_light) to the body the batched call would run for it, the direct element loop or the
// block-parallel decoder.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp and decompress_warp: as in nvcomp/device/lz4.cuh --
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - Compressed streams, inputs and outputs are global memory; any alignment is accepted, and the decoder reads
//     only what the batched decoder reads.
//   - `smem` is this warp's own shared-memory region, aligned to kSmemAlignment: kCompressSmemBytes for
//     compress_warp, kDecompressSmemBytes for decompress_warp (multiples of kSmemAlignment).  The region holds
//     nothing between calls; decompress_warp initializes its mbarrier on entry, has no bulk copy in flight on any
//     return, invalidates the mbarrier before it returns, and every return passes a __syncwarp.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n)).  A successful decode writes exactly *actual bytes.
//   - A chunk that cannot be decoded returns nvcompErrorCannotDecompress with *actual = 0.
//   - Several warps of one CTA may run any mix of LZ4 and Snappy compression and decompression at once, each with
//     its own region.  No call uses global scratch memory.
#pragma once

#include "nvcomp/snappy.h"
#include "nvcomp/device/detail/snappy_decode.cuh"
#include "nvcomp/device/detail/snappy_encode.cuh"
#include "nvcomp/device/detail/lz_region.cuh"

namespace nvcomp {
namespace device {
namespace snappy {

// Largest chunk compress_warp accepts (2^24 bytes).
constexpr size_t kMaxChunkBytes = nvcompSnappyCompressionMaxAllowedChunkSize;

// Alignment of each warp's shared-memory region.
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decompressing warp: the batched block decoder's per-warp region (7 248 bytes).
constexpr size_t kDecompressSmemBytes = lz::detail::kLzWarpSmem;

// Shared memory of one compressing warp: the matcher's hash table (8 KB).
constexpr size_t kCompressSmemBytes = lz::detail::kHashBytesPerWarp;

static_assert(kDecompressSmemBytes % kSmemAlignment == 0 && kCompressSmemBytes % kSmemAlignment == 0,
              "warp regions stay aligned");

// Upper bound of one compressed chunk of n bytes (snappy::MaxCompressedLength: 32 + n + n/6);
// nvcompBatchedSnappyCompressGetMaxOutputChunkSize returns the same.  0 for n > kMaxChunkBytes.
__host__ __device__ inline size_t max_compressed_bytes(size_t n) {
  return n > kMaxChunkBytes ? 0 : 32 + n + n / 6;
}

// Uncompressed size in the varint preamble of `comp`, or 0 if the preamble is malformed -- what
// nvcompBatchedSnappyGetDecompressSizeAsync reports for the chunk.  Any thread may call it on its own.
__device__ inline size_t decompressed_size(const void* comp, size_t comp_bytes) {
  uint32_t ip = 0;
  uint64_t ulen = 0;
  const bool ok = comp_bytes <= 0xffffffffull &&
                  lz::detail::snappy_read_preamble((const uint8_t*)comp, (uint32_t)comp_bytes, ip, ulen);
  return ok ? (size_t)ulen : 0;
}

// Decode the comp_bytes-byte Snappy stream at `comp` into [out, out + capacity) with `smem` (kDecompressSmemBytes
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
      [&](uint32_t* produced) { return snappy_decode_chunk(in, n, o, (uint64_t)capacity, produced, lane); },
      [&](uint32_t* produced, uint8_t* ring, uint32_t& parity) {
        return snappy_decode_chunk_v2(in, n, o, (uint64_t)capacity, produced, ring, parity, lane, false);
      });
}

// Compress the n_bytes bytes at `in` into the Snappy stream at `out` (max_compressed_bytes(n_bytes) bytes) and its
// size into *comp_bytes, with `smem` (kCompressSmemBytes bytes) as the hash table.  The Snappy options are reserved,
// so there are none.  Warp-collective (see above).  n_bytes > kMaxChunkBytes returns nvcompErrorChunkSizeTooLarge
// with *comp_bytes = 0 and nothing else written.
__device__ inline nvcompStatus_t compress_warp(const void* in, size_t n_bytes, void* out, size_t* comp_bytes,
                                               void* smem) {
  using namespace lz::detail;
  const int lane = lane_id();
  if (n_bytes > kMaxChunkBytes) {
    if (lane == 0 && comp_bytes) *comp_bytes = 0;
    __syncwarp();
    return nvcompErrorChunkSizeTooLarge;
  }
  SnappyEmitter em{(uint8_t*)out, 0};
  em.begin((uint32_t)n_bytes, lane);
  snappy_compress_chunk((const uint8_t*)in, (uint32_t)n_bytes, em, (uint16_t*)smem, lane);
  if (lane == 0 && comp_bytes) *comp_bytes = em.op;
  __syncwarp();
  return nvcompSuccess;
}

}  // namespace snappy
}  // namespace device
}  // namespace nvcomp
