// nvcomp/device/lz4frame.cuh -- warp-level LZ4 frame-format decompression inside a user's own kernels.
//
// This is this library's own interface.  decompress_warp returns, for every chunk and capacity, the status, size and
// bytes that nvcompBatchedLZ4FrameDecompressAsync (nvcomp/lz4frame.h) returns: a chunk is zero or more LZ4 frames and
// skippable frames, back to back, as a loop of liblz4's LZ4F_decompress reads it.  decompressed_size_warp returns
// what nvcompBatchedLZ4FrameGetDecompressSizeAsync returns.  Both run the batched kernel's own code
// (detail/lz4frame_decode.cuh), whose compressed blocks go to the LZ4 block bodies of nvcomp/device/lz4.cuh, routed
// with the same rule.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of decompress_warp and decompressed_size_warp: as in nvcomp/device/lz4.cuh --
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual is written once (by lane 0; the pointer may be null).
//   - Compressed streams and outputs are global memory and must not overlap (the decoder stages compressed blocks
//     with cp.async.bulk from global memory).  Any alignment is accepted.
//   - `smem` is this warp's own shared-memory region of kDecompressSmemBytes bytes, aligned to kSmemAlignment; warp
//     w of a CTA can use smem_base + w * kDecompressSmemBytes.  The region holds nothing between calls: the caller
//     may use it for anything else in between.  decompress_warp initializes the region's mbarrier on entry, has no
//     bulk copy in flight on any return (failures included), invalidates the mbarrier (mbarrier.inval) before it
//     returns, and every return passes a __syncwarp.  decompressed_size_warp uses no shared memory.
//   - decompress_warp writes only inside [out, out + capacity).  A successful decode writes exactly *actual bytes.
//   - A header, block or content checksum mismatch whose preceding output fits in the capacity returns
//     nvcompErrorBadChecksum, any other chunk that cannot be decoded (malformed, larger than capacity, or comp_bytes
//     or capacity of 2^32 or more) nvcompErrorCannotDecompress; both with *actual = 0.  No input causes an
//     out-of-bounds access.
//   - Several warps of one CTA may run any mix of LZ4 frame, LZ4 and Snappy calls at once, each with its own region.
//     No call uses global scratch memory.
#pragma once

#include "nvcomp/shared_types.h"
#include "nvcomp/lz4frame.h"
#include "nvcomp/device/detail/lz4frame_decode.cuh"

namespace nvcomp {
namespace device {
namespace lz4frame {

// Alignment of each warp's shared-memory region (16-byte vector accesses and bulk-copy destinations).
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decompressing warp: the LZ4 block decoder's per-warp region (7 248 bytes), the same as
// nvcomp::device::lz4::kDecompressSmemBytes.
constexpr size_t kDecompressSmemBytes = lz::detail::kLzWarpSmem;

static_assert(kDecompressSmemBytes % kSmemAlignment == 0, "warp regions stay aligned");

// Decoded size of the chunk at `comp` -- what nvcompBatchedLZ4FrameGetDecompressSizeAsync reports for it: every frame
// is walked without writing (the content-size field is not trusted).  0 for a rejected chunk.  Warp-collective (see
// above).
__device__ inline size_t decompressed_size_warp(const void* comp, size_t comp_bytes) {
  using namespace detail;
  const int lane = lz::detail::lane_id();
  uint32_t produced = 0, parity = 0;
  int r = kLz4fBad;
  if (comp_bytes <= 0xffffffffull)
    r = lz4f_chunk<true>((const uint8_t*)comp, (uint32_t)comp_bytes, nullptr, 0xffffffffu, &produced, nullptr,
                         parity, lane);
  __syncwarp();
  return r == kLz4fOk ? (size_t)produced : 0;
}

// Decode the comp_bytes-byte chunk at `comp` into [out, out + capacity) with `smem` (kDecompressSmemBytes bytes).
// Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem) {
  using namespace detail;
  const int lane = lz::detail::lane_id();
  uint8_t* ring = (uint8_t*)smem;
  const uint32_t ra = lz::detail::smem_addr(ring);
  // the region's mbarrier lives for this call only (see lz::detail::lz_decompress_in_region)
  lz::detail::lz_warp_init(ra, lane);
  uint32_t parity = 0, produced = 0;
  int r = kLz4fBad;
  if (comp_bytes <= 0xffffffffull && capacity <= 0xffffffffull)
    r = lz4f_chunk<false>((const uint8_t*)comp, (uint32_t)comp_bytes, (uint8_t*)out, (uint32_t)capacity, &produced,
                          ring, parity, lane);
  __syncwarp();
  if (lane == 0) {
    lz::detail::mbar_inval(ra + lz::detail::kSmemMbar);
    if (actual) *actual = r == kLz4fOk ? (size_t)produced : 0;
  }
  __syncwarp();
  return r == kLz4fOk ? nvcompSuccess : r == kLz4fBadChecksum ? nvcompErrorBadChecksum : nvcompErrorCannotDecompress;
}

}  // namespace lz4frame
}  // namespace device
}  // namespace nvcomp
