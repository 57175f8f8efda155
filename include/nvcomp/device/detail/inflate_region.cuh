// nvcomp/device/detail/inflate_region.cuh -- one Deflate or Gzip chunk decoded (or walked, for the size query) in a
// caller's per-warp shared-memory region: what nvcomp/device/deflate.cuh and gzip.cuh share.
#pragma once

#include "nvcomp/shared_types.h"
#include "nvcomp/device/detail/crc32.cuh"
#include "nvcomp/device/detail/inflate_decode.cuh"

namespace nvcomp {
namespace device {
namespace deflate {
namespace detail {

// The Gzip region: the decoder's tables (kInfWarpSmem bytes), then the CRC-32 byte table (256 words) and the
// x^(2^k) table (32 words), 1 152 bytes
constexpr uint32_t kInfCrcWords = 256 + 32;
constexpr size_t kGzipWarpSmem = kInfWarpSmem + 4 * kInfCrcWords;

// inflate_chunk<kGzip, kCount> as the batched inflate_kernel calls it, with the decoder state in `smem`.  The batched
// kernel builds the CRC tables once per CTA and keeps a warp's fixed-code tables from chunk to chunk; here the region
// holds nothing between calls, so the warp builds the CRC tables (Gzip only) on every call and starts with
// fixed_ready = false.  A chunk or capacity of 2^32 bytes or more is rejected, as in the batched kernel.  Returns an
// InflateResult and *produced; every lane is past the closing __syncwarp.
template <bool kGzip, bool kCount>
__device__ __forceinline__ int inflate_in_region(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 uint32_t* produced, void* smem) {
  const int lane = lz::detail::lane_id();
  uint32_t* crc = (uint32_t*)((uint8_t*)smem + kInfWarpSmem);
  if (kGzip) {
    for (uint32_t i = (uint32_t)lane; i < kInfCrcWords; i += 32u)
      crc[i] = i < 256u ? crc::detail::crc_table_entry(i) : crc::detail::crc_x2n_entry((int)(i - 256u));
    __syncwarp();
  }
  InflateWarp ws{lz::detail::smem_addr(smem), false};
  *produced = 0;
  int r = kInflateBad;
  if (comp_bytes <= 0xffffffffull && capacity <= 0xffffffffull)
    r = inflate_chunk<kGzip, kCount>((const uint8_t*)comp, (uint32_t)comp_bytes, (uint8_t*)out, (uint32_t)capacity,
                                     produced, ws, crc, crc + 256, lane);
  __syncwarp();
  return r;
}

// decompress_warp of deflate.cuh and gzip.cuh: the statuses and sizes the batched inflate_kernel reports
template <bool kGzip>
__device__ __forceinline__ nvcompStatus_t inflate_decompress_warp(const void* comp, size_t comp_bytes, void* out,
                                                                  size_t capacity, size_t* actual, void* smem) {
  uint32_t produced = 0;
  const int r = inflate_in_region<kGzip, false>(comp, comp_bytes, out, capacity, &produced, smem);
  if (lz::detail::lane_id() == 0 && actual) *actual = r == kInflateOk ? (size_t)produced : 0;
  __syncwarp();
  return r == kInflateOk ? nvcompSuccess
         : r == kInflateBadChecksum ? nvcompErrorBadChecksum : nvcompErrorCannotDecompress;
}

// decompressed_size_warp of deflate.cuh and gzip.cuh: the kCount walk, as the batched size query runs it (capacity
// 2^32 - 1); 0 for a chunk it rejects
template <bool kGzip>
__device__ __forceinline__ size_t inflate_size_warp(const void* comp, size_t comp_bytes, void* smem) {
  uint32_t produced = 0;
  const int r = inflate_in_region<kGzip, true>(comp, comp_bytes, nullptr, 0xffffffffull, &produced, smem);
  return r == kInflateOk ? (size_t)produced : 0;
}

}  // namespace detail
}  // namespace deflate
}  // namespace device
}  // namespace nvcomp
