// nvcomp/device/detail/xxhash64.cuh -- XXH64 (seed 0) of a span of global memory by one warp: the Zstandard content
// checksum (RFC 8878 §3.1.1: the low 32 bits of XXH64 of the frame's decoded bytes).  Lanes 0-3 run the four accumulators over the
// 32-byte stripes (lane k takes the k-th 8-byte word of every stripe), lane 0 merges them and hashes the tail.  Plain
// loads only, so tests/emu runs it unchanged.
// The out-of-line (__noinline__) functions of this header are declared inline: the header is included by every
// translation unit that uses the device API, and inline linkage lets several of them be linked into one program.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"

namespace nvcomp {
namespace device {
namespace zstd {
namespace detail {

using lz::detail::kFull;

constexpr uint64_t kXxP1 = 0x9E3779B185EBCA87ull, kXxP2 = 0xC2B2AE3D27D4EB4Full, kXxP3 = 0x165667B19E3779F9ull,
                   kXxP4 = 0x85EBCA77C2B2AE63ull, kXxP5 = 0x27D4EB2F165667C5ull;

__device__ __forceinline__ uint64_t xx_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xx_round(uint64_t acc, uint64_t in) {
  acc += in * kXxP2;
  return xx_rotl(acc, 31) * kXxP1;
}
__device__ __forceinline__ uint64_t xx_merge(uint64_t h, uint64_t v) {
  h ^= xx_round(0, v);
  return h * kXxP1 + kXxP4;
}
// little-endian load of 4 / 8 bytes at any alignment: aligned words when p is 4-byte aligned, bytes otherwise
__device__ __forceinline__ uint32_t xx_le32(const uint8_t* p) {
  if (((uintptr_t)p & 3u) == 0) return *(const uint32_t*)p;
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t xx_le64(const uint8_t* p) {
  return (uint64_t)xx_le32(p) | ((uint64_t)xx_le32(p + 4) << 32);
}

// XXH64(p[0, n), seed 0), returned to every lane.  The caller has made the bytes visible to the warp (__syncwarp).
inline __device__ __noinline__ uint64_t xxh64_warp(const uint8_t* p, uint64_t n, int lane) {
  const uint64_t stripes = n >> 5;
  uint64_t v = 0;
  if (lane < 4) {
    v = lane == 0 ? kXxP1 + kXxP2 : lane == 1 ? kXxP2 : lane == 2 ? 0ull : 0ull - kXxP1;
    const uint8_t* q = p + 8 * lane;
    for (uint64_t s = 0; s < stripes; ++s) v = xx_round(v, xx_le64(q + 32 * s));
  }
  const uint64_t v2 = __shfl_sync(kFull, v, 1), v3 = __shfl_sync(kFull, v, 2), v4 = __shfl_sync(kFull, v, 3);
  uint64_t h = 0;
  if (lane == 0) {
    if (stripes) {
      h = xx_rotl(v, 1) + xx_rotl(v2, 7) + xx_rotl(v3, 12) + xx_rotl(v4, 18);
      h = xx_merge(h, v);
      h = xx_merge(h, v2);
      h = xx_merge(h, v3);
      h = xx_merge(h, v4);
    } else {
      h = kXxP5;
    }
    h += n;
    const uint8_t* t = p + (stripes << 5);
    uint64_t r = n & 31u;
    for (; r >= 8; r -= 8, t += 8) h = xx_rotl(h ^ xx_round(0, xx_le64(t)), 27) * kXxP1 + kXxP4;
    if (r >= 4) {
      h = xx_rotl(h ^ ((uint64_t)xx_le32(t) * kXxP1), 23) * kXxP2 + kXxP3;
      r -= 4;
      t += 4;
    }
    for (; r; --r, ++t) h = xx_rotl(h ^ ((uint64_t)*t * kXxP5), 11) * kXxP1;
    h ^= h >> 33;
    h *= kXxP2;
    h ^= h >> 29;
    h *= kXxP3;
    h ^= h >> 32;
  }
  return __shfl_sync(kFull, h, 0);
}

}  // namespace detail
}  // namespace zstd
}  // namespace device
}  // namespace nvcomp
