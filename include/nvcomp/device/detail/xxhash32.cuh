// nvcomp/device/detail/xxhash32.cuh -- XXH32 (seed 0) of a span of global memory by one warp: the LZ4 frame's header,
// block and content checksums (lz4frame_decode.cuh).  Lanes 0-3 run the four accumulators over the 16-byte stripes
// (lane k takes the k-th 4-byte word of every stripe), lane 0 merges them and hashes the tail.  Plain loads only, so
// tests/emu runs it unchanged.
// The out-of-line (__noinline__) function of this header is declared inline: the header is included by every
// translation unit that uses the device API, and inline linkage lets several of them be linked into one program.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"

namespace nvcomp {
namespace device {
namespace lz4frame {
namespace detail {

using lz::detail::kFull;

constexpr uint32_t kXx32P1 = 0x9E3779B1u, kXx32P2 = 0x85EBCA77u, kXx32P3 = 0xC2B2AE3Du, kXx32P4 = 0x27D4EB2Fu,
                   kXx32P5 = 0x165667B1u;

__device__ __forceinline__ uint32_t xx32_rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ __forceinline__ uint32_t xx32_round(uint32_t acc, uint32_t in) {
  acc += in * kXx32P2;
  return xx32_rotl(acc, 13) * kXx32P1;
}
// little-endian load of 4 bytes at any alignment: an aligned word when p is 4-byte aligned, bytes otherwise
__device__ __forceinline__ uint32_t xx32_le32(const uint8_t* p) {
  if (((uintptr_t)p & 3u) == 0) return *(const uint32_t*)p;
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// XXH32(p[0, n), seed 0), returned to every lane.  The caller has made the bytes visible to the warp (__syncwarp).
inline __device__ __noinline__ uint32_t xxh32_warp(const uint8_t* p, uint32_t n, int lane) {
  const uint32_t stripes = n >> 4;
  uint32_t v = 0;
  if (lane < 4) {
    v = lane == 0 ? kXx32P1 + kXx32P2 : lane == 1 ? kXx32P2 : lane == 2 ? 0u : 0u - kXx32P1;
    const uint8_t* q = p + 4 * lane;
    uint32_t s = 0;
    // four stripes per iteration: their loads are independent of the accumulator chain
    for (; s + 4 <= stripes; s += 4) {
      const uint32_t w0 = xx32_le32(q + 16 * s), w1 = xx32_le32(q + 16 * s + 16);
      const uint32_t w2 = xx32_le32(q + 16 * s + 32), w3 = xx32_le32(q + 16 * s + 48);
      v = xx32_round(xx32_round(xx32_round(xx32_round(v, w0), w1), w2), w3);
    }
    for (; s < stripes; ++s) v = xx32_round(v, xx32_le32(q + 16 * s));
  }
  const uint32_t v2 = __shfl_sync(kFull, v, 1), v3 = __shfl_sync(kFull, v, 2), v4 = __shfl_sync(kFull, v, 3);
  uint32_t h = 0;
  if (lane == 0) {
    h = stripes ? xx32_rotl(v, 1) + xx32_rotl(v2, 7) + xx32_rotl(v3, 12) + xx32_rotl(v4, 18) : kXx32P5;
    h += n;
    const uint8_t* t = p + (stripes << 4);
    uint32_t r = n & 15u;
    for (; r >= 4; r -= 4, t += 4) h = xx32_rotl(h + xx32_le32(t) * kXx32P3, 17) * kXx32P4;
    for (; r; --r, ++t) h = xx32_rotl(h + (uint32_t)*t * kXx32P5, 11) * kXx32P1;
    h ^= h >> 15;
    h *= kXx32P2;
    h ^= h >> 13;
    h *= kXx32P3;
    h ^= h >> 16;
  }
  return __shfl_sync(kFull, h, 0);
}

}  // namespace detail
}  // namespace lz4frame
}  // namespace device
}  // namespace nvcomp
