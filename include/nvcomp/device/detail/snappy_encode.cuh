// nvcomp/device/detail/snappy_encode.cuh -- Snappy raw-format emitter of the warp-per-chunk LZ77 matcher
// (lz77_compress.cuh).  The batched compressor (nvcomp_b200/csrc/snappy.cu) and the device API
// (nvcomp/device/snappy.cuh) share it.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"
#include "nvcomp/device/detail/lz77_compress.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

struct SnappyEmitter {
  uint8_t* out;
  uint32_t op;

  __device__ __forceinline__ void begin(uint32_t n, int lane) {
    // varint32 of the uncompressed length
    uint32_t v = n, k = 0;
    while (v >= 0x80u) { if (lane == 0) out[op + k] = (uint8_t)(v | 0x80u); v >>= 7; ++k; }
    if (lane == 0) out[op + k] = (uint8_t)v;
    op += k + 1;
  }
  __device__ __forceinline__ void literal(const uint8_t* lit, uint32_t ll, int lane) {
    if (ll == 0) return;
    const uint32_t n1 = ll - 1;
    if (n1 < 60) {
      if (lane == 0) out[op] = (uint8_t)(n1 << 2);
      op += 1;
    } else {
      const uint32_t nb = n1 < (1u << 8) ? 1u : n1 < (1u << 16) ? 2u : n1 < (1u << 24) ? 3u : 4u;
      if (lane == 0) {
        out[op] = (uint8_t)((59u + nb) << 2);
        for (uint32_t i = 0; i < nb; ++i) out[op + 1 + i] = (uint8_t)(n1 >> (8 * i));
      }
      op += 1 + nb;
    }
    warp_copy<true>(out + op, lit, ll, lane);
    op += ll;
  }
  __device__ __forceinline__ void copy_tail(uint32_t off, uint32_t len, int lane) {   // len 4..64 (or 1..64)
    if (len < 12 && off < 2048 && len >= 4) {
      if (lane == 0) {
        out[op] = (uint8_t)(1u | ((len - 4) << 2) | ((off >> 8) << 5));
        out[op + 1] = (uint8_t)(off & 255u);
      }
      op += 2;
    } else {
      if (lane == 0) {
        out[op] = (uint8_t)(2u | ((len - 1) << 2));
        out[op + 1] = (uint8_t)(off & 255u);
        out[op + 2] = (uint8_t)(off >> 8);
      }
      op += 3;
    }
  }
  __device__ __forceinline__ void sequence(const uint8_t* lit, uint32_t ll, uint32_t off,
                                           uint32_t ml, int lane) {
    literal(lit, ll, lane);
    // long matches split into copy-2 elements of 64 bytes; emitted lane-parallel
    const uint32_t q = (ml >= 68) ? (ml - 4) / 64 : 0;
    for (uint32_t i = lane; i < q; i += kWarp) {
      uint8_t* p = out + op + 3 * i;
      p[0] = (uint8_t)(2u | (63u << 2));
      p[1] = (uint8_t)(off & 255u);
      p[2] = (uint8_t)(off >> 8);
    }
    op += 3 * q;
    uint32_t rem = ml - 64 * q;
    if (rem > 64) { copy_tail(off, 60, lane); rem -= 60; }
    copy_tail(off, rem, lane);
  }
  __device__ __forceinline__ void finish(const uint8_t* lit, uint32_t ll, int lane) {
    literal(lit, ll, lane);
  }
};

// The matcher's parse of the n bytes at `in` after the preamble, into em (a SnappyEmitter, after em.begin(n), writes
// the stream).  Snappy has no end-of-block rules; a match starts at least 4 bytes before the end, which keeps the
// 4-byte probe in bounds.
template <class Emitter>
__device__ __forceinline__ void snappy_compress_chunk(const uint8_t* __restrict__ in, uint32_t n, Emitter& em,
                                                      uint16_t* table, int lane) {
  lz77_compress_chunk(in, n, em, table, 1u, 0u, 4u, lane);
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
