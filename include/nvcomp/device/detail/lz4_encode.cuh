// nvcomp/device/detail/lz4_encode.cuh -- LZ4 block-format emitter of the warp-per-chunk LZ77 matcher
// (lz77_compress.cuh) and the candidate stride of each data_type.  The batched compressor
// (nvcomp_b200/csrc/lz4.cu) and the device API (nvcomp/device/lz4.cuh) share them.
#pragma once

#include "nvcomp/shared_types.h"
#include "nvcomp/device/detail/lz_common.cuh"
#include "nvcomp/device/detail/lz77_compress.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

struct Lz4Emitter {
  uint8_t* out;
  uint32_t op;

  __device__ __forceinline__ void ext(uint32_t rem, int lane) {   // rem = len - 15
    const uint32_t nb = rem / 255u + 1u;
    for (uint32_t i = lane; i < nb; i += kWarp)
      out[op + i] = (i + 1 < nb) ? (uint8_t)255 : (uint8_t)(rem - 255u * (nb - 1));
    op += nb;
  }
  __device__ __forceinline__ void sequence(const uint8_t* lit, uint32_t ll, uint32_t off,
                                           uint32_t ml, int lane) {
    const uint32_t mlc = ml - 4;
    if (lane == 0) out[op] = (uint8_t)((min(ll, 15u) << 4) | min(mlc, 15u));
    op += 1;
    if (ll >= 15) ext(ll - 15, lane);
    if (ll) warp_copy<true>(out + op, lit, ll, lane);
    op += ll;
    if (lane == 0) { out[op] = (uint8_t)(off & 255u); out[op + 1] = (uint8_t)(off >> 8); }
    op += 2;
    if (mlc >= 15) ext(mlc - 15, lane);
  }
  __device__ __forceinline__ void finish(const uint8_t* lit, uint32_t ll, int lane) {
    if (lane == 0) out[op] = (uint8_t)(min(ll, 15u) << 4);
    op += 1;
    if (ll >= 15) ext(ll - 15, lane);
    if (ll) warp_copy<true>(out + op, lit, ll, lane);
    op += ll;
  }
};

// The matcher's parse of one LZ4 block of the n bytes at `in`, into em (an Lz4Emitter writes the block).  LZ4's
// end-of-block rules: the last 5 bytes are literals, and the last match starts at least 12 bytes before the end
// (reference CHANGELOG.md:195).  step: the data_type's candidate stride.
template <class Emitter>
__device__ __forceinline__ void lz4_compress_chunk(const uint8_t* __restrict__ in, uint32_t n, Emitter& em,
                                                   uint16_t* table, uint32_t step, int lane) {
  lz77_compress_chunk(in, n, em, table, step, 5u, 12u, lane);
}

// Candidate stride (bytes) of the matcher for an LZ4 data_type; *ok = false for a type the LZ4 calls reject.
__host__ __device__ inline uint32_t lz4_step_for(nvcompType_t t, bool* ok) {
  *ok = true;
  switch (t) {
    case NVCOMP_TYPE_CHAR: case NVCOMP_TYPE_UCHAR: case NVCOMP_TYPE_BITS: return 1;
    case NVCOMP_TYPE_SHORT: case NVCOMP_TYPE_USHORT: return 2;
    case NVCOMP_TYPE_INT: case NVCOMP_TYPE_UINT: return 4;
    default: *ok = false; return 1;
  }
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
