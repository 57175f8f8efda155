// nvcomp/device/detail/bitcomp_impl.cuh -- the Bitcomp stream and its per-block coder, shared by the batched kernels
// (nvcomp_b200/csrc/bitcomp.cu) and the warp-level device API (nvcomp/device/bitcomp.cuh).  Header-only device code
// for sm_90a; not a public interface.
//
// Bitcomp is proprietary and undocumented in the reference, so this library defines its own lossless stream with the
// same options: algorithm 0 "default" and 1 "sparse", element types CHAR..ULONGLONG.
//
// Chunk stream (8-byte aligned):
//   u32 magic 'BTC1', u32 algo | type<<8, u32 uncompressed_bytes, u32 nblocks
//   u16 desc[nblocks] (padded to 8 bytes)
//   block payloads, 8-byte aligned, in order; a block covers 128 consecutive elements
//   if uncompressed_bytes is not a multiple of the element size: one more 8-byte word holding the
//   uncompressed_bytes % size trailing bytes verbatim (zero padded), so any chunk length round-trips
// algo 0: desc = bits.  payload = u64 first element, then 128*bits bits: zig-zag of the
//         delta to the previous element of the block (slot 0 holds 0).
// algo 1: desc = nz | bits<<8.  payload = 128-bit non-zero mask, then nz*bits bits of the
//         non-zero elements in order (rounded up to 8 bytes).
//
// Every block function here is called by a whole warp on one block, 4 consecutive elements per lane; the callers own
// the block offsets, the shared memory and the barriers between blocks.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include "nvcomp/bitcomp.h"

namespace nvcomp {
namespace device {
namespace bitcomp {
namespace detail {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr uint32_t kWarpSize = 32;
constexpr uint32_t kBtcMagic = 0x31435442u;  // "BTC1"
constexpr uint32_t kBtcBlock = 128;          // elements per block

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__host__ __device__ inline uint32_t btc_type_size(int t) {
  switch (t) {
    case NVCOMP_TYPE_CHAR: case NVCOMP_TYPE_UCHAR: return 1;
    case NVCOMP_TYPE_SHORT: case NVCOMP_TYPE_USHORT: return 2;
    case NVCOMP_TYPE_INT: case NVCOMP_TYPE_UINT: return 4;
    case NVCOMP_TYPE_LONGLONG: case NVCOMP_TYPE_ULONGLONG: return 8;
    default: return 0;
  }
}

__device__ __forceinline__ uint32_t btc_block_bytes(int algo, uint32_t desc) {
  if (algo == 0) return 8u + 16u * (desc & 0xffu);
  const uint32_t nz = desc & 0xffu, bits = desc >> 8;
  return 16u + 8u * ((nz * bits + 63u) / 64u);
}

// A descriptor the decoder rejects: algo 0 wider than 64 bits; algo 1 wider than 64 bits or more than 128 non-zeros.
__device__ __forceinline__ bool btc_desc_bad(int algo, uint32_t d) {
  return algo == 0 ? (d & 0xff) > 64u : ((d >> 8) > 64u || (d & 0xff) > 128u);
}

template <int TS> struct BtcElem;
template <> struct BtcElem<1> { using T = uint8_t; };
template <> struct BtcElem<2> { using T = uint16_t; };
template <> struct BtcElem<4> { using T = uint32_t; };
template <> struct BtcElem<8> { using T = uint64_t; };

template <int TS> __device__ __forceinline__ uint64_t btc_trunc(uint64_t v) {
  return TS == 8 ? v : (v & ((1ull << (8 * TS)) - 1ull));
}
template <int TS> __device__ __forceinline__ uint64_t btc_zigzag(uint64_t d) {   // d: wrapped delta in TS bytes
  const int sh = 64 - 8 * TS;
  const int64_t s = ((int64_t)(d << sh)) >> sh;
  return btc_trunc<TS>(((uint64_t)s << 1) ^ (uint64_t)(s >> 63));
}
__device__ __forceinline__ uint64_t btc_unzigzag(uint64_t z) {
  return (z >> 1) ^ (0ull - (z & 1ull));
}

__device__ __forceinline__ uint64_t btc_unpack(const uint64_t* __restrict__ words, uint32_t k, uint32_t bits) {
  const uint32_t bitpos = k * bits;
  const uint32_t w = bitpos >> 6, s = bitpos & 63;
  uint64_t v = words[w] >> s;
  if (s + bits > 64) v |= words[w + 1] << (64 - s);
  if (bits < 64) v &= ((1ull << bits) - 1ull);
  return v;
}

struct BtcHeader { uint32_t algo, type, uncompressed, nblocks; };

__device__ __forceinline__ bool btc_read_header(const uint8_t* in, size_t in_bytes, BtcHeader& h) {
  if (in_bytes < 16 || ((uintptr_t)in & 7)) return false;
  const uint32_t* w = (const uint32_t*)in;
  if (w[0] != kBtcMagic) return false;
  h.algo = w[1] & 0xff; h.type = (w[1] >> 8) & 0xff; h.uncompressed = w[2]; h.nblocks = w[3];
  const uint32_t ts = btc_type_size(h.type);
  if (ts == 0 || h.algo > 1) return false;
  const uint32_t n = h.uncompressed / ts;
  if (h.nblocks != (n + kBtcBlock - 1) / kBtcBlock) return false;
  if (16ull + 2ull * h.nblocks > in_bytes) return false;
  return true;
}

// four consecutive elements (16-byte vector stores when 4*sizeof(T) >= 16)
template <class T>
struct alignas(sizeof(T) * 4 > 16 ? 16 : sizeof(T) * 4) BtcQuad { T e[4]; };

// Decode this lane's four consecutive elements of one block into v (zero-extended to 64 bits; slots past the chunk's
// end hold whatever the payload gives them).  Returns false for a malformed block (sparse mask that disagrees with
// its non-zero count); the result is warp-uniform.
template <int TS>
__device__ __forceinline__ bool btc_decode_values(int algo, uint32_t desc, const uint8_t* __restrict__ payload,
                                                  int lane, uint64_t v[4]) {
  const uint64_t* p64 = (const uint64_t*)payload;
  bool good = true;
  if (algo == 0) {
    const uint32_t bits = desc & 0xffu;
    const uint64_t first = p64[0];
    if (bits <= 16u) {
      // Small deltas (the common case for sorted / smooth columns): the zigzag codes fit 16 bits, so
      // the lane-local prefix and the warp scan run in 32-bit arithmetic (|sum of 128 deltas| < 2^23);
      // only the final "first + prefix" is 64-bit.  bits is uniform over the block: no divergence.
      uint32_t z[4];
      if (bits <= 8u) {
        // the lane's four codes lie inside 32 bits: one or two 32-bit words and a funnel shift
        const uint32_t* p32 = (const uint32_t*)(p64 + 1);
        const uint32_t bitpos = 4u * (uint32_t)lane * bits;
        const uint32_t w0 = bitpos >> 5, s0 = bitpos & 31u;
        uint32_t lo = 0, hi = 0;
        if (bits) {
          lo = p32[w0];
          if (s0 + 4u * bits > 32u) hi = p32[w0 + 1];
        }
        const uint32_t x = __funnelshift_r(lo, hi, s0);
        const uint32_t mask = (1u << bits) - 1u;
#pragma unroll
        for (int j = 0; j < 4; ++j) z[j] = (x >> ((uint32_t)j * bits)) & mask;
      } else {
        // four codes span at most 64 + 63 bits: two 64-bit word loads, then shifts
        const uint32_t bitpos = 4u * (uint32_t)lane * bits;
        const uint32_t w0 = bitpos >> 6, s0 = bitpos & 63u;
        const uint64_t lo = p64[1 + w0];
        const uint64_t hi = (s0 + 4u * bits > 64u) ? p64[2 + w0] : 0ull;
        const uint64_t mask = (1ull << bits) - 1ull;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t sj = s0 + (uint32_t)j * bits;          // < 128
          uint64_t zz;
          if (sj < 64u) zz = (lo >> sj) | (sj ? (hi << (64u - sj)) : 0ull);
          else zz = hi >> (sj - 64u);
          z[j] = (uint32_t)(zz & mask);
        }
      }
      uint32_t pre[4], acc = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) { acc += (z[j] >> 1) ^ (0u - (z[j] & 1u)); pre[j] = acc; }
      uint32_t incl = acc;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(kFullMask, incl, d);
        if (lane >= d) incl += o;
      }
      const uint32_t base = incl - acc;
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = first + (uint64_t)(int64_t)(int32_t)(base + pre[j]);
    } else {
      uint64_t sum = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint64_t z = btc_unpack(p64 + 1, 4 * lane + j, bits);
        sum += btc_unzigzag(z);
        v[j] = sum;
      }
      uint64_t incl = sum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint64_t o = __shfl_up_sync(kFullMask, incl, d);
        if (lane >= d) incl += o;
      }
      const uint64_t base = first + incl - sum;
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] += base;
    }
  } else {
    const uint32_t bits = desc >> 8;
    const uint64_t mlo = p64[0], mhi = p64[1];
    // the payload holds exactly nz packed values: a mask with more bits set would read past it
    good = (uint32_t)(__popcll(mlo) + __popcll(mhi)) == (desc & 0xffu);
    // rank of this lane's first element among the non-zeros
    const uint32_t e0 = 4 * lane;
    uint32_t rank;
    if (e0 < 64) rank = __popcll(mlo & ((1ull << e0) - 1ull));
    else rank = __popcll(mlo) + __popcll(mhi & ((1ull << (e0 - 64)) - 1ull));
    const uint64_t mw = (e0 < 64) ? (mlo >> e0) : (mhi >> (e0 - 64));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if ((mw >> j) & 1ull) { v[j] = (bits && good) ? btc_unpack(p64 + 2, rank, bits) : 0ull; ++rank; }
      else v[j] = 0;
    }
  }
  return good;
}

// Decode one block to out (the block's first element); returns btc_decode_values' verdict.
template <int TS>
__device__ __forceinline__ bool btc_decode_block(int algo, uint32_t desc, const uint8_t* __restrict__ payload,
                                                 typename BtcElem<TS>::T* out, uint32_t n_valid, int lane) {
  using T = typename BtcElem<TS>::T;
  uint64_t v[4];
  const bool good = btc_decode_values<TS>(algo, desc, payload, lane, v);
  const uint32_t e = 4 * lane;
  // the lane's four consecutive elements leave as one vector store when the chunk pointer allows it
  BtcQuad<T> q;
#pragma unroll
  for (int j = 0; j < 4; ++j) q.e[j] = (T)v[j];
  if (e + 3u < n_valid && ((uintptr_t)out & (alignof(BtcQuad<T>) - 1)) == 0) {
    *(BtcQuad<T>*)(out + e) = q;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (e + j < n_valid) out[e + j] = q.e[j];
  }
  return good;
}

template <int TS>
__device__ __forceinline__ void btc_load4(const typename BtcElem<TS>::T* in, uint32_t n_valid, int lane, uint64_t v[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t e = 4 * lane + j;
    v[j] = (e < n_valid) ? (uint64_t)in[e] : 0ull;
  }
}

// zig-zag deltas of the 4 elements of this lane (slot 0 of the block -> 0); invalid slots -> 0
template <int TS>
__device__ __forceinline__ void btc_deltas(const uint64_t v[4], uint32_t n_valid, int lane, uint64_t z[4]) {
  uint64_t prev = __shfl_up_sync(kFullMask, v[3], 1);
  if (lane == 0) prev = v[0];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t e = 4 * lane + j;
    z[j] = (e < n_valid) ? btc_zigzag<TS>(btc_trunc<TS>(v[j] - prev)) : 0ull;
    prev = v[j];
  }
}

// The block's descriptor (warp-uniform).
template <int TS>
__device__ __forceinline__ uint32_t btc_analyse_block(int algo, const typename BtcElem<TS>::T* in,
                                                      uint32_t n_valid, int lane) {
  uint64_t v[4];
  btc_load4<TS>(in, n_valid, lane, v);
  if (algo == 0) {
    uint64_t z[4];
    btc_deltas<TS>(v, n_valid, lane, z);
    uint64_t m = z[0] | z[1] | z[2] | z[3];
#pragma unroll
    for (int d = 16; d; d >>= 1) m |= __shfl_xor_sync(kFullMask, m, d);
    return m ? 64 - __clzll((long long)m) : 0;
  }
  uint64_t m = v[0] | v[1] | v[2] | v[3];
  uint32_t nz = (v[0] != 0) + (v[1] != 0) + (v[2] != 0) + (v[3] != 0);
#pragma unroll
  for (int d = 16; d; d >>= 1) { m |= __shfl_xor_sync(kFullMask, m, d); nz += __shfl_xor_sync(kFullMask, nz, d); }
  const uint32_t bits = m ? 64 - __clzll((long long)m) : 0;
  return nz | (bits << 8);
}

// OR a value of `bits` bits at bit position `bitpos` into the u64 word array (shared memory)
__device__ __forceinline__ void btc_put(unsigned long long* words, uint32_t bitpos, uint32_t bits, uint64_t v) {
  const uint32_t w = bitpos >> 6, s = bitpos & 63;
  atomicOr(&words[w], v << s);
  if (s + bits > 64) atomicOr(&words[w + 1], v >> (64 - s));
}

// Pack one block with descriptor `desc` at `payload` (btc_block_bytes(algo, desc) bytes).  `words` is the warp's
// shared-memory packing area of kBtcPackWords words.
constexpr uint32_t kBtcPackWords = 132;
template <int TS>
__device__ __forceinline__ void btc_pack_block(int algo, uint32_t desc, const typename BtcElem<TS>::T* in,
                                               uint32_t n_valid, uint8_t* payload,
                                               unsigned long long* words, int lane) {
  uint64_t v[4];
  btc_load4<TS>(in, n_valid, lane, v);
  unsigned long long* p64 = (unsigned long long*)payload;
  if (algo == 0) {
    const uint32_t bits = desc & 0xffu;
    const uint32_t nwords = 2 * bits;              // 128*bits/64
    for (uint32_t i = lane; i < nwords + 1; i += kWarpSize) words[i] = 0ull;
    __syncwarp();
    uint64_t z[4];
    btc_deltas<TS>(v, n_valid, lane, z);
    if (bits) {
#pragma unroll
      for (int j = 0; j < 4; ++j) btc_put(words, (4 * lane + j) * bits, bits, z[j]);
    }
    __syncwarp();
    if (lane == 0) p64[0] = v[0];
    for (uint32_t i = lane; i < nwords; i += kWarpSize) p64[1 + i] = words[i];
  } else {
    const uint32_t nz = desc & 0xffu, bits = desc >> 8;
    const uint32_t nwords = (nz * bits + 63u) / 64u;
    for (uint32_t i = lane; i < nwords + 1; i += kWarpSize) words[i] = 0ull;
    __syncwarp();
    uint32_t mine = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) mine |= (v[j] != 0 ? 1u : 0u) << j;
    // 128-bit mask: lane contributes 4 bits at position 4*lane
    uint64_t part_lo = (lane < 16) ? ((uint64_t)mine << (4 * lane)) : 0ull;
    uint64_t part_hi = (lane >= 16) ? ((uint64_t)mine << (4 * (lane - 16))) : 0ull;
    uint32_t cnt = __popc(mine), incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(kFullMask, incl, d);
      if (lane >= d) incl += o;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      part_lo |= __shfl_xor_sync(kFullMask, part_lo, d);
      part_hi |= __shfl_xor_sync(kFullMask, part_hi, d);
    }
    uint32_t rank = incl - cnt;
    if (bits) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (v[j] != 0) { btc_put(words, rank * bits, bits, v[j]); ++rank; }
    }
    __syncwarp();
    if (lane == 0) { p64[0] = part_lo; p64[1] = part_hi; }
    for (uint32_t i = lane; i < nwords; i += kWarpSize) p64[2 + i] = words[i];
  }
  __syncwarp();
}

}  // namespace detail
}  // namespace bitcomp
}  // namespace device
}  // namespace nvcomp
