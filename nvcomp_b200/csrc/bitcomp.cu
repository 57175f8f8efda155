// bitcomp.cu -- batched Bitcomp-style typed bit-packing codec for H100 (sm_90a) + C ABI.
//
// Replaces the closed nvcompBatchedBitcomp* entry points (include/nvcomp/bitcomp.h;
// reference benchmarks/benchmark_bitcomp_chunked.cu:114-118).  Bitcomp is proprietary
// and undocumented in the reference, so this library defines its own lossless stream
// with the same options: algorithm 0 "default" and 1 "sparse", element types CHAR..ULONGLONG.
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
// Decode: one CTA per chunk; block payload offsets come from a block-wide scan of the
// descriptor table, 512 blocks per tile; every warp then decodes whole blocks (4
// consecutive elements per lane, warp-scan for the delta prefix) -- pure streaming.
#include "common.cuh"
#include "nvcomp/bitcomp.h"

namespace b200 {

constexpr uint32_t kBtcMagic = 0x31435442u;  // "BTC1"
constexpr int kBtcWarps = 4;
constexpr int kBtcThreads = kBtcWarps * 32;
constexpr uint32_t kBtcBlock = 128;          // elements per block
constexpr uint32_t kBtcTile = 512;           // blocks per offset tile (4 per thread)
constexpr uint32_t kBtcStage = 12288;        // bytes of packed payload staged per tile by one TMA bulk copy

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

// block-wide exclusive scan of 4 values per thread; returns tile total.  scratch: kBtcWarps+1 u32
__device__ __forceinline__ uint32_t btc_block_scan4(uint32_t v[4], uint32_t excl[4], uint32_t* scratch) {
  const int lane = lane_id(), w = threadIdx.x >> 5;
  uint32_t local = v[0] + v[1] + v[2] + v[3];
  uint32_t incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t o = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) scratch[w] = incl;
  __syncthreads();
  uint32_t wbase = 0, total = 0;
#pragma unroll
  for (int i = 0; i < kBtcWarps; ++i) {
    const uint32_t s = scratch[i];
    if (i < w) wbase += s;
    total += s;
  }
  uint32_t e = wbase + incl - local;
  excl[0] = e; excl[1] = e + v[0]; excl[2] = excl[1] + v[1]; excl[3] = excl[2] + v[2];
  __syncthreads();
  return total;
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

// returns false for a malformed block (sparse mask that disagrees with its non-zero count)
template <int TS>
__device__ __forceinline__ bool btc_decode_block(int algo, uint32_t desc, const uint8_t* __restrict__ payload,
                                                 typename BtcElem<TS>::T* out, uint32_t n_valid, int lane) {
  using T = typename BtcElem<TS>::T;
  const uint64_t* p64 = (const uint64_t*)payload;
  uint64_t v[4];
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
        const uint32_t o = __shfl_up_sync(kFull, incl, d);
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
        const uint64_t o = __shfl_up_sync(kFull, incl, d);
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

__global__ void __launch_bounds__(kBtcThreads)
bitcomp_decompress_kernel(const void* const* __restrict__ comp_ptrs,
                          const size_t* __restrict__ comp_bytes,
                          const size_t* __restrict__ out_caps,
                          size_t* actual_bytes, size_t batch,
                          void* const* __restrict__ out_ptrs,
                          nvcompStatus_t* statuses,
                          unsigned long long* ticket) {
  __shared__ uint32_t s_off[kBtcTile];
  __shared__ uint16_t s_desc[kBtcTile];
  __shared__ uint32_t s_scratch[kBtcWarps + 1];
  __shared__ unsigned long long s_chunk;
  __shared__ int s_fail;
  // packed payload of one tile, staged by a TMA bulk copy (cp.async.bulk -> mbarrier): the unpack
  // loads then hit shared memory instead of stalling on global memory (long-scoreboard was the top stall)
  __shared__ __align__(128) uint8_t s_stage[kBtcStage];
  __shared__ __align__(8) unsigned long long s_mbar;
  const uint32_t mbar = (uint32_t)__cvta_generic_to_shared(&s_mbar);
  const uint32_t stage_s = (uint32_t)__cvta_generic_to_shared(s_stage);
  uint32_t parity = 0;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  if (threadIdx.x == 0) mbar_init(mbar, 1);
  __syncthreads();
  size_t static_next = blockIdx.x;
  while (true) {
    if (threadIdx.x == 0) {
      s_chunk = ticket ? atomicAdd(ticket, 1ull) : (unsigned long long)static_next;
      s_fail = 0;
    }
    static_next += gridDim.x;
    __syncthreads();
    const size_t c = (size_t)s_chunk;
    if (c >= batch) break;
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    const size_t in_bytes = comp_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    BtcHeader h;
    bool ok = btc_read_header(in, in_bytes, h);
    const uint32_t ts = ok ? btc_type_size(h.type) : 1;
    if (ok && (h.uncompressed > out_caps[c] || ((uintptr_t)out & (ts - 1)))) ok = false;
    if (ok) {
      const uint16_t* desc = (const uint16_t*)(in + 16);
      const uint32_t n_elems = h.uncompressed / ts;
      uint32_t base_off = (16u + 2u * h.nblocks + 7u) & ~7u;
      for (uint32_t tile = 0; tile < h.nblocks; tile += kBtcTile) {
        uint32_t sz[4], ex[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t b = tile + 4 * threadIdx.x + j;
          uint32_t d = 0;
          if (b < h.nblocks) d = desc[b];
          sz[j] = (b < h.nblocks) ? btc_block_bytes(h.algo, d) : 0u;
          if (h.algo == 0 ? (d & 0xff) > 64u : ((d >> 8) > 64u || (d & 0xff) > 128u)) s_fail = 1;
          s_desc[4 * threadIdx.x + j] = (uint16_t)d;
        }
        const uint32_t total = btc_block_scan4(sz, ex, s_scratch);
#pragma unroll
        for (int j = 0; j < 4; ++j) s_off[4 * threadIdx.x + j] = base_off + ex[j];
        if ((uint64_t)base_off + total > in_bytes) s_fail = 1;
        __syncthreads();
        if (!s_fail) {
          const uint32_t nb = min(kBtcTile, h.nblocks - tile);
          // stage [base_off, base_off + total) (16-byte aligned span around it) if it fits
          const uint8_t* tile_src = in + base_off;
          const uint32_t delta = (uint32_t)((uintptr_t)tile_src & 15u);
          const uint32_t span = (delta + total + 15u) & ~15u;
          const bool staged = total != 0u && span <= kBtcStage;
          if (staged) {
            if (threadIdx.x == 0) {
              fence_proxy_async_smem();
              mbar_expect_tx(mbar, span);
              tma_bulk_g2s(stage_s, tile_src - delta, span, mbar);
            }
            mbar_wait(mbar, parity);
            parity ^= 1u;
          }
          const uint8_t* pay_base = staged ? (const uint8_t*)s_stage + delta - base_off : in;
          for (uint32_t b = w; b < nb; b += kBtcWarps) {
            const uint32_t blk = tile + b;
            const uint32_t e0 = blk * kBtcBlock;
            const uint32_t nv = min(kBtcBlock, n_elems - e0);
            const uint8_t* payload = pay_base + s_off[b];
            const uint32_t d = s_desc[b];
            bool bok;
            switch (ts) {
              case 1: bok = btc_decode_block<1>(h.algo, d, payload, (uint8_t*)out + e0, nv, lane); break;
              case 2: bok = btc_decode_block<2>(h.algo, d, payload, (uint16_t*)out + e0, nv, lane); break;
              case 4: bok = btc_decode_block<4>(h.algo, d, payload, (uint32_t*)out + e0, nv, lane); break;
              default: bok = btc_decode_block<8>(h.algo, d, payload, (uint64_t*)out + e0, nv, lane); break;
            }
            if (!bok && lane == 0) s_fail = 1;
          }
        }
        base_off += total;
        __syncthreads();
      }
      // trailing bytes of a chunk whose length is not a multiple of the element size: stored verbatim
      const uint32_t tail = h.uncompressed - n_elems * ts;
      if (tail) {
        if ((uint64_t)base_off + 8u > in_bytes) s_fail = 1;
        else if (threadIdx.x < tail && !s_fail) out[n_elems * ts + threadIdx.x] = in[base_off + threadIdx.x];
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const bool good = ok && !s_fail;
      if (actual_bytes) actual_bytes[c] = good ? (size_t)h.uncompressed : 0;
      if (statuses) statuses[c] = good ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    __syncthreads();
  }
}

__global__ void bitcomp_size_kernel(const void* const* __restrict__ comp_ptrs,
                                    const size_t* __restrict__ comp_bytes,
                                    size_t* out_sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= batch) return;
  BtcHeader h;
  const bool ok = btc_read_header((const uint8_t*)comp_ptrs[c], comp_bytes[c], h);
  out_sizes[c] = ok ? (size_t)h.uncompressed : 0;
}

// ---------------------------------------------------------------------------
// Compression: one CTA per chunk, two passes per 512-block tile
//   pass 1: every warp analyses whole blocks -> descriptor (bits / nz)
//   scan  : block-wide scan of payload sizes -> offsets
//   pass 2: every warp packs its blocks at their final offsets
// ---------------------------------------------------------------------------
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
  uint64_t prev = __shfl_up_sync(kFull, v[3], 1);
  if (lane == 0) prev = v[0];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t e = 4 * lane + j;
    z[j] = (e < n_valid) ? btc_zigzag<TS>(btc_trunc<TS>(v[j] - prev)) : 0ull;
    prev = v[j];
  }
}

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
    for (int d = 16; d; d >>= 1) m |= __shfl_xor_sync(kFull, m, d);
    return m ? 64 - __clzll((long long)m) : 0;
  }
  uint64_t m = v[0] | v[1] | v[2] | v[3];
  uint32_t nz = (v[0] != 0) + (v[1] != 0) + (v[2] != 0) + (v[3] != 0);
#pragma unroll
  for (int d = 16; d; d >>= 1) { m |= __shfl_xor_sync(kFull, m, d); nz += __shfl_xor_sync(kFull, nz, d); }
  const uint32_t bits = m ? 64 - __clzll((long long)m) : 0;
  return nz | (bits << 8);
}

// OR a value of `bits` bits at bit position `bitpos` into the u64 word array (shared memory)
__device__ __forceinline__ void btc_put(unsigned long long* words, uint32_t bitpos, uint32_t bits, uint64_t v) {
  const uint32_t w = bitpos >> 6, s = bitpos & 63;
  atomicOr(&words[w], v << s);
  if (s + bits > 64) atomicOr(&words[w + 1], v >> (64 - s));
}

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
    for (uint32_t i = lane; i < nwords + 1; i += kWarp) words[i] = 0ull;
    __syncwarp();
    uint64_t z[4];
    btc_deltas<TS>(v, n_valid, lane, z);
    if (bits) {
#pragma unroll
      for (int j = 0; j < 4; ++j) btc_put(words, (4 * lane + j) * bits, bits, z[j]);
    }
    __syncwarp();
    if (lane == 0) p64[0] = v[0];
    for (uint32_t i = lane; i < nwords; i += kWarp) p64[1 + i] = words[i];
  } else {
    const uint32_t nz = desc & 0xffu, bits = desc >> 8;
    const uint32_t nwords = (nz * bits + 63u) / 64u;
    for (uint32_t i = lane; i < nwords + 1; i += kWarp) words[i] = 0ull;
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
      const uint32_t o = __shfl_up_sync(kFull, incl, d);
      if (lane >= d) incl += o;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      part_lo |= __shfl_xor_sync(kFull, part_lo, d);
      part_hi |= __shfl_xor_sync(kFull, part_hi, d);
    }
    uint32_t rank = incl - cnt;
    if (bits) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (v[j] != 0) { btc_put(words, rank * bits, bits, v[j]); ++rank; }
    }
    __syncwarp();
    if (lane == 0) { p64[0] = part_lo; p64[1] = part_hi; }
    for (uint32_t i = lane; i < nwords; i += kWarp) p64[2 + i] = words[i];
  }
  __syncwarp();
}

__global__ void __launch_bounds__(kBtcThreads)
bitcomp_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                        size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                        int algo, int type, unsigned long long* ticket) {
  __shared__ uint32_t s_off[kBtcTile];
  __shared__ uint16_t s_desc[kBtcTile];
  __shared__ uint32_t s_scratch[kBtcWarps + 1];
  __shared__ unsigned long long s_words[kBtcWarps][132];
  __shared__ unsigned long long s_chunk;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const uint32_t ts = btc_type_size(type);
  size_t static_next = blockIdx.x;
  while (true) {
    if (threadIdx.x == 0) s_chunk = ticket ? atomicAdd(ticket, 1ull) : (unsigned long long)static_next;
    static_next += gridDim.x;
    __syncthreads();
    const size_t c = (size_t)s_chunk;
    if (c >= batch) break;
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    const uint32_t n_bytes = (uint32_t)in_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    const uint32_t n_elems = n_bytes / ts;
    const uint32_t nblocks = (n_elems + kBtcBlock - 1) / kBtcBlock;
    if (threadIdx.x == 0) {
      uint32_t* hw = (uint32_t*)out;
      hw[0] = kBtcMagic; hw[1] = (uint32_t)algo | ((uint32_t)type << 8); hw[2] = n_bytes; hw[3] = nblocks;
    }
    uint16_t* desc = (uint16_t*)(out + 16);
    uint32_t base_off = (16u + 2u * nblocks + 7u) & ~7u;
    // clear the descriptor pad so the stream is deterministic
    if (threadIdx.x < 4) { const uint32_t i = nblocks + threadIdx.x; if (16u + 2u * i < base_off) desc[i] = 0; }
    for (uint32_t tile = 0; tile < nblocks; tile += kBtcTile) {
      const uint32_t nb = min(kBtcTile, nblocks - tile);
      for (uint32_t b = w; b < nb; b += kBtcWarps) {
        const uint32_t e0 = (tile + b) * kBtcBlock;
        const uint32_t nv = min(kBtcBlock, n_elems - e0);
        uint32_t d;
        switch (ts) {
          case 1: d = btc_analyse_block<1>(algo, (const uint8_t*)in + e0, nv, lane); break;
          case 2: d = btc_analyse_block<2>(algo, (const uint16_t*)in + e0, nv, lane); break;
          case 4: d = btc_analyse_block<4>(algo, (const uint32_t*)in + e0, nv, lane); break;
          default: d = btc_analyse_block<8>(algo, (const uint64_t*)in + e0, nv, lane); break;
        }
        if (lane == 0) { s_desc[b] = (uint16_t)d; desc[tile + b] = (uint16_t)d; }
      }
      __syncthreads();
      uint32_t sz[4], ex[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t b = 4 * threadIdx.x + j;
        sz[j] = (b < nb) ? btc_block_bytes(algo, s_desc[b]) : 0u;
      }
      const uint32_t total = btc_block_scan4(sz, ex, s_scratch);
#pragma unroll
      for (int j = 0; j < 4; ++j) s_off[4 * threadIdx.x + j] = base_off + ex[j];
      __syncthreads();
      for (uint32_t b = w; b < nb; b += kBtcWarps) {
        const uint32_t e0 = (tile + b) * kBtcBlock;
        const uint32_t nv = min(kBtcBlock, n_elems - e0);
        uint8_t* payload = out + s_off[b];
        const uint32_t d = s_desc[b];
        switch (ts) {
          case 1: btc_pack_block<1>(algo, d, (const uint8_t*)in + e0, nv, payload, s_words[w], lane); break;
          case 2: btc_pack_block<2>(algo, d, (const uint16_t*)in + e0, nv, payload, s_words[w], lane); break;
          case 4: btc_pack_block<4>(algo, d, (const uint32_t*)in + e0, nv, payload, s_words[w], lane); break;
          default: btc_pack_block<8>(algo, d, (const uint64_t*)in + e0, nv, payload, s_words[w], lane); break;
        }
      }
      base_off += total;
      __syncthreads();
    }
    const uint32_t tail = n_bytes - n_elems * ts;
    if (tail && threadIdx.x < 8) out[base_off + threadIdx.x] = threadIdx.x < tail ? in[n_elems * ts + threadIdx.x] : (uint8_t)0;
    if (threadIdx.x == 0) out_bytes[c] = base_off + (tail ? 8u : 0u);
    __syncthreads();
  }
}

inline nvcompStatus_t btc_check_opts(const nvcompBatchedBitcompFormatOpts& o) {
  if (btc_type_size(o.data_type) == 0) return nvcompErrorInvalidValue;
  if (o.algorithm_type < 0 || o.algorithm_type > 1) return nvcompErrorInvalidValue;
  return nvcompSuccess;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedBitcompCompressGetTempSize(
    size_t, size_t max_chunk, nvcompBatchedBitcompFormatOpts opts, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = btc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompBitcompCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompCompressGetTempSizeEx(
    size_t b, size_t m, nvcompBatchedBitcompFormatOpts o, size_t* t, const size_t) {
  return nvcompBatchedBitcompCompressGetTempSize(b, m, o, t);
}

nvcompStatus_t nvcompBatchedBitcompCompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedBitcompFormatOpts opts, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = btc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompBitcompCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  const size_t ts = btc_type_size(opts.data_type);
  const size_t n = max_chunk / ts;
  const size_t nblocks = (n + kBtcBlock - 1) / kBtcBlock;
  // header + descriptors + per block: 16 bytes of header/mask + 128 elements at full width
  // (+ the trailing-bytes word)
  *max_compressed_bytes = 16 + ((2 * nblocks + 7) & ~(size_t)7) + nblocks * (16 + kBtcBlock * ts) + 16;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompCompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedBitcompFormatOpts opts, cudaStream_t stream) {
  log_call("nvcompBatchedBitcompCompressAsync", batch, max_chunk, stream);
  const nvcompStatus_t st = btc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompBitcompCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const int grid = persistent_grid(8, batch, 1);
  bitcomp_compress_kernel<<<grid, kBtcThreads, 0, stream>>>(
      in_ptrs, in_bytes, batch, out_ptrs, out_bytes, opts.algorithm_type, (int)opts.data_type, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompDecompressGetTempSizeEx(size_t n, size_t m, size_t* t, size_t) {
  return nvcompBatchedBitcompDecompressGetTempSize(n, m, t);
}

nvcompStatus_t nvcompBatchedBitcompGetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedBitcompGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  bitcomp_size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompDecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedBitcompDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const int grid = persistent_grid(12, batch, 1);
  bitcomp_decompress_kernel<<<grid, kBtcThreads, 0, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"
