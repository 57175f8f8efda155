// cascaded.cu -- batched Cascaded codec (RLE x n, delta x m, frame-of-reference
// bit-packing) for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedCascaded* entry points
// (include/nvcomp/cascaded.h; reference benchmarks/benchmark_cascaded_chunked.cu:138-142).
// Algorithm: reference doc/cascaded_overview.md:7-42 -- RLE and delta layers are
// interleaved (values out of RLE i feed delta i), then every resulting stream
// (all run-length streams and the final value stream) is bit-packed against its
// minimum.  The reference bitstream is undocumented, so this is our own:
//
// Chunk stream (8-byte aligned):
//   u32 magic 'CSC1' | u8 type | u8 num_RLEs | u8 num_deltas | u8 use_bp
//   u32 uncompressed_bytes, u32 part_bytes, u32 num_parts
//   u32 part_off[num_parts+1]      byte offsets of each partition payload (8-aligned)
//   zero pad to 8 bytes (4 bytes when num_parts is odd)
//   partition payloads
//   if uncompressed_bytes is not a multiple of the element size: one 8-byte word at part_off[num_parts]
//   with the trailing uncompressed_bytes % size bytes verbatim (partitions cover the whole elements)
// Partition payload (independent, opts.chunk_size bytes of input each):
//   u64 first[num_deltas]          first value removed by delta layer i
//   stream runs_0 .. runs_{R-1}, stream vals
// Stream: u32 count, u32 bits, u64 min, then ceil(count*bits/64) u64 words;
//   value k = min + bits [k*bits, (k+1)*bits) (little-endian bit order).
//   use_bp = 0 forces bits = 8*sizeof(T) (runs: 16), min = 0.
//
// Decode: one CTA per chunk (persistent ticket), one warp per partition; all
// layers run out of shared memory (unpack -> warp-tile prefix sums -> run
// expansion by head-flag scatter + max-scan) and the partition is written once
// with coalesced stores.
#include "common.cuh"
#include "nvcomp/cascaded.h"

namespace b200 {

constexpr uint32_t kCascMagic = 0x31435343u;  // "CSC1"
constexpr int kCascWarps = 16;       // decode CTA: up to 16 warps, one partition each
#ifndef CASC_DEC_CTAS
#define CASC_DEC_CTAS 2
#endif
// decode CTAs per SM (96 KB of shared memory each).  2 CTAs cap the kernel at 64 registers and it spills; on H100 it
// is still 14 % faster than 1 CTA at 125 registers without spills
constexpr int kCascDecCtasPerSm = CASC_DEC_CTAS;
constexpr int kCascCompWarps = 4;    // compress CTA
constexpr uint32_t kCascMaxPart = 16384;
// per-warp shared memory of the decoder: one value buffer (P bytes; two when more than one layer pair
// is configured) + a run-index u16 array (2 * P/TS bytes).  The CTA owns 96 KB and activates as many
// warps (<= 16) as fit: 16 for 4/8-byte elements with one layer pair and 4 KB partitions, ... 1 for a
// 16 KB partition of 1-byte elements.
constexpr uint32_t kCascSmem = 96 * 1024;

__host__ __device__ inline uint32_t casc_type_size(int t) {
  switch (t) {
    case NVCOMP_TYPE_CHAR: case NVCOMP_TYPE_UCHAR: return 1;
    case NVCOMP_TYPE_SHORT: case NVCOMP_TYPE_USHORT: return 2;
    case NVCOMP_TYPE_INT: case NVCOMP_TYPE_UINT: return 4;
    case NVCOMP_TYPE_LONGLONG: case NVCOMP_TYPE_ULONGLONG: return 8;
    default: return 0;
  }
}
__host__ __device__ inline bool casc_type_signed(int t) {
  return t == NVCOMP_TYPE_CHAR || t == NVCOMP_TYPE_SHORT || t == NVCOMP_TYPE_INT || t == NVCOMP_TYPE_LONGLONG;
}

__device__ __forceinline__ uint32_t warp_incl_max_u32(uint32_t v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t o = __shfl_up_sync(kFull, v, d);
    if (lane >= d) v = max(v, o);
  }
  return v;
}

// Inclusive warp scans of a lane total (add / max); the loops below block 4 consecutive elements per
// lane, so one scan serves 128 elements.
template <class S>
__device__ __forceinline__ S warp_incl_scan(S v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const S o = __shfl_up_sync(kFull, v, d);
    if (lane >= d) v += o;
  }
  return v;
}

template <int TS> struct ScanType { using S = uint32_t; };
template <> struct ScanType<8> { using S = uint64_t; };

// four consecutive elements of type T (16-byte vector accesses when 4*sizeof(T) >= 16)
template <class T>
struct alignas(sizeof(T) * 4 > 16 ? 16 : sizeof(T) * 4) Quad4 { T e[4]; };

// typed smem element access with values carried as u64 (wrapping arithmetic)
template <int TS> struct Elem;
template <> struct Elem<1> { using T = uint8_t; };
template <> struct Elem<2> { using T = uint16_t; };
template <> struct Elem<4> { using T = uint32_t; };
template <> struct Elem<8> { using T = uint64_t; };

template <int TS> __device__ __forceinline__ uint64_t sext(uint64_t v) {
  if (TS == 8) return v;
  const int sh = 64 - 8 * TS;
  return (uint64_t)(((int64_t)(v << sh)) >> sh);
}

// ----- packed stream reader ---------------------------------------------------
struct StreamHdr { uint32_t count, bits; uint64_t minv; };

__device__ __forceinline__ uint64_t unpack_at(const uint64_t* __restrict__ words, uint32_t k,
                                              uint32_t bits, uint64_t minv) {
  if (bits == 0) return minv;
  const uint64_t bitpos = (uint64_t)k * bits;
  const uint32_t w = (uint32_t)(bitpos >> 6), s = (uint32_t)(bitpos & 63);
  uint64_t v = __ldg(words + w) >> s;
  if (s + bits > 64) v |= __ldg(words + w + 1) << (64 - s);
  if (bits < 64) v &= ((1ull << bits) - 1ull);
  return v + minv;
}

// bits <= 32: the stream is read as 32-bit words, one funnel shift per value (bits is uniform over a
// stream, so callers branch once per stream, not per value)
__device__ __forceinline__ uint64_t unpack32_at(const uint32_t* __restrict__ w32, uint32_t k,
                                                uint32_t bits, uint32_t mask, uint64_t minv) {
  const uint32_t bitpos = k * bits;                  // < 2^19: count <= 16384, bits <= 32
  const uint32_t w = bitpos >> 5, s = bitpos & 31u;
  const uint32_t lo = __ldg(w32 + w);
  const uint32_t hi = (s + bits > 32u) ? __ldg(w32 + w + 1) : 0u;
  return (uint64_t)(__funnelshift_r(lo, hi, s) & mask) + minv;
}

__host__ __device__ inline uint32_t stream_bytes(uint32_t count, uint32_t bits) {
  return 16u + 8u * (uint32_t)(((uint64_t)count * bits + 63) / 64);
}

// ---------------------------------------------------------------------------
// Layer 0 of a configuration with run-length encoding, in one pass: the lane that owns four consecutive runs
// produces their values (straight from the packed stream when this is the only layer, else from the shared-memory
// buffer the layers above left; with a delta layer the exclusive prefix sum is taken on the fly), their start
// positions (prefix sum of the run lengths) and fills the runs into the staging buffer, which then leaves with
// coalesced 16-byte stores.  Two warp scans per 128 runs; no head-flag array, no max-scan, no gather.
// Shared memory is addressed with 32-bit window addresses (st.shared with immediate offsets).
// SRC: 0 packed stream of <= 32-bit values, 1 packed stream (any width), 2 shared-memory values.
// The run-length stream has <= 32-bit values (the caller checks).
// ---------------------------------------------------------------------------
template <int TS, int J>
__device__ __forceinline__ void sts_elem(uint32_t a, typename ScanType<TS>::S v) {
  if (TS == 1) asm volatile("st.shared.u8 [%0+%2], %1;" :: "r"(a), "r"((uint32_t)v), "n"(J * TS) : "memory");
  else if (TS == 2) asm volatile("st.shared.u16 [%0+%2], %1;" :: "r"(a), "h"((uint16_t)v), "n"(J * TS) : "memory");
  else if (TS == 4) asm volatile("st.shared.u32 [%0+%2], %1;" :: "r"(a), "r"((uint32_t)v), "n"(J * TS) : "memory");
  else asm volatile("st.shared.u64 [%0+%2], %1;" :: "r"(a), "l"((uint64_t)v), "n"(J * TS) : "memory");
}

// raw value k (without the stream minimum) of a stream of `bits` <= 32 bit values; k is inside the stream
__device__ __forceinline__ uint32_t unpack32_raw(const uint32_t* __restrict__ w32, uint32_t k, uint32_t bits, uint32_t mask) {
  const uint32_t bitpos = k * bits;                  // < 2^19: count <= 16384, bits <= 32
  const uint32_t w = bitpos >> 5, s = bitpos & 31u;
  const uint32_t lo = __ldg(w32 + w);               // (read-only path: LDG, not a generic load)
  const uint32_t hi = (s + bits > 32u) ? __ldg(w32 + w + 1) : 0u;
  return __funnelshift_r(lo, hi, s) & mask;
}

// raw values k0 .. k0+3 of such a stream (indices clamped to klast: what lies past it is never used).  Up to 8 bits per
// value the four lie inside two consecutive words: two loads and four 64-bit shifts instead of eight loads.
// nw32: 32-bit words the stream has.
__device__ __forceinline__ void unpack32_x4(const uint32_t* __restrict__ w32, uint32_t k0, uint32_t klast, uint32_t bits,
                                            uint32_t mask, uint32_t nw32, uint32_t r[4]) {
  if (bits <= 8u) {
    const uint32_t bitpos = min(k0, klast) * bits;
    const uint32_t w = bitpos >> 5, s = bitpos & 31u;
    const uint32_t lo = __ldg(w32 + w);
    const uint32_t hi = (s + 4u * bits > 32u && w + 1u < nw32) ? __ldg(w32 + w + 1) : 0u;
    const uint64_t x = ((uint64_t)hi << 32) | lo;
#pragma unroll
    for (int e = 0; e < 4; ++e) r[e] = (uint32_t)(x >> (s + (uint32_t)e * bits)) & mask;
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) r[e] = unpack32_raw(w32, min(k0 + e, klast), bits, mask);
  }
}

template <int TS, int SRC>
__device__ __forceinline__ bool casc_final_rle(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ vwords,
                                               const StreamHdr vh, const typename Elem<TS>::T* cur, uint32_t count,
                                               bool has_delta, uint64_t first, uint32_t c_in,
                                               const StreamHdr rh, const uint64_t* __restrict__ rwords,
                                               typename Elem<TS>::T* stage, uint32_t cap,
                                               uint8_t* out, uint32_t n_out, int lane) {
  using T = typename Elem<TS>::T;
  using S = typename ScanType<TS>::S;                  // 32-bit wrapping sums suffice for <= 4-byte elements
  uint32_t nvals = count;
  if (has_delta) {
    if (c_in == 0u) { if (count != 0u) return false; has_delta = false; }   // the layer saw an empty list
    else { if (c_in != count + 1u || c_in > cap) return false; nvals = count + 1u; }
  }
  if (rh.count != nvals) return false;
  if (nvals == 0u) return n_out == 0u;
  // an empty (0-bit) stream has no words: point the loads at the payload header instead, the mask drops what they read
  const uint32_t* const vw32 = vh.bits ? (const uint32_t*)vwords : (const uint32_t*)payload;
  const uint32_t vmask = vh.bits >= 32u ? 0xffffffffu : ((1u << vh.bits) - 1u);
  const S vmin = (S)vh.minv;
  const uint32_t vlast = count ? count - 1u : 0u;      // (count == 0: one value, no deltas; nothing is read)
  auto val = [&](uint32_t k) -> S {                    // k is clamped by the caller: every load stays inside the stream
    if (SRC == 0) return (S)unpack32_raw(vw32, k, vh.bits, vmask) + vmin;
    if (SRC == 1) return (S)unpack_at(vwords, k, vh.bits, vh.minv);
    return (S)cur[k];
  };
  const uint32_t* const rw32 = rh.bits ? (const uint32_t*)rwords : (const uint32_t*)payload;
  const uint32_t rmask = rh.bits >= 32u ? 0xffffffffu : ((1u << rh.bits) - 1u);
  const uint32_t rlast = nvals - 1u;
  const uint32_t vnw32 = (uint32_t)(((uint64_t)count * vh.bits + 63u) >> 6) << 1;   // 32-bit words of the two streams
  const uint32_t rnw32 = (uint32_t)(((uint64_t)nvals * rh.bits + 63u) >> 6) << 1;
  const uint32_t stage_s = smem_addr(stage);
  S vcarry = (S)first;
  uint32_t lcarry = 0;
  for (uint32_t base = 0; base < nvals; base += 4u * kWarp) {
    const uint32_t k0 = base + 4u * (uint32_t)lane;
    S v[4];
    if (has_delta) {
      // value k = first + sum of the deltas before it (k = 0 .. count).  Deltas read past the last one (clamped
      // index) only reach values past the last one, which no run stores.
      S d[4];
      if (SRC == 0) {
        uint32_t r4[4] = {0u, 0u, 0u, 0u};
        if (count != 0u) unpack32_x4(vw32, k0, vlast, vh.bits, vmask, vnw32, r4);
#pragma unroll
        for (int e = 0; e < 4; ++e) d[e] = (count != 0u) ? (S)r4[e] + vmin : (S)0;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) d[e] = (count != 0u) ? val(min(k0 + e, vlast)) : (S)0;
      }
      const S x2 = d[0] + d[1], x3 = x2 + d[2], tot = x3 + d[3];
      const S incl = warp_incl_scan<S>(tot, lane);
      const S ex = incl - tot + vcarry;
      v[0] = ex; v[1] = ex + d[0]; v[2] = ex + x2; v[3] = ex + x3;
      vcarry += __shfl_sync(kFull, incl, 31);
    } else {
      if (SRC == 0) {
        uint32_t r4[4];
        unpack32_x4(vw32, k0, vlast, vh.bits, vmask, vnw32, r4);
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = (S)r4[e] + vmin;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = val(min(k0 + e, vlast));
      }
    }
    uint32_t len[4];
    unpack32_x4(rw32, k0, rlast, rh.bits, rmask, rnw32, len);
    bool zero = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // the length is the full 64-bit raw + min, clipped to cap + 1 (no wrap-around in the sums below)
      len[e] = (k0 + e < nvals) ? (uint32_t)min((uint64_t)len[e] + rh.minv, (uint64_t)cap + 1u) : 0u;
      zero |= k0 + e < nvals && len[e] == 0u;
    }
    if (__any_sync(kFull, zero)) return false;         // a run of length 0
    const uint32_t ltot = len[0] + len[1] + len[2] + len[3];
    const uint32_t lincl = warp_incl_scan<uint32_t>(ltot, lane);
    const uint32_t pos0 = lincl - ltot + lcarry;
    lcarry += __shfl_sync(kFull, lincl, 31);
    if (lcarry > cap) return false;                   // every store below stays inside the staging buffer
    // fill: the owner writes the first eight elements of each run (two at a time while any run of the warp is that
    // long), the whole warp what a longer run has beyond
    const uint32_t mx = max(max(len[0], len[1]), max(len[2], len[3]));
    const unsigned m2 = __ballot_sync(kFull, mx > 2u);
    uint32_t addr[4];
    addr[0] = stage_s + (uint32_t)TS * pos0;
    addr[1] = addr[0] + (uint32_t)TS * len[0];
    addr[2] = addr[1] + (uint32_t)TS * len[1];
    addr[3] = addr[2] + (uint32_t)TS * len[2];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (len[e] > 0u) sts_elem<TS, 0>(addr[e], v[e]);
      if (len[e] > 1u) sts_elem<TS, 1>(addr[e], v[e]);
    }
    if (m2) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (len[e] > 2u) sts_elem<TS, 2>(addr[e], v[e]);
        if (len[e] > 3u) sts_elem<TS, 3>(addr[e], v[e]);
      }
      if (__any_sync(kFull, mx > 4u)) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (len[e] > 4u) sts_elem<TS, 4>(addr[e], v[e]);
          if (len[e] > 5u) sts_elem<TS, 5>(addr[e], v[e]);
          if (len[e] > 6u) sts_elem<TS, 6>(addr[e], v[e]);
          if (len[e] > 7u) sts_elem<TS, 7>(addr[e], v[e]);
        }
        unsigned longm = __ballot_sync(kFull, mx > 8u);
        while (longm) {
          const int t = __ffs((int)longm) - 1;
          longm &= longm - 1u;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const uint32_t tl = __shfl_sync(kFull, len[e], t), ta = __shfl_sync(kFull, addr[e], t);
            const S tv = __shfl_sync(kFull, v[e], t);
            for (uint32_t j = 8u + (uint32_t)lane; j < tl; j += kWarp) sts_elem<TS, 0>(ta + (uint32_t)TS * j, tv);
          }
        }
      }
    }
  }
  const uint32_t total = lcarry;
  if (total < nvals || total != n_out) return false;
  __syncwarp();
  // coalesced write-out
  const uint32_t nbytes = total * (uint32_t)TS;
  if ((((uintptr_t)out | stage_s) & 15u) == 0u) {
    uint32_t j = 16u * (uint32_t)lane;
    for (; j + 16u * kWarp + 16u <= nbytes; j += 32u * kWarp) {      // two vectors per lane in flight
      const uint4 x0 = lds_v4(stage_s + j), x1 = lds_v4(stage_s + j + 16u * kWarp);
      st_v4((uint4*)(out + j), x0);
      st_v4((uint4*)(out + j + 16u * kWarp), x1);
    }
    for (; j + 16u <= nbytes; j += 16u * kWarp) st_v4((uint4*)(out + j), lds_v4(stage_s + j));
    for (uint32_t t = (nbytes & ~15u) + (uint32_t)lane; t < nbytes; t += kWarp) out[t] = (uint8_t)lds_u8(stage_s + t);
  } else {
    T* const o = (T*)out;
    for (uint32_t k = lane; k < total; k += kWarp) o[k] = stage[k];
  }
  return true;
}

// The first (up to) 256 bytes of a partition payload -- delta bases, element counts, the stream headers of a compressed
// partition -- are fetched with two independent coalesced loads and parked in the warp's (still unused) staging
// buffer; header fields are then shared-memory reads instead of one dependent global miss after the other (the walk
// decides where the next header lies).  Offsets beyond the window fall back to a global load.
struct CascHead {
  uint32_t n, scratch;
  const uint8_t* base;
  __device__ __forceinline__ CascHead(const uint8_t* __restrict__ payload, uint32_t payload_bytes, uint32_t scratch_s, int lane) {
    base = payload;
    scratch = scratch_s;
    n = min(payload_bytes & ~3u, 256u);
    const uint32_t* p32 = (const uint32_t*)payload;       // (8-byte aligned)
    const uint32_t w0 = (4u * (uint32_t)lane + 4u <= n) ? __ldg(p32 + lane) : 0u;
    const uint32_t w1 = (4u * (uint32_t)lane + 132u <= n) ? __ldg(p32 + 32 + lane) : 0u;
    sts_u32(scratch_s + 4u * (uint32_t)lane, w0);
    sts_u32(scratch_s + 128u + 4u * (uint32_t)lane, w1);
    __syncwarp();
  }
  // off: the same in every lane, a multiple of 4, off + 4 <= payload bytes
  __device__ __forceinline__ uint32_t u32(uint32_t off) const {
    return (off + 4u <= n) ? lds_u32(scratch + off) : __ldg((const uint32_t*)(base + off));
  }
  __device__ __forceinline__ uint64_t u64(uint32_t off) const { return (uint64_t)u32(off) | ((uint64_t)u32(off + 4u) << 32); }
};

// ---------------------------------------------------------------------------
// Decode one partition with one warp.  `n_out` elements expected.
// sm layout (per warp): A [P] | (B [P] when two_bufs) | idx u16[P/TS]
// Delta layers are undone in place; the outermost run-length expansion writes straight to the
// output (global memory), so the common one-layer configurations need a single value buffer.
// Returns false on a malformed partition.
// ---------------------------------------------------------------------------
template <int TS>
__device__ bool casc_decode_part(const uint8_t* __restrict__ payload, uint32_t payload_bytes,
                                 uint8_t* out, uint32_t n_out, int R, int D,
                                 uint8_t* sm, uint32_t P, bool two_bufs, int lane) {
  using T = typename Elem<TS>::T;
  T* bufA = (T*)sm;
  T* bufB = (T*)(sm + P);                    // only valid when two_bufs
  const uint32_t cap = P / TS;
  uint16_t* idx = (uint16_t*)(sm + (two_bufs ? 2u : 1u) * P);
  if (n_out > cap) return false;

  // walk stream headers
  const uint32_t firsts_bytes = 8u * (uint32_t)D + ((4u * (uint32_t)D + 7u) & ~7u);
  if (payload_bytes < firsts_bytes) return false;
  const uint64_t* firsts = (const uint64_t*)payload;
  const uint32_t* cin = (const uint32_t*)(payload + 8u * (uint32_t)D);   // element count entering delta i
  // The first 256 bytes of the payload (delta bases, element counts, the stream headers of a compressed partition) come
  // in with two independent coalesced loads; header fields are then picked with shuffles instead of one dependent
  // global load after the other (a miss each: the walk below decides where the next header lies).
  // (no per-layer arrays: a dynamically indexed local array lives in local memory; the header of run stream 0 --
  // the only one the common configurations have -- stays in registers, deeper layers walk the headers again)
  const CascHead head(payload, payload_bytes, smem_addr(sm), lane);
  // (every field is in a register before anything is written to the staging buffer: __syncwarp below)
  uint32_t off = firsts_bytes;
  StreamHdr rh0; rh0.count = 0; rh0.bits = 0; rh0.minv = 0;
  uint32_t roff0 = 0;
#pragma unroll 1
  for (int i = 0; i < R; ++i) {
    if (off + 16 > payload_bytes) return false;
    const uint32_t cnt = head.u32(off), bits = head.u32(off + 4u);
    if (bits > 64 || cnt > cap) return false;
    if (i == 0) { rh0.count = cnt; rh0.bits = bits; rh0.minv = head.u64(off + 8u); roff0 = off + 16; }
    off += stream_bytes(cnt, bits);
    if (off > payload_bytes) return false;
  }
  if (off + 16 > payload_bytes) return false;
  StreamHdr vh;
  vh.count = head.u32(off); vh.bits = head.u32(off + 4u);
  vh.minv = head.u64(off + 8u);
  if (vh.bits > 64 || vh.count > cap) return false;
  const uint64_t* vwords = (const uint64_t*)(payload + off + 16);
  if (off + stream_bytes(vh.count, vh.bits) > payload_bytes) return false;

  const uint64_t first0 = D > 0 ? head.u64(0u) : 0ull;          // base and element count of delta layer 0
  const uint32_t cin0 = D > 0 ? head.u32(8u * (uint32_t)D) : 0u;
  __syncwarp();                                                // the header window is dead: the buffer may be written

  uint32_t count = vh.count;
  const int L = R > D ? R : D;
  if (L == 1 && R == 1 && rh0.bits <= 32u) {
    // the common configuration (one run-length layer, at most one delta layer): straight from the packed streams
    const uint64_t* rwords = (const uint64_t*)(payload + roff0);
    const bool hd = D > 0;
    const uint64_t first = first0;
    const uint32_t c_in = cin0;
    if (vh.bits <= 32u)
      return casc_final_rle<TS, 0>(payload, vwords, vh, nullptr, count, hd, first, c_in, rh0, rwords, bufA, cap, out, n_out, lane);
    return casc_final_rle<TS, 1>(payload, vwords, vh, nullptr, count, hd, first, c_in, rh0, rwords, bufA, cap, out, n_out, lane);
  }
  // unpack the final value stream into A
  if (vh.bits != 0u && vh.bits <= 32u) {
    const uint32_t* w32 = (const uint32_t*)vwords;
    const uint32_t mask = vh.bits == 32u ? 0xffffffffu : ((1u << vh.bits) - 1u);
    for (uint32_t k = lane; k < count; k += kWarp) bufA[k] = (T)unpack32_at(w32, k, vh.bits, mask, vh.minv);
  } else {
    for (uint32_t k = lane; k < count; k += kWarp) bufA[k] = (T)unpack_at(vwords, k, vh.bits, vh.minv);
  }
  __syncwarp();
  T* cur = bufA;
  for (int i = L - 1; i >= 0; --i) {
    if (i == 0 && R > 0 && rh0.bits <= 32u) {
      // layer 0 with run-length encoding: fused delta + expansion from the buffer the layers above left
      const uint64_t* rwords = (const uint64_t*)(payload + roff0);
      const bool hd = D > 0;
      return casc_final_rle<TS, 2>(payload, nullptr, vh, cur, count, hd, first0, cin0, rh0, rwords,
                                   cur == bufA ? bufB : bufA, cap, out, n_out, lane);
    }
    if (i < D) {
      // undo delta i in place: cur[0..count) deltas -> cur[0..count] values.  cin == 0: the layer saw
      // an empty list.
      const uint32_t c_in = cin[i];
      if (c_in == 0 && count != 0) return false;
      if (c_in != 0) {
        if (c_in != count + 1 || c_in > cap) return false;
        // Exclusive scan in place: out[k] = first + sum(d[0..k)), k = 0..count.  Each lane owns four
        // consecutive elements (one vector load / store, one warp scan per 128 elements); element k
        // is read and written by the same lane, so the pass needs no staging.
        using S = typename ScanType<TS>::S;          // 32-bit wrapping sums suffice for <= 4-byte elements
        S carry = (S)firsts[i];
        const bool vec_ok = (cap & 3u) == 0u && ((uintptr_t)cur & 15u) == 0u;   // quads inside the buffer, aligned
        for (uint32_t base = 0; base <= count; base += 4u * kWarp) {
          const uint32_t k0 = base + 4u * (uint32_t)lane;
          Quad4<T> q;
          if (vec_ok && k0 < cap) q = *(const Quad4<T>*)(cur + k0);
          else {
#pragma unroll
            for (int e = 0; e < 4; ++e) q.e[e] = (k0 + e < cap) ? cur[k0 + e] : (T)0;
          }
          S d0 = (k0 + 0 < count) ? (S)q.e[0] : (S)0, d1 = (k0 + 1 < count) ? (S)q.e[1] : (S)0;
          S d2 = (k0 + 2 < count) ? (S)q.e[2] : (S)0, d3 = (k0 + 3 < count) ? (S)q.e[3] : (S)0;
          const S x1 = d0, x2 = d0 + d1, x3 = x2 + d2, tot = x3 + d3;
          const S incl = warp_incl_scan<S>(tot, lane);
          const S ex = incl - tot + carry;
          q.e[0] = (T)ex; q.e[1] = (T)(ex + x1); q.e[2] = (T)(ex + x2); q.e[3] = (T)(ex + x3);
          if (vec_ok && k0 + 3u <= count) *(Quad4<T>*)(cur + k0) = q;
          else {
#pragma unroll
            for (int e = 0; e < 4; ++e) if (k0 + e <= count) cur[k0 + e] = q.e[e];
          }
          carry += __shfl_sync(kFull, incl, 31);
        }
        count += 1;
        __syncwarp();
      }
    }
    if (i < R) {
      // expand with runs_i: cur holds `count` values, runs_i holds `count` lengths
      // header of run stream i (validated by the walk above)
      StreamHdr rh = rh0;
      uint32_t roff = roff0;
      for (int k = 1; k <= i; ++k) {
        const uint32_t o = roff - 16u + stream_bytes(rh.count, rh.bits);
        const uint32_t* h = (const uint32_t*)(payload + o);
        rh.count = h[0]; rh.bits = h[1]; rh.minv = *(const uint64_t*)(payload + o + 8);
        roff = o + 16u;
      }
      if (rh.count != count) return false;
      const bool last = (i == 0);
      if (!last && !two_bufs) return false;                  // cannot happen: one buffer only when L == 1
      T* dst = last ? (T*)out : (cur == bufA ? bufB : bufA);
      const uint64_t* rwords = (const uint64_t*)(payload + roff);
      // head flags: idx[start of run k] = k, zero elsewhere
      {
        uint32_t* z = (uint32_t*)idx;
        for (uint32_t j = lane; j < (cap + 1) / 2; j += kWarp) z[j] = 0u;
      }
      __syncwarp();
      // run starts: each lane owns four consecutive runs (one warp scan per 128 runs)
      uint32_t carry = 0;
      const bool narrow = rh.bits != 0u && rh.bits <= 32u;
      const uint32_t* rw32 = (const uint32_t*)rwords;
      const uint32_t rmask = rh.bits >= 32u ? 0xffffffffu : ((1u << rh.bits) - 1u);
      for (uint32_t base = 0; base < count; base += 4u * kWarp) {
        const uint32_t k0 = base + 4u * (uint32_t)lane;
        uint32_t len[4];
        bool zero = false;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          uint64_t l = 0u;
          if (k0 + e < count) {
            l = narrow ? unpack32_at(rw32, k0 + e, rh.bits, rmask, rh.minv) : unpack_at(rwords, k0 + e, rh.bits, rh.minv);
            zero |= l == 0u;
          }
          len[e] = (uint32_t)min(l, (uint64_t)cap + 1u);   // the full 64-bit length, clipped: no wrap-around below
        }
        if (__any_sync(kFull, zero)) return false;     // a run of length 0
        const uint32_t p1 = len[0], p2 = p1 + len[1], p3 = p2 + len[2], tot = p3 + len[3];
        const uint32_t incl = warp_incl_scan<uint32_t>(tot, lane);
        const uint32_t ex = incl - tot + carry;
        carry += __shfl_sync(kFull, incl, 31);
        if (carry > cap) return false;
        if (k0 + 0 < count && len[0]) idx[ex] = (uint16_t)(k0 + 0);
        if (k0 + 1 < count && len[1]) idx[ex + p1] = (uint16_t)(k0 + 1);
        if (k0 + 2 < count && len[2]) idx[ex + p2] = (uint16_t)(k0 + 2);
        if (k0 + 3 < count && len[3]) idx[ex + p3] = (uint16_t)(k0 + 3);
      }
      const uint32_t total = carry;
      if (total > cap || total < count) return false;
      if (last && total != n_out) return false;
      __syncwarp();
      // run index of every output element: running maximum of the head flags, four consecutive
      // elements per lane (one warp max-scan per 128 outputs), written back over the flags ...
      uint32_t mcarry = 0;
      const bool ivec = ((uintptr_t)idx & 7u) == 0u;
      for (uint32_t base = 0; base < total; base += 4u * kWarp) {
        const uint32_t j0 = base + 4u * (uint32_t)lane;
        Quad4<uint16_t> q;
        if (ivec && j0 < (cap & ~3u)) q = *(const Quad4<uint16_t>*)(idx + j0);
        else {
#pragma unroll
          for (int e = 0; e < 4; ++e) q.e[e] = (j0 + e < cap) ? idx[j0 + e] : (uint16_t)0;
        }
        const uint32_t m0 = q.e[0], m1 = max(m0, (uint32_t)q.e[1]), m2 = max(m1, (uint32_t)q.e[2]),
                       m3 = max(m2, (uint32_t)q.e[3]);
        const uint32_t incl = warp_incl_max_u32(m3, lane);
        uint32_t ex = __shfl_up_sync(kFull, incl, 1);
        ex = max(lane ? ex : 0u, mcarry);
        q.e[0] = (uint16_t)max(ex, m0); q.e[1] = (uint16_t)max(ex, m1);
        q.e[2] = (uint16_t)max(ex, m2); q.e[3] = (uint16_t)max(ex, m3);
        if (ivec && j0 < (cap & ~3u)) *(Quad4<uint16_t>*)(idx + j0) = q;
        else {
#pragma unroll
          for (int e = 0; e < 4; ++e) if (j0 + e < cap) idx[j0 + e] = q.e[e];
        }
        mcarry = max(mcarry, __shfl_sync(kFull, incl, 31));
      }
      __syncwarp();
      // ... then a coalesced gather: consecutive lanes write consecutive outputs
      for (uint32_t j = lane; j < total; j += kWarp) dst[j] = cur[idx[j]];
      if (last) return true;
      count = total;
      __syncwarp();
      cur = dst;
    }
  }
  if (count != n_out) return false;
  // coalesced write-out (out is at least TS-aligned: chunk pointers are 8-aligned
  // and partitions are multiples of TS)
  T* o = (T*)out;
  for (uint32_t k = lane; k < count; k += kWarp) o[k] = cur[k];
  return true;
}

struct CascHeader {
  uint32_t magic, uncompressed, part_bytes, num_parts;
  int type, R, D, bp;
};

// the five header words -> fields + validation
__device__ __forceinline__ bool casc_parse_header(uint32_t w0, uint32_t cfg, uint32_t w2, uint32_t w3, uint32_t w4,
                                                  size_t in_bytes, CascHeader& h) {
  h.magic = w0;
  h.type = cfg & 0xff; h.R = (cfg >> 8) & 0xff; h.D = (cfg >> 16) & 0xff; h.bp = (cfg >> 24) & 0xff;
  h.uncompressed = w2; h.part_bytes = w3; h.num_parts = w4;
  if (h.magic != kCascMagic) return false;
  const uint32_t ts = casc_type_size(h.type);
  if (ts == 0 || h.R > 7 || h.D > 7) return false;
  // the same limits the compressor enforces: the decoder carves 16-byte aligned shared-memory arrays out of it
  if (h.part_bytes < 512 || h.part_bytes > kCascMaxPart || (h.part_bytes % 8)) return false;
  const uint32_t whole = h.uncompressed - h.uncompressed % ts;      // bytes of whole elements
  if ((uint64_t)h.num_parts * h.part_bytes < whole) return false;
  if (h.num_parts && (uint64_t)(h.num_parts - 1) * h.part_bytes >= whole) return false;
  if (20ull + 4ull * (h.num_parts + 1ull) > in_bytes) return false;
  return true;
}

__device__ __forceinline__ bool casc_read_header(const uint8_t* in, size_t in_bytes, CascHeader& h) {
  if (in_bytes < 20 || ((uintptr_t)in & 7)) return false;
  const uint32_t* w = (const uint32_t*)in;
  return casc_parse_header(w[0], w[1], w[2], w[3], w[4], in_bytes, h);
}

__global__ void __launch_bounds__(kCascWarps * 32, kCascDecCtasPerSm)
cascaded_decompress_kernel(const void* const* __restrict__ comp_ptrs,
                           const size_t* __restrict__ comp_bytes,
                           const size_t* __restrict__ out_caps,
                           size_t* actual_bytes, size_t batch,
                           void* const* __restrict__ out_ptrs,
                           nvcompStatus_t* statuses,
                           unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  // Chunk indices and failure flags live in a ring of three slots: thread 0 draws the ticket two chunks ahead while
  // this one decodes and parks it just before the one barrier per chunk, so no warp ever waits for the atomic.
  // The descriptor of a chunk (stream pointer and size, output pointer and capacity) is fetched one chunk ahead by
  // four lanes of warp 1 -- loads issued at the top of the loop, parked in shared memory before the barrier -- so the
  // sixteen warps do not start every chunk with a miss on the four descriptor arrays.
  __shared__ unsigned long long s_chunk[3];
  __shared__ unsigned long long s_desc[3][4];
  __shared__ int s_fail[3];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  auto load_desc = [&](size_t c, int which) -> unsigned long long {
    return which == 0 ? (unsigned long long)comp_ptrs[c] : which == 1 ? (unsigned long long)comp_bytes[c]
         : which == 2 ? (unsigned long long)out_ptrs[c] : (unsigned long long)out_caps[c];
  };
  unsigned long long static_next = blockIdx.x;
  if (threadIdx.x == 0) {
    s_chunk[0] = ticket ? atomicAdd(ticket, 1ull) : static_next;
    s_chunk[1] = ticket ? atomicAdd(ticket, 1ull) : static_next + gridDim.x;
    s_fail[0] = 0; s_fail[1] = 0;
  }
  static_next += 2ull * gridDim.x;
  __syncthreads();
  if (w == 1 && lane < 4 && s_chunk[0] < batch) s_desc[0][lane] = load_desc((size_t)s_chunk[0], lane);
  __syncthreads();
  for (uint32_t cur = 0, nxt = 1, nn = 2;; ) {
    const size_t c = (size_t)s_chunk[cur];
    if (c >= batch) break;
    // the ticket two chunks ahead is drawn now and parked before the barrier: warp 0 does not wait for the atomic
    unsigned long long drawn = static_next;
    if (threadIdx.x == 0 && ticket) drawn = atomicAdd(ticket, 1ull);
    static_next += gridDim.x;
    unsigned long long pre = 0;                        // the next chunk's descriptor word of this lane (warp 1)
    const bool pre_lane = w == 1 && lane < 4 && s_chunk[nxt] < batch;
    if (pre_lane) pre = load_desc((size_t)s_chunk[nxt], lane);
    const uint8_t* in = (const uint8_t*)s_desc[cur][0];
    const size_t in_bytes = (size_t)s_desc[cur][1];
    uint8_t* out = (uint8_t*)s_desc[cur][2];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    const size_t cap = (size_t)s_desc[cur][3];
    // the chunk header and the first 27 partition offsets in one coalesced load (lane l holds word l of the chunk);
    // fields are broadcast with shuffles: one miss instead of a header miss followed by an offset miss
    CascHeader h;
    bool ok = in_bytes >= 20 && ((uintptr_t)in & 7) == 0;
    uint32_t cw = 0;
    if (ok && 4u * (uint32_t)lane + 4u <= in_bytes) cw = __ldg((const uint32_t*)in + lane);
    ok = ok && casc_parse_header(__shfl_sync(kFull, cw, 0), __shfl_sync(kFull, cw, 1), __shfl_sync(kFull, cw, 2),
                                 __shfl_sync(kFull, cw, 3), __shfl_sync(kFull, cw, 4), in_bytes, h);
    if (ok && (h.uncompressed > cap || ((uintptr_t)out & (casc_type_size(h.type) - 1)))) ok = false;
    if (ok) {
      const uint32_t* part_off = (const uint32_t*)(in + 20);
      const uint32_t ts0 = casc_type_size(h.type);
      const uint32_t P = h.part_bytes;
      const bool two_bufs = (h.R > h.D ? h.R : h.D) > 1;
      const uint32_t need = ((two_bufs ? 2u : 1u) * P + 2u * (P >> (__ffs((int)ts0) - 1)) + 4u + 15u) & ~15u;
      const int nw = 16u * need <= kCascSmem ? kCascWarps : (int)(kCascSmem / need);   // (kCascWarps == 16)
      uint8_t* sm = smem + (size_t)w * need;
      if (w < nw) {
        for (uint32_t p = w; p < h.num_parts; p += nw) {
          uint32_t o0, o1;
          if (p + 6u < 32u) { o0 = __shfl_sync(kFull, cw, (int)(p + 5u)); o1 = __shfl_sync(kFull, cw, (int)(p + 6u)); }
          else { o0 = part_off[p]; o1 = part_off[p + 1]; }
          bool pok = (o0 & 7) == 0 && o0 <= o1 && o1 <= in_bytes;
          if (pok) {
            const uint32_t begin = p * h.part_bytes;
            const uint32_t nbytes = min(h.part_bytes, h.uncompressed - h.uncompressed % ts0 - begin);
            switch (ts0) {
              case 1: pok = casc_decode_part<1>(in + o0, o1 - o0, out + begin, nbytes, h.R, h.D, sm, P, two_bufs, lane); break;
              case 2: pok = casc_decode_part<2>(in + o0, o1 - o0, out + begin, nbytes / 2, h.R, h.D, sm, P, two_bufs, lane); break;
              case 4: pok = casc_decode_part<4>(in + o0, o1 - o0, out + begin, nbytes / 4, h.R, h.D, sm, P, two_bufs, lane); break;
              default: pok = casc_decode_part<8>(in + o0, o1 - o0, out + begin, nbytes / 8, h.R, h.D, sm, P, two_bufs, lane); break;
            }
          }
          if (!pok && lane == 0) s_fail[cur] = 1;
          __syncwarp();
        }
      }
      // trailing bytes of a chunk whose length is not a multiple of the element size
      const uint32_t tail = h.uncompressed % ts0;
      if (tail && w == 0) {
        const uint32_t to = part_off[h.num_parts];
        if ((uint64_t)to + 8u > in_bytes) { if (lane == 0) s_fail[cur] = 1; }
        else if ((uint32_t)lane < tail) out[h.uncompressed - tail + lane] = in[to + lane];
      }
    }
    if (threadIdx.x == 0) { s_chunk[nn] = drawn; s_fail[nn] = 0; }
    if (pre_lane) s_desc[nxt][lane] = pre;
    __syncthreads();                                   // every partition of chunk c is done; the tickets are visible
    if (threadIdx.x == 0) {
      const bool good = ok && !s_fail[cur];
      const size_t c2 = (size_t)s_chunk[cur];
      if (actual_bytes) actual_bytes[c2] = good ? (size_t)h.uncompressed : 0;
      if (statuses) statuses[c2] = good ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    const uint32_t t = cur; cur = nxt; nxt = nn; nn = t;
  }
}

__global__ void cascaded_size_kernel(const void* const* __restrict__ comp_ptrs,
                                     const size_t* __restrict__ comp_bytes,
                                     size_t* out_sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= batch) return;
  CascHeader h;
  const bool ok = casc_read_header((const uint8_t*)comp_ptrs[c], comp_bytes[c], h);
  out_sizes[c] = ok ? (size_t)h.uncompressed : 0;
}

// ---------------------------------------------------------------------------
// Compression: one warp per chunk walks its partitions in order, so partition
// payloads are appended without a compaction pass.
// per-warp smem: A [P] | B [P] | pack words [2P + 64] | runs u16 [P elements]
// ---------------------------------------------------------------------------
template <int TS>
__device__ __forceinline__ uint64_t load_elem(const uint8_t* p, uint32_t k) {
  return (uint64_t)((const typename Elem<TS>::T*)p)[k];
}

// min/max over count values produced by f(k), signed or unsigned compare on TS bytes
template <int TS, bool SIGNED, class F>
__device__ __forceinline__ void warp_minmax(F f, uint32_t count, uint64_t& mn, uint64_t& mx, int lane) {
  uint64_t lo = ~0ull, hi = 0ull;   // in biased (order-preserving unsigned) space
  const uint64_t bias = SIGNED ? (1ull << 63) : 0ull;
  for (uint32_t k = lane; k < count; k += kWarp) {
    uint64_t v = f(k);
    v = (SIGNED ? sext<TS>(v) : v) ^ bias;
    lo = min(lo, v); hi = max(hi, v);
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    lo = min(lo, __shfl_xor_sync(kFull, lo, d));
    hi = max(hi, __shfl_xor_sync(kFull, hi, d));
  }
  mn = lo ^ bias; mx = hi ^ bias;
}

// Pack count values f(k) into dst (global, 8-aligned) via smem word buffer.
// Returns bytes written.  SIGNED selects the ordering used for the minimum.
template <int TS, class F>
__device__ uint32_t casc_pack_stream(F f, uint32_t count, bool use_bp, bool is_signed, uint32_t raw_bits,
                                     uint8_t* dst, unsigned long long* words, int lane) {
  uint64_t mn = 0, mx = 0;
  uint32_t bits = raw_bits;
  if (use_bp) {
    if (count == 0) { bits = 0; }
    else {
      if (is_signed) warp_minmax<TS, true>(f, count, mn, mx, lane);
      else warp_minmax<TS, false>(f, count, mn, mx, lane);
      const uint64_t range = mx - mn;   // wrapping subtract is exact in both orderings
      bits = range ? 64 - __clzll((long long)range) : 0;
    }
  }
  const uint32_t nwords = (uint32_t)(((uint64_t)count * bits + 63) / 64);
  for (uint32_t i = lane; i < nwords + 1; i += kWarp) words[i] = 0ull;
  __syncwarp();
  if (bits) {
    const uint64_t mask = bits < 64 ? ((1ull << bits) - 1ull) : ~0ull;
    for (uint32_t k = lane; k < count; k += kWarp) {
      uint64_t v = f(k);
      if (use_bp) v = (is_signed ? sext<TS>(v) : v) - mn;
      v &= mask;
      const uint64_t bitpos = (uint64_t)k * bits;
      const uint32_t w = (uint32_t)(bitpos >> 6), s = (uint32_t)(bitpos & 63);
      atomicOr(&words[w], v << s);
      if (s + bits > 64) atomicOr(&words[w + 1], v >> (64 - s));
    }
  }
  __syncwarp();
  if (lane == 0) {
    ((uint32_t*)dst)[0] = count;
    ((uint32_t*)dst)[1] = bits;
    *(uint64_t*)(dst + 8) = use_bp ? mn : 0ull;
  }
  unsigned long long* d64 = (unsigned long long*)(dst + 16);
  for (uint32_t i = lane; i < nwords; i += kWarp) d64[i] = words[i];
  __syncwarp();
  return 16u + 8u * nwords;
}

template <int TS>
__device__ uint32_t casc_encode_part(const uint8_t* __restrict__ in, uint32_t n, int R, int D, bool use_bp,
                                     bool type_signed, uint8_t* dst, uint8_t* sm, uint32_t P, int lane) {
  using T = typename Elem<TS>::T;
  T* cur = (T*)sm;
  T* nxt = (T*)(sm + P);
  // pack buffer: a run-length stream of 1-byte elements can need 16 bits per run -> 2*P bytes
  unsigned long long* words = (unsigned long long*)(sm + 2 * P);          // 2*P + 64 bytes
  uint16_t* runs = (uint16_t*)(sm + 4 * P + 64);                           // 2 * (P/TS) bytes max
  for (uint32_t k = lane; k < n; k += kWarp) cur[k] = ((const T*)in)[k];
  __syncwarp();
  uint32_t count = n;
  uint32_t off = 8u * (uint32_t)D + ((4u * (uint32_t)D + 7u) & ~7u);
  uint64_t* firsts = (uint64_t*)dst;
  uint32_t* cin = (uint32_t*)(dst + 8u * (uint32_t)D);
  if (lane < ((D + 1) & ~1)) cin[lane] = 0;   // also clears the pad word (odd D)
  __syncwarp();
  const int L = R > D ? R : D;
  bool had_delta = false;
  for (int i = 0; i < L; ++i) {
    if (i < R) {
      // run-length encode cur[0..count) -> nxt values, runs lengths
      uint32_t carry = 0;
      for (uint32_t base = 0; base < count; base += kWarp) {
        const uint32_t k = base + lane;
        const bool head = (k < count) && (k == 0 || cur[k] != cur[k - 1]);
        const unsigned m = __ballot_sync(kFull, head);
        const uint32_t pos = carry + __popc(m & ((1u << lane) - 1u));
        if (head) { nxt[pos] = cur[k]; runs[pos] = (uint16_t)k; }   // runs[] holds start index for now
        carry += __popc(m);
      }
      const uint32_t m_runs = carry;
      __syncwarp();
      // lengths = next start - start
      auto run_len = [&](uint32_t k) -> uint64_t {
        const uint32_t s0 = runs[k];
        const uint32_t s1 = (k + 1 < m_runs) ? (uint32_t)runs[k + 1] : count;
        return (uint64_t)(s1 - s0);
      };
      off += casc_pack_stream<2>(run_len, m_runs, use_bp, false, 16, dst + off, words, lane);
      count = m_runs;
      T* t = cur; cur = nxt; nxt = t;
      __syncwarp();
    }
    if (i < D) {
      if (lane == 0) { firsts[i] = count ? (uint64_t)cur[0] : 0ull; cin[i] = count; }
      for (uint32_t k = lane; k + 1 < count; k += kWarp) nxt[k] = (T)(cur[k + 1] - cur[k]);
      count = count ? count - 1 : 0;
      had_delta = true;
      T* t = cur; cur = nxt; nxt = t;
      __syncwarp();
    }
  }
  auto val = [&](uint32_t k) -> uint64_t { return (uint64_t)cur[k]; };
  // signedness only matters for the min/max of un-delta'd values (doc/cascaded_overview.md:35)
  off += casc_pack_stream<TS>(val, count, use_bp, had_delta ? true : type_signed, 8 * TS, dst + off, words, lane);
  return off;
}

constexpr uint32_t kCascCompSmemPerWarp(uint32_t P) { return 4 * P + 64 + 2 * P + 64; }

__global__ void __launch_bounds__(kCascCompWarps * 32)
cascaded_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                         size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                         nvcompBatchedCascadedOpts_t opts, uint32_t smem_per_warp,
                         unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  uint8_t* sm = smem + (size_t)w * smem_per_warp;
  const size_t warp_global = (size_t)blockIdx.x * (blockDim.x >> 5) + w;
  const size_t warps_total = (size_t)gridDim.x * (blockDim.x >> 5);
  WarpTicket sched(ticket, warp_global, warps_total);
  const uint32_t ts = casc_type_size(opts.type);
  const uint32_t P = (uint32_t)opts.chunk_size;
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    const uint32_t n = (uint32_t)in_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    const uint32_t tail = n % ts, whole = n - tail;
    const uint32_t num_parts = (whole + P - 1) / P;
    if (lane == 0) {
      uint32_t* hw = (uint32_t*)out;
      hw[0] = kCascMagic;
      hw[1] = (uint32_t)(opts.type & 0xff) | ((uint32_t)opts.num_RLEs << 8) | ((uint32_t)opts.num_deltas << 16)
              | ((uint32_t)(opts.use_bp ? 1 : 0) << 24);
      hw[2] = n; hw[3] = P; hw[4] = num_parts;
    }
    uint32_t* part_off = (uint32_t*)(out + 20);
    uint32_t off = (20u + 4u * (num_parts + 1) + 7u) & ~7u;
    // pad bytes are zero: an odd partition count leaves one word between the offset table and the first partition
    if (lane == 0 && (num_parts & 1u)) part_off[num_parts + 1] = 0u;
    for (uint32_t p = 0; p < num_parts; ++p) {
      if (lane == 0) part_off[p] = off;
      const uint32_t begin = p * P;
      const uint32_t nb = min(P, whole - begin);
      uint32_t sz;
      switch (ts) {
        case 1: sz = casc_encode_part<1>(in + begin, nb, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                         casc_type_signed(opts.type), out + off, sm, P, lane); break;
        case 2: sz = casc_encode_part<2>(in + begin, nb / 2, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                         casc_type_signed(opts.type), out + off, sm, P, lane); break;
        case 4: sz = casc_encode_part<4>(in + begin, nb / 4, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                         casc_type_signed(opts.type), out + off, sm, P, lane); break;
        default: sz = casc_encode_part<8>(in + begin, nb / 8, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                          casc_type_signed(opts.type), out + off, sm, P, lane); break;
      }
      off += (sz + 7u) & ~7u;
    }
    if (lane == 0) { part_off[num_parts] = off; out_bytes[c] = off + (tail ? 8u : 0u); }
    if (tail && lane < 8) out[off + lane] = (uint32_t)lane < tail ? in[whole + lane] : (uint8_t)0;
    __syncwarp();
  }
}

inline nvcompStatus_t casc_check_opts(const nvcompBatchedCascadedOpts_t& o) {
  const uint32_t ts = casc_type_size(o.type);
  if (ts == 0) return nvcompErrorInvalidValue;
  if (o.num_RLEs < 0 || o.num_RLEs > 7 || o.num_deltas < 0 || o.num_deltas > 7) return nvcompErrorInvalidValue;
  if (o.chunk_size < 512 || o.chunk_size > kCascMaxPart || (o.chunk_size % 8)) return nvcompErrorInvalidValue;
  return nvcompSuccess;
}

// worst-case bytes of one partition payload
inline size_t casc_part_bound(const nvcompBatchedCascadedOpts_t& o) {
  const size_t ts = casc_type_size(o.type);
  const size_t n = o.chunk_size / ts;
  size_t b = 8 * (size_t)o.num_deltas + ((4 * (size_t)o.num_deltas + 7) & ~(size_t)7);
  b += (size_t)o.num_RLEs * (16 + ((n * 16 + 63) / 64) * 8);   // run streams: <= 16 bits each
  b += 16 + ((n * ts * 8 + 63) / 64) * 8;                       // value stream
  return (b + 7) & ~(size_t)7;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedCascadedCompressGetTempSize(
    size_t, size_t max_chunk, nvcompBatchedCascadedOpts_t opts, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = casc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompCascadedCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedCompressGetTempSizeEx(
    size_t b, size_t m, nvcompBatchedCascadedOpts_t o, size_t* t, const size_t) {
  return nvcompBatchedCascadedCompressGetTempSize(b, m, o, t);
}

nvcompStatus_t nvcompBatchedCascadedCompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedCascadedOpts_t opts, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = casc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompCascadedCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  const size_t parts = (max_chunk + opts.chunk_size - 1) / opts.chunk_size;
  *max_compressed_bytes = ((20 + 4 * (parts + 1) + 7) & ~(size_t)7) + parts * casc_part_bound(opts) + 16;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedCompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedCascadedOpts_t opts, cudaStream_t stream) {
  log_call("nvcompBatchedCascadedCompressAsync", batch, max_chunk, stream);
  const nvcompStatus_t st = casc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompCascadedCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const uint32_t per_warp = (kCascCompSmemPerWarp((uint32_t)opts.chunk_size) + 15u) & ~15u;
  int nw = (int)((220u * 1024u) / per_warp);
  if (nw > kCascCompWarps) nw = kCascCompWarps;
  if (nw < 1) return nvcompErrorInvalidValue;
  const size_t smem = (size_t)nw * per_warp;
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(cascaded_compress_kernel, 227 * 1024, smem_set));
  const int ctas_per_sm = (int)((227 * 1024) / (smem + 1024));
  const int grid = persistent_grid(ctas_per_sm < 1 ? 1 : (ctas_per_sm > 8 ? 8 : ctas_per_sm), batch, nw);
  cascaded_compress_kernel<<<grid, nw * 32, smem, stream>>>(
      in_ptrs, in_bytes, batch, out_ptrs, out_bytes, opts, per_warp, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedDecompressGetTempSizeEx(size_t n, size_t m, size_t* t, size_t) {
  return nvcompBatchedCascadedDecompressGetTempSize(n, m, t);
}

nvcompStatus_t nvcompBatchedCascadedGetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedCascadedGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  cascaded_size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedDecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedCascadedDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(cascaded_decompress_kernel, (int)kCascSmem, smem_set));
  const int grid = persistent_grid(kCascDecCtasPerSm, batch, 1);
  cascaded_decompress_kernel<<<grid, kCascWarps * 32, kCascSmem, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"
