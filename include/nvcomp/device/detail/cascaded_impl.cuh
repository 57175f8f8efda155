// nvcomp/device/detail/cascaded_impl.cuh -- the Cascaded stream and its per-partition coder, shared by the batched
// kernels (nvcomp_b200/csrc/cascaded.cu) and the warp-level device API (nvcomp/device/cascaded.cuh).  Header-only
// device code for sm_90a; not a public interface.
//
// Algorithm: reference doc/cascaded_overview.md:7-42 -- RLE and delta layers are interleaved (values out of RLE i
// feed delta i), then every resulting stream (all run-length streams and the final value stream) is bit-packed
// against its minimum.  The reference bitstream is undocumented, so this is our own:
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
// Every partition function here is called by a whole warp on one partition, out of that warp's own shared-memory
// region; the callers own the partition offsets, the chunk header and the trailing word.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include "nvcomp/cascaded.h"

namespace nvcomp {
namespace device {
namespace cascaded {
namespace detail {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr uint32_t kCascMagic = 0x31435343u;  // "CSC1"
constexpr uint32_t kCascMaxPart = 16384;

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

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

// ----- shared-memory and streaming accesses on 32-bit shared-window addresses --------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void st_v4(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a) : "memory");
  return r;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(v) : "r"(a), "n"(0) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory");
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
// What a partition walk (casc_decode_part, casc_final_rle) does with a partition it accepts:
//   kCascDecode writes its elements to `out`;
//   kCascCheck  unpacks only the run-length streams and makes every check kCascDecode makes -- all of them depend on
//               headers, counts and run lengths, none on value bits -- and writes nothing but the warp's shared memory;
//   kCascVisit  decodes like kCascDecode but, instead of storing, calls f(const T (&v)[4], k, valid) on every lane for
//               each 128-element block: v[0..3] are elements k .. k + 3 of the partition (k = 128 * block + 4 * lane),
//               the first `valid` of them exist.  Blocks come in order and never cross the partition.
// ---------------------------------------------------------------------------
enum CascMode { kCascDecode = 0, kCascCheck = 1, kCascVisit = 2 };

struct CascNoVisit {
  template <class T> __device__ __forceinline__ void operator()(const T (&)[4], uint32_t, uint32_t) const {}
};

// Visit `total` elements get(k) in 128-element blocks (kCascVisit)
template <class T, class G, class F>
__device__ __forceinline__ void casc_visit_blocks(uint32_t total, G get, const F& f, int lane) {
  for (uint32_t base = 0; base < total; base += 4u * kWarp) {
    const uint32_t k0 = base + 4u * (uint32_t)lane;
    T v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = k0 + e < total ? get(k0 + e) : (T)0;
    f(v, k0, k0 < total ? min(4u, total - k0) : 0u);
  }
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

template <int TS, int SRC, int MODE = kCascDecode, class F = CascNoVisit>
__device__ __forceinline__ bool casc_final_rle(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ vwords,
                                               const StreamHdr vh, const typename Elem<TS>::T* cur, uint32_t count,
                                               bool has_delta, uint64_t first, uint32_t c_in,
                                               const StreamHdr rh, const uint64_t* __restrict__ rwords,
                                               typename Elem<TS>::T* stage, uint32_t cap,
                                               uint8_t* out, uint32_t n_out, int lane, const F& f = F()) {
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
    if constexpr (MODE != kCascCheck) {
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
    if constexpr (MODE != kCascCheck) {
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
  }
  const uint32_t total = lcarry;
  if (total < nvals || total != n_out) return false;
  if constexpr (MODE == kCascCheck) return true;
  __syncwarp();
  if constexpr (MODE == kCascVisit) {
    // the staged elements, four per lane: one vector load each when the buffer is aligned for it
    const bool vec = (stage_s & (uint32_t)(alignof(Quad4<T>) - 1)) == 0u;
    for (uint32_t base = 0; base < total; base += 4u * kWarp) {
      const uint32_t k0 = base + 4u * (uint32_t)lane;
      Quad4<T> q;
      if (vec && k0 + 4u <= total) q = *(const Quad4<T>*)(stage + k0);
      else {
#pragma unroll
        for (int e = 0; e < 4; ++e) q.e[e] = k0 + e < total ? stage[k0 + e] : (T)0;
      }
      f(q.e, k0, k0 < total ? min(4u, total - k0) : 0u);
    }
    return true;
  }
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

// Shared memory one warp needs to decode a partition of P bytes of 2^ts_shift-byte elements: one value buffer (P
// bytes; two when more than one layer pair is configured) + a run-index u16 array (2 * P/TS bytes), 16-byte rounded.
__host__ __device__ constexpr uint32_t casc_decode_smem_bytes(uint32_t P, uint32_t ts_shift, bool two_bufs) {
  return ((two_bufs ? 2u : 1u) * P + 2u * (P >> ts_shift) + 4u + 15u) & ~15u;
}

// ---------------------------------------------------------------------------
// Decode one partition with one warp.  `n_out` elements expected.
// sm layout (per warp): A [P] | (B [P] when two_bufs) | idx u16[P/TS]
// Delta layers are undone in place; the outermost run-length expansion writes straight to the
// output (global memory), so the common one-layer configurations need a single value buffer.
// Returns false on a malformed partition.  MODE: see CascMode (kCascCheck and kCascVisit never touch `out`).
// ---------------------------------------------------------------------------
template <int TS, int MODE = kCascDecode, class F = CascNoVisit>
__device__ bool casc_decode_part(const uint8_t* __restrict__ payload, uint32_t payload_bytes,
                                 uint8_t* out, uint32_t n_out, int R, int D,
                                 uint8_t* sm, uint32_t P, bool two_bufs, int lane, const F& f = F()) {
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
      return casc_final_rle<TS, 0, MODE>(payload, vwords, vh, nullptr, count, hd, first, c_in, rh0, rwords, bufA, cap, out, n_out, lane, f);
    return casc_final_rle<TS, 1, MODE>(payload, vwords, vh, nullptr, count, hd, first, c_in, rh0, rwords, bufA, cap, out, n_out, lane, f);
  }
  // unpack the final value stream into A
  if constexpr (MODE != kCascCheck) {
    if (vh.bits != 0u && vh.bits <= 32u) {
      const uint32_t* w32 = (const uint32_t*)vwords;
      const uint32_t mask = vh.bits == 32u ? 0xffffffffu : ((1u << vh.bits) - 1u);
      for (uint32_t k = lane; k < count; k += kWarp) bufA[k] = (T)unpack32_at(w32, k, vh.bits, mask, vh.minv);
    } else {
      for (uint32_t k = lane; k < count; k += kWarp) bufA[k] = (T)unpack_at(vwords, k, vh.bits, vh.minv);
    }
  }
  __syncwarp();
  T* cur = bufA;
  for (int i = L - 1; i >= 0; --i) {
    if (i == 0 && R > 0 && rh0.bits <= 32u) {
      // layer 0 with run-length encoding: fused delta + expansion from the buffer the layers above left
      const uint64_t* rwords = (const uint64_t*)(payload + roff0);
      const bool hd = D > 0;
      return casc_final_rle<TS, 2, MODE>(payload, nullptr, vh, cur, count, hd, first0, cin0, rh0, rwords,
                                         cur == bufA ? bufB : bufA, cap, out, n_out, lane, f);
    }
    if (i < D) {
      // undo delta i in place: cur[0..count) deltas -> cur[0..count] values.  cin == 0: the layer saw
      // an empty list.
      const uint32_t c_in = cin[i];
      if (c_in == 0 && count != 0) return false;
      if (c_in != 0) {
        if (c_in != count + 1 || c_in > cap) return false;
        if constexpr (MODE != kCascCheck) {
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
      if constexpr (MODE != kCascCheck) {
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
        if constexpr (MODE != kCascCheck) {
          if (k0 + 0 < count && len[0]) idx[ex] = (uint16_t)(k0 + 0);
          if (k0 + 1 < count && len[1]) idx[ex + p1] = (uint16_t)(k0 + 1);
          if (k0 + 2 < count && len[2]) idx[ex + p2] = (uint16_t)(k0 + 2);
          if (k0 + 3 < count && len[3]) idx[ex + p3] = (uint16_t)(k0 + 3);
        }
      }
      const uint32_t total = carry;
      if (total > cap || total < count) return false;
      if (last && total != n_out) return false;
      if constexpr (MODE == kCascCheck) {
        if (last) return true;
        count = total;
        continue;
      }
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
      if constexpr (MODE == kCascVisit) {
        if (last) {
          // the last expansion gathers into registers instead of storing
          casc_visit_blocks<T>(total, [&](uint32_t j) { return cur[idx[j]]; }, f, lane);
          return true;
        }
      }
      // ... then a coalesced gather: consecutive lanes write consecutive outputs
      for (uint32_t j = lane; j < total; j += kWarp) dst[j] = cur[idx[j]];
      if (last) return true;
      count = total;
      __syncwarp();
      cur = dst;
    }
  }
  if (count != n_out) return false;
  if constexpr (MODE == kCascCheck) return true;
  if constexpr (MODE == kCascVisit) {
    casc_visit_blocks<T>(count, [&](uint32_t k) { return cur[k]; }, f, lane);
    return true;
  }
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

// partition p's payload [o0, o1) of a stream of in_bytes bytes: 8-byte aligned and inside the stream
__device__ __forceinline__ bool casc_part_span_ok(uint32_t o0, uint32_t o1, size_t in_bytes) {
  return (o0 & 7) == 0 && o0 <= o1 && o1 <= in_bytes;
}

// ---------------------------------------------------------------------------
// Compression: one warp per chunk walks its partitions in order, so partition
// payloads are appended without a compaction pass.
// per-warp smem: A [P] | B [P] | pack words [2P + 64] | runs u16 [P elements]
// ---------------------------------------------------------------------------

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

__host__ __device__ constexpr uint32_t kCascCompSmemPerWarp(uint32_t P) { return 4 * P + 64 + 2 * P + 64; }

__host__ __device__ inline nvcompStatus_t casc_check_opts(const nvcompBatchedCascadedOpts_t& o) {
  const uint32_t ts = casc_type_size(o.type);
  if (ts == 0) return nvcompErrorInvalidValue;
  if (o.num_RLEs < 0 || o.num_RLEs > 7 || o.num_deltas < 0 || o.num_deltas > 7) return nvcompErrorInvalidValue;
  if (o.chunk_size < 512 || o.chunk_size > kCascMaxPart || (o.chunk_size % 8)) return nvcompErrorInvalidValue;
  return nvcompSuccess;
}

// worst-case bytes of one partition payload
__host__ __device__ inline size_t casc_part_bound(const nvcompBatchedCascadedOpts_t& o) {
  const size_t ts = casc_type_size(o.type);
  const size_t n = o.chunk_size / ts;
  size_t b = 8 * (size_t)o.num_deltas + ((4 * (size_t)o.num_deltas + 7) & ~(size_t)7);
  b += (size_t)o.num_RLEs * (16 + ((n * 16 + 63) / 64) * 8);   // run streams: <= 16 bits each
  b += 16 + ((n * ts * 8 + 63) / 64) * 8;                       // value stream
  return (b + 7) & ~(size_t)7;
}

// worst-case bytes of the stream of a chunk of max_chunk bytes under valid options
__host__ __device__ inline size_t casc_max_output_bytes(size_t max_chunk, const nvcompBatchedCascadedOpts_t& o) {
  const size_t parts = (max_chunk + o.chunk_size - 1) / o.chunk_size;
  return ((20 + 4 * (parts + 1) + 7) & ~(size_t)7) + parts * casc_part_bound(o) + 16;
}

}  // namespace detail
}  // namespace cascaded
}  // namespace device
}  // namespace nvcomp
