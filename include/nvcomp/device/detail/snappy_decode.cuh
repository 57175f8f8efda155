// nvcomp/device/detail/snappy_decode.cuh -- Snappy raw-format decode for one chunk owned by one warp: the format policy
// of the lane-parallel decoder (lz_decode.cuh), the serial element path and the direct loop for chunks that compressed
// >= 4x.  The batched kernels are in nvcomp_b200/csrc/snappy.cu, the device API in nvcomp/device/snappy.cuh.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"
#include "nvcomp/device/detail/lz_decode.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

// varint32 preamble; returns false when malformed.  Warp-uniform.
__device__ __forceinline__ bool snappy_read_preamble(const uint8_t* __restrict__ in, uint32_t in_n,
                                                     uint32_t& ip, uint64_t& ulen) {
  ulen = 0;
  uint32_t shift = 0;
  while (true) {
    if (ip >= in_n || shift > 28) return false;
    const uint32_t b = in[ip++];
    ulen |= (uint64_t)(b & 0x7fu) << shift;
    if (!(b & 0x80u)) break;
    shift += 7;
  }
  return ulen <= 0xffffffffull;
}

// ---------------------------------------------------------------------------
// Run-length steps of the direct loop.  Typed run-length data compresses to short elements: a literal of a few bytes
// (one value), then copies whose offset is the value's width or less.  A step decodes up to 32 such elements at once,
// one per lane, from a 124-byte register window of input, and never reads the output back:
//   - element boundaries by pointer doubling over the window (every byte's "next element if this byte were a tag");
//   - each element is a map from the 8 output bytes before it to the 8 output bytes after it (every new byte is a
//     byte of the old 8 or a literal constant); a warp scan composes the maps, so every lane learns the 8 bytes in
//     front of its element, which hold the whole period of a copy with offset <= 8;
//   - a scan of the output lengths places the elements, and each lane writes its own element with aligned 8-byte
//     stores.
// A step takes the longest prefix of elements that are literals of 1..8 bytes or copy-1 / copy-2 elements with
// offset 1..8, that lie wholly inside the window and pass the checks the serial path makes.  Any other element goes
// to the serial element code, which also gives the verdict on invalid ones.
// ---------------------------------------------------------------------------
constexpr uint32_t kRlWindow = 124;     // bytes of a step's input window (31 whole words, lane 31's is ragged)
constexpr uint32_t kRlNone = 255;       // position outside the window

// 4 byte-wide indices (0..7 in the low 3 bits of each byte) -> the nibble selector __byte_perm takes
__device__ __forceinline__ uint32_t rl_nibbles(uint32_t s) {
  uint32_t u = s & 0x07070707u;
  u |= u >> 4;
  return (u & 0xffu) | ((u >> 8) & 0xff00u);
}

// 0xff in every byte whose top bit is set (a map's constant bytes)
__device__ __forceinline__ uint32_t rl_const_mask(uint32_t s) { return ((s >> 7) & 0x01010101u) * 0xffu; }

// An 8-byte state map: byte i of the new state is byte s[i] of the old state, or the constant v[i] when s[i] = 0x80.
struct RlMap {
  uint32_t s0, s1, v0, v1;
  // this = this o f (f applies first)
  __device__ __forceinline__ void after(uint32_t fs0, uint32_t fs1, uint32_t fv0, uint32_t fv1) {
    const uint32_t n0 = rl_nibbles(s0), n1 = rl_nibbles(s1);
    const uint32_t m0 = rl_const_mask(s0), m1 = rl_const_mask(s1);
    const uint32_t gs0 = __byte_perm(fs0, fs1, n0), gs1 = __byte_perm(fs0, fs1, n1);
    const uint32_t gv0 = __byte_perm(fv0, fv1, n0), gv1 = __byte_perm(fv0, fv1, n1);
    s0 = (gs0 & ~m0) | (s0 & m0); s1 = (gs1 & ~m1) | (s1 & m1);
    v0 = (gv0 & ~m0) | (v0 & m0); v1 = (gv1 & ~m1) | (v1 & m1);
  }
  __device__ __forceinline__ uint64_t apply(uint64_t st) const {
    const uint32_t a = (uint32_t)st, b = (uint32_t)(st >> 32);
    const uint32_t m0 = rl_const_mask(s0), m1 = rl_const_mask(s1);
    const uint32_t r0 = (__byte_perm(a, b, rl_nibbles(s0)) & ~m0) | (v0 & m0);
    const uint32_t r1 = (__byte_perm(a, b, rl_nibbles(s1)) & ~m1) | (v1 & m1);
    return ((uint64_t)r1 << 32) | r0;
  }
};

// 8 bytes of x picked by the 8 nibbles of sel
__device__ __forceinline__ uint64_t rl_perm(uint64_t x, uint32_t sel) {
  const uint32_t a = (uint32_t)x, b = (uint32_t)(x >> 32);
  return ((uint64_t)__byte_perm(a, b, sel >> 16) << 32) | __byte_perm(a, b, sel);
}

// Lane l holds input bytes ip + 4l .. ip + 4l + 3 (little-endian).  Loads stay in the 16-byte granules that hold
// [in, in + in_n); bytes past them read as 0.
__device__ __forceinline__ uint32_t rl_window(const uint8_t* __restrict__ in, uint32_t ip, uintptr_t end16,
                                              uint32_t ul) {
  const uintptr_t a = (uintptr_t)(in + ip);
  const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3) + ul;
  const uint32_t x = (uintptr_t)w < end16 ? *w : 0u;
  const uint32_t y = __shfl_down_sync(kFull, x, 1);
  return __funnelshift_r(x, y, 8u * (uint32_t)(a & 3u));
}

// Byte q (< kRlWindow, or kRlNone -> kRlNone) of the per-position table t (4 positions per lane, one per byte).
__device__ __forceinline__ uint32_t rl_lookup(uint32_t t, uint32_t q) {
  const uint32_t w = __shfl_sync(kFull, t, (int)((q >> 2) & 31u));
  return q == kRlNone ? kRlNone : (w >> (8u * (q & 3u))) & 0xffu;
}

// The 8 output bytes in front of op (byte 7 = out[op - 1]; bytes before out[0] read as 0).  The caller made the
// warp's stores visible (__syncwarp).
__device__ __forceinline__ uint64_t rl_reload(const uint8_t* out, uint32_t op, uint32_t ul) {
  uint32_t b = 0;
  if (ul < 8u && op + ul >= 8u) b = out[op + ul - 8u];
  const uint32_t placed = b << (8u * (ul & 3u));
  const uint32_t lo = __reduce_or_sync(kFull, ul < 4u ? placed : 0u);
  const uint32_t hi = __reduce_or_sync(kFull, ul - 4u < 4u ? placed : 0u);
  return ((uint64_t)hi << 32) | lo;
}

__device__ __forceinline__ bool snappy_decode_chunk(const uint8_t* __restrict__ in, uint32_t in_n,
                                                    uint8_t* out, uint64_t out_cap,
                                                    uint32_t* produced, int lane) {
  uint32_t ip = 0;
  uint64_t ulen;
  if (!snappy_read_preamble(in, in_n, ip, ulen)) return false;
  if (ulen > out_cap) return false;
  const uint32_t n_out = (uint32_t)ulen;
  uint32_t op = 0;
  const uint32_t ul = (uint32_t)lane;
  const uintptr_t end16 = ((uintptr_t)(in + in_n) + 15u) & ~(uintptr_t)15u;
  uint64_t st = 0;                               // the 8 output bytes in front of op
  uint32_t win = rl_window(in, ip, end16, ul);   // input bytes ip .. ip + kRlWindow
  while (ip < in_n) {
    // element 0 of the window: a run element?  (else straight to the serial code)
    const uint32_t h0 = __shfl_sync(kFull, win, 0);
    const uint32_t k0 = h0 & 3u;
    const uint32_t off0 = k0 == 1u ? ((h0 & 0xe0u) << 3) | ((h0 >> 8) & 0xffu) : (h0 >> 8) & 0xffffu;
    if (k0 == 0u ? (h0 & 0xffu) < 32u : k0 != 3u && off0 - 1u < 8u) {
      const uint32_t avail = min(in_n - ip, kRlWindow);
      // nx: for each of this lane's 4 window positions, where the next element starts if an element started there
      uint32_t nx = 0;
#pragma unroll
      for (uint32_t t = 0; t < 4u; ++t) {
        const uint32_t p = 4u * ul + t, tag = (win >> (8u * t)) & 0xffu, k = tag & 3u;
        const uint32_t sz = k == 0u ? ((tag >> 2) < 60u ? (tag >> 2) + 2u : kRlNone) : k == 1u ? 2u : k == 2u ? 3u : 5u;
        nx |= (p + sz < kRlWindow ? p + sz : kRlNone) << (8u * t);
      }
      // pointer doubling: j[r] jumps 2^r elements; lane k composes the jumps of the bits of k
      uint32_t j[5];
      j[0] = nx;
#pragma unroll
      for (int r = 1; r < 5; ++r) {
        uint32_t nj = 0;
#pragma unroll
        for (uint32_t t = 0; t < 4u; ++t) nj |= rl_lookup(j[r - 1], (j[r - 1] >> (8u * t)) & 0xffu) << (8u * t);
        j[r] = nj;
      }
      uint32_t pos = 0;
#pragma unroll
      for (int r = 0; r < 5; ++r) {
        const uint32_t q = rl_lookup(j[r], pos);
        if ((ul >> r) & 1u) pos = q;
      }
      // this lane's element: 9 bytes from pos
      const uint32_t pw = pos == kRlNone ? 0u : pos;
      const uint32_t wi = pw >> 2, sh = 8u * (pw & 3u);
      const uint32_t wa = __shfl_sync(kFull, win, (int)wi), wb = __shfl_sync(kFull, win, (int)((wi + 1u) & 31u)),
                     wc = __shfl_sync(kFull, win, (int)((wi + 2u) & 31u));
      const uint32_t t0 = __funnelshift_r(wa, wb, sh), t1 = __funnelshift_r(wb, wc, sh), t2 = wc >> sh;
      const uint32_t tag = t0 & 0xffu, kind = tag & 3u;
      uint32_t size, len, off;
      if (kind == 0u) { len = (tag >> 2) + 1u; size = len + 1u; off = 0u; }
      else if (kind == 1u) { len = 4u + ((tag >> 2) & 7u); size = 2u; off = ((tag >> 5) << 8) | ((t0 >> 8) & 0xffu); }
      else if (kind == 2u) { len = (tag >> 2) + 1u; size = 3u; off = (t0 >> 8) & 0xffffu; }
      else { len = 0u; size = 5u; off = 0u; }
      const bool run_kind = kind == 0u ? len <= 8u : kind != 3u && off - 1u < 8u;
      const bool in_win = pos != kRlNone && pos + size <= avail;
      // place the elements: op_k = op + the output of the elements before this one
      uint32_t incl = run_kind ? len : 0u;
#pragma unroll
      for (uint32_t d = 1; d < 32u; d <<= 1) {
        const uint32_t x = __shfl_up_sync(kFull, incl, d);
        if (ul >= d) incl += x;
      }
      const uint32_t excl = incl - (run_kind ? len : 0u);
      const uint32_t opk = op + excl;
      // the serial path's checks, for this element in stream order (valid for lanes of the prefix)
      const bool fast = run_kind && in_win && len <= n_out - opk && (kind == 0u || off <= opk);
      const unsigned fm = __ballot_sync(kFull, fast);
      const uint32_t nfast = fm == kFull ? 32u : (uint32_t)__ffs((int)~fm) - 1u;
      // element nfast goes to the serial code unless only the window's end stopped it (the next step takes it)
      const bool to_serial = pos != kRlNone && pos < avail && (!run_kind || in_win);
      const bool serial_next = nfast < 32u && ((__ballot_sync(kFull, to_serial) >> nfast) & 1u);
      if (nfast != 0u) {
        const uint32_t last = nfast - 1u;
        const uint32_t used = __shfl_sync(kFull, pos + size, (int)last);
        const uint32_t made = __shfl_sync(kFull, incl, (int)last);
        const uint32_t next_win = rl_window(in, ip + used, end16, ul);   // in flight during the stores
        // the element's map from the 8 bytes before it to the 8 bytes after it
        const uint32_t o = run_kind && kind != 0u ? off : 1u;
        uint64_t lit = ((uint64_t)__funnelshift_r(t1, t2, 8u) << 32) | __funnelshift_r(t0, t1, 8u);
        RlMap f;
        uint32_t sel8 = 0;                       // nibble i: 8 - off + (i mod off), the copy's bytes from the state
        {
          uint32_t c = 0;
#pragma unroll
          for (uint32_t i = 0; i < 8u; ++i) {
            sel8 |= (8u - o + c) << (4u * i);
            c = c + 1u == o ? 0u : c + 1u;
          }
        }
        if (kind == 0u) {
          const uint32_t l = run_kind ? len : 8u;
          // new byte i = old byte i + l, or literal byte i + l - 8
          uint32_t a = 0x03020100u + l * 0x01010101u, b = 0x07060504u + l * 0x01010101u;
          const uint32_t ca = (a >> 3) & 0x01010101u, cb = (b >> 3) & 0x01010101u;
          f.s0 = (a & ~(ca * 0xffu)) | (ca << 7);
          f.s1 = (b & ~(cb * 0xffu)) | (cb << 7);
          const uint64_t v = lit << (8u * (8u - l));
          f.v0 = (uint32_t)v; f.v1 = (uint32_t)(v >> 32);
        } else {
          // new byte i = old byte len + i, or copy byte len + i - 8 = old byte 8 - off + ((len + i - 8) mod off)
          uint32_t c = (len + 8u * o - 8u) % o, s = 0;
          f.s0 = f.s1 = 0;
#pragma unroll
          for (uint32_t i = 0; i < 8u; ++i) {
            s = len + i < 8u ? len + i : 8u - o + c;
            if (i < 4u) f.s0 |= s << (8u * i); else f.s1 |= s << (8u * (i - 4u));
            c = c + 1u == o ? 0u : c + 1u;
          }
          f.v0 = f.v1 = 0;
        }
        // inclusive scan: lane k's map takes the 8 bytes before element 0 to the 8 bytes after element k
#pragma unroll
        for (uint32_t d = 1; d < 32u; d <<= 1) {
          const uint32_t a0 = __shfl_up_sync(kFull, f.s0, d), a1 = __shfl_up_sync(kFull, f.s1, d),
                         b0 = __shfl_up_sync(kFull, f.v0, d), b1 = __shfl_up_sync(kFull, f.v1, d);
          if (ul >= d) f.after(a0, a1, b0, b1);
        }
        const uint64_t after = f.apply(st);
        uint64_t before = __shfl_up_sync(kFull, after, 1);
        if (ul == 0u) before = st;
        st = __shfl_sync(kFull, after, (int)last);
        if (ul < nfast) {
          // the element's bytes, 8 at a time from its start (word m + 1 = word m through sel8, for a copy); stored as
          // aligned 8-byte words, bytewise where a word is shared with a neighbour
          uint8_t* dst = out + opk;
          const uint32_t hd = (uint32_t)((uintptr_t)dst & 7u);
          uint64_t* aw = (uint64_t*)(dst - hd);
          uint64_t cur = kind == 0u ? lit : rl_perm(before, sel8), prev = 0;
          const uint32_t nw = (hd + len + 7u) >> 3;
#pragma unroll 1
          for (uint32_t m = 0; m < nw; ++m) {
            const uint64_t w = hd ? (cur << (8u * hd)) | (prev >> (64u - 8u * hd)) : cur;
            const int jp = (int)(8u * m) - (int)hd;     // element byte at the word's first byte
            if (jp >= 0 && jp + 8 <= (int)len) {
              aw[m] = w;
            } else {
              uint8_t* bw = (uint8_t*)(aw + m);
#pragma unroll
              for (int t = 0; t < 8; ++t)
                if (jp + t >= 0 && jp + t < (int)len) bw[t] = (uint8_t)(w >> (8 * t));
            }
            prev = cur;
            cur = rl_perm(cur, sel8);
          }
        }
        op += made;
        ip += used;
        win = next_win;
        if (!serial_next) continue;
        __syncwarp();                            // the serial code may read these bytes back
      }
    }
    // serial element
    const uint32_t tag = in[ip++];
    uint32_t len, off;
    const uint32_t kind = tag & 3u;
    if (kind == 0) {
      len = (tag >> 2) + 1;
      if (len > 60) {
        const uint32_t nb = len - 60;
        if (in_n - ip < nb) return false;
        uint32_t v = 0;
        for (uint32_t i = 0; i < nb; ++i) v |= (uint32_t)in[ip + i] << (8 * i);
        ip += nb;
        if (v == 0xffffffffu) return false;
        len = v + 1;
      }
      if (len > in_n - ip || len > n_out - op) return false;
      warp_copy<true>(out + op, in + ip, len, lane);
      ip += len;
      op += len;
      __syncwarp();
      st = rl_reload(out, op, ul);
      win = rl_window(in, ip, end16, ul);
      continue;
    }
    if (kind == 1) {
      if (ip >= in_n) return false;
      len = 4 + ((tag >> 2) & 7u);
      off = ((tag >> 5) << 8) | in[ip++];
    } else if (kind == 2) {
      if (in_n - ip < 2) return false;
      len = (tag >> 2) + 1;
      off = load_u16(in + ip);
      ip += 2;
      // a run of copy-2 elements with the same offset is one long match (64 bytes per element, so
      // only a full-length element can have a continuation): lane i inspects element i, the run is
      // merged and copied once
      if (len == 64u) {
        const uint32_t q = ip + 3u * (uint32_t)lane;
        uint32_t flen = 0;
        bool same = false;
        if (q + 3u <= in_n) {
          const uint32_t t2 = in[q];
          same = ((t2 & 3u) == 2u) && (load_u16(in + q + 1) == off);
          flen = (t2 >> 2) + 1;
        }
        const unsigned m = __ballot_sync(kFull, same);
        const uint32_t nf = (m == kFull) ? 32u : (uint32_t)(__ffs(~m) - 1);
        uint32_t add = ((uint32_t)lane < nf) ? flen : 0u;
#pragma unroll
        for (int d = 16; d; d >>= 1) add += __shfl_xor_sync(kFull, add, d);
        if (len <= n_out - op && add <= n_out - op - len) { len += add; ip += 3u * nf; }
      }
    } else {
      if (in_n - ip < 4) return false;
      len = (tag >> 2) + 1;
      off = (uint32_t)in[ip] | ((uint32_t)in[ip + 1] << 8) | ((uint32_t)in[ip + 2] << 16)
            | ((uint32_t)in[ip + 3] << 24);
      ip += 4;
    }
    if (off == 0 || off > op || len > n_out - op) return false;
    __syncwarp();
    warp_match_copy(out + op, off, len, lane);
    __syncwarp();
    op += len;
    st = rl_reload(out, op, ul);
    win = rl_window(in, ip, end16, ul);
  }
  if (op != n_out) return false;
  *produced = op;
  return true;
}


// ---------------------------------------------------------------------------
// v2 decode (lz_decode.cuh): lane-parallel short-element path + this slow path
// ---------------------------------------------------------------------------
struct SnappyDecode : SnappyPolicy {
  __device__ static __forceinline__ bool at_end(const LzState& s) { return s.ip >= s.in_n; }
  // one element (literal or copy).  A run of copy-2 elements with the same offset -- how Snappy
  // spells one long match (64 bytes per element) -- is merged and emitted as a single match.
  __device__ static __forceinline__ int serial_token(LzState& s, int lane) {
    const uint8_t* __restrict__ in = s.in;
    const uint32_t in_n = s.in_n;
    uint32_t ip = s.ip;
    const uint32_t n_out = (uint32_t)s.out_cap;
    const uint32_t tag = in[ip++];
    const uint32_t kind = tag & 3u;
    uint32_t len, off;
    if (kind == 0) {
      len = (tag >> 2) + 1;
      if (len > 60) {
        const uint32_t nb = len - 60;
        if (in_n - ip < nb) return -1;
        uint32_t v = 0;
        for (uint32_t i = 0; i < nb; ++i) v |= (uint32_t)in[ip + i] << (8 * i);
        ip += nb;
        if (v == 0xffffffffu) return -1;
        len = v + 1;
      }
      if (len > in_n - ip || len > n_out - s.op) return -1;
      lz_serial_lookahead<SnappyPolicy>(s, ip + len, lane);
      lz_emit_literals(s, in + ip, len, lane);
      s.ip = ip + len;
      return 1;
    }
    if (kind == 1) {
      if (ip >= in_n) return -1;
      len = 4 + ((tag >> 2) & 7u);
      off = ((tag >> 5) << 8) | in[ip++];
    } else if (kind == 2) {
      if (in_n - ip < 2) return -1;
      len = (tag >> 2) + 1;
      off = load_u16(in + ip);
      ip += 2;
      // merge following copy-2 elements with the same offset (lane i inspects element i); only a
      // full-length element can have a continuation
      if (len == 64u) {
        const uint32_t q = ip + 3u * (uint32_t)lane;
        uint32_t flen = 0;
        bool same = false;
        if (q + 3u <= in_n) {
          const uint32_t t2 = in[q];
          same = ((t2 & 3u) == 2u) && (load_u16(in + q + 1) == off);
          flen = (t2 >> 2) + 1;
        }
        const unsigned m = __ballot_sync(kFull, same);
        const uint32_t nf = (m == kFull) ? 32u : (uint32_t)(__ffs(~m) - 1);
        uint32_t add = ((uint32_t)lane < nf) ? flen : 0u;
#pragma unroll
        for (int d = 16; d; d >>= 1) add += __shfl_xor_sync(kFull, add, d);
        if (add <= n_out - s.op - min(len, n_out - s.op)) { len += add; ip += 3u * nf; }
      }
    } else {
      if (in_n - ip < 4) return -1;
      len = (tag >> 2) + 1;
      off = (uint32_t)in[ip] | ((uint32_t)in[ip + 1] << 8) | ((uint32_t)in[ip + 2] << 16)
            | ((uint32_t)in[ip + 3] << 24);
      ip += 4;
    }
    if (off == 0 || off > s.op || len > n_out - s.op) return -1;
    lz_serial_lookahead<SnappyPolicy>(s, ip, lane);
    lz_emit_match(s, off, len, lane);
    s.ip = ip;
    return 1;
  }
};

__device__ __forceinline__ bool snappy_decode_chunk_v2(const uint8_t* in, uint32_t in_n, uint8_t* out,
                                                       uint64_t out_cap, uint32_t* produced,
                                                       uint8_t* ring, uint32_t& tma_parity, int lane, bool allow_direct = true) {
  uint32_t ip = 0;
  uint64_t ulen;
  if (!snappy_read_preamble(in, in_n, ip, ulen)) return false;
  if (ulen > out_cap) return false;
  // Adaptive strategy (see lz4.cu): chunks that compressed >= 4x are long-match dominated and
  // take the direct global-memory token loop.
  if (allow_direct && ulen >= 4ull * in_n) return snappy_decode_chunk(in, in_n, out, out_cap, produced, lane);
  LzState s;
  s.in = in; s.in_n = in_n; s.out = out; s.out_cap = ulen;
  s.ip = ip; s.op = 0; s.flushed = 0; s.ring_lo = 0;
  s.align = (uint32_t)((uintptr_t)out & 15u);
  s.ring = smem_addr(ring);
  s.cur = 0; s.pf_ip = kNoPrefetch; s.parity = tma_parity; s.next = kNextUnknown;
  const bool ok = lz_decode_stream<SnappyDecode>(s, lane);
  tma_parity = s.parity;                 // the barrier outlives the chunk: carry its phase to the next one
  if (!ok) return false;
  if (s.op != (uint32_t)ulen) return false;
  *produced = s.op;
  return true;
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
