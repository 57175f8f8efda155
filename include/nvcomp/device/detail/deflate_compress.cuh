// nvcomp/device/detail/deflate_compress.cuh -- warp-per-chunk Deflate (RFC 1951) encoder behind
// nvcompBatchedDeflateCompressAsync and deflate::compress_warp (nvcomp/device/deflate.cuh).  The batched kernel of
// deflate.cu (nvcomp_b200/csrc/deflate_compress.cuh re-exports these names) and the device API share it.
//
// One warp owns one chunk (<= 64 KB) and writes one raw Deflate stream with a single final block (zlib wbits = -15
// reads it).  Two passes over the same parse, no token buffer:
//   pass A  the parse (lz77_compress.cuh, or literals only for algo 2) fills the literal/length (286) and distance
//           (30) histograms in the warp's shared memory;
//   choice  the exact bit cost of a stored, a fixed-code and a dynamic-code encoding is computed from the histograms,
//           and the cheapest is taken (ties: stored, then fixed);
//   pass B  unless stored, the same parse runs again and each sequence is coded as it comes: literal codes are looked
//           up lane-parallel, placed by a warp scan of their bit lengths and OR-ed into a shared staging window; the
//           match is coded by one lane; whole 32-bit words of the window are flushed to global memory.
// Re-running the parse costs matcher time but needs no workspace, and gives one block per chunk.
//
// Stream rules (tests/deflate_encode_model.py restates them and re-encodes every stream to the same bytes):
//   * Parse: algo 0 greedy (4096-entry hash), algo 1 greedy + one-position lazy step (32 768-entry hash; the
//     next position's match is taken when it is longer and no farther back), algo 2 no
//     matches.  Matches are 4..258 bytes, at distance <= 32 768, and do not start in the last 4 bytes of the chunk.
//     Hash inserts are deterministic (lz77_compress.cuh), so the parse is a function of the input alone.
//   * Stored: blocks of 65 535 bytes, the last one shorter (one empty block for an empty chunk); costs 8 * (n + 5 *
//     blocks) bits, and is the largest output: n + 5 * (n / 65535 + 1) bounds every stream.
//   * Code lengths: package-merge (optimal under the limit: 15 for literal/length and distance codes, 7 for the
//     code-length code).  Leaves are ordered by (frequency, symbol); in each merge a leaf goes before a package of
//     equal weight.  A code with one used symbol gets length 1.  A block without matches carries one distance code,
//     symbol 0, of length 1.  A code-length code with one used symbol would be incomplete, which zlib rejects: such a
//     dynamic block is never chosen (it cannot arise: the lengths always contain a zero run and a nonzero length).
//   * Header: HLIT >= 257 and HDIST >= 1 are minimal.  The HLIT + HDIST lengths are one sequence, run-length coded
//     greedily: a zero run of r >= 3 takes 18 (11..138) or 17 (3..10) pieces of min(r, 138) while r >= 3, then single
//     zeros; a nonzero run emits the length once, then 16 pieces of min(r, 6) while r >= 3, then single lengths.
//     HCLEN is trimmed to the last nonzero code-length length in the RFC order (at least 4).
//   * The last byte is zero-padded.
#pragma once

#include "nvcomp/device/detail/lz77_compress.cuh"

namespace nvcomp {
namespace device {
namespace deflate {
namespace detail {

using lz::detail::kWarp;
using lz::detail::kFull;
using lz::detail::warp_copy;
using lz::detail::LzParams;
using lz::detail::kHashBytesPerWarp;
using lz::detail::lz77_compress_chunk;

constexpr int kDeflateLitSyms = 286;
constexpr int kDeflateDistSyms = 30;
constexpr int kDeflateClenSyms = 19;
constexpr int kDeflateDistBase = kDeflateLitSyms;                       // index of distance symbol 0 in hist / code
constexpr int kDeflateClenBase = kDeflateLitSyms + kDeflateDistSyms;    // index of code-length symbol 0
constexpr int kDeflateSymWords = 336;                                   // 335 used
constexpr int kDeflateStageWords = 66;   // 1023 bits before a flush + at most 480 bits of one literal round
constexpr uint32_t kDeflateFlushBits = 1024;
constexpr uint32_t kDeflateMaxChunk = 65536;
constexpr uint32_t kStoredMax = 65535;

// package-merge workspace (32-bit words) inside the warp's hash table, which pass B clears anyway:
//   leaf weights [286] | leaf symbols [286] | two level lists [571 each, 572] | leaf flags [15 levels x 18 words]
constexpr int kPmFlagWords = 18;
constexpr int kPmWords = 2 * kDeflateLitSyms + 2 * 572 + 15 * kPmFlagWords;
static_assert(kPmWords * 4 <= kHashBytesPerWarp, "package-merge workspace fits in the smallest hash table");

template <int kAlgo> struct DeflateAlgo;
template <> struct DeflateAlgo<0> : LzParams {          // high throughput: the greedy matcher
  static constexpr uint32_t kMaxDist = 32768u, kMaxLen = 258u;
  static constexpr bool kParse = true;
};
template <> struct DeflateAlgo<1> : DeflateAlgo<0> {    // high compression: bigger table, lazy step
  static constexpr int kHashLog = 15;
  static constexpr bool kLazy = true;
};
template <> struct DeflateAlgo<2> : DeflateAlgo<0> {    // entropy only: literals
  static constexpr bool kParse = false;
};

// shared memory bytes per warp
template <int kAlgo>
constexpr size_t kDeflateWarpSmem =
    ((size_t)(2u << DeflateAlgo<kAlgo>::kHashLog) + 4u * (2 * kDeflateSymWords + kDeflateStageWords) + 15) & ~(size_t)15;

// The warp's shared memory: hash table (package-merge workspace between the passes) | hist | code | stage
struct DeflateWarp {
  uint16_t* table;
  uint32_t* hist;    // frequencies: literal/length 0..285, distance at kDeflateDistBase, code-length at kDeflateClenBase
  uint32_t* code;    // same indices: bit-reversed code | length << 16
  uint32_t* stage;   // output bit window
  template <int kAlgo>
  __device__ __forceinline__ static DeflateWarp carve(uint8_t* base) {
    DeflateWarp w;
    w.table = (uint16_t*)base;
    w.hist = (uint32_t*)(base + (2u << DeflateAlgo<kAlgo>::kHashLog));
    w.code = w.hist + kDeflateSymWords;
    w.stage = w.code + kDeflateSymWords;
    return w;
  }
};

// length 3..258 -> (symbol 257..285, extra bits, extra value)
__device__ __forceinline__ void deflate_len_code(uint32_t len, uint32_t& sym, uint32_t& nb, uint32_t& ev) {
  const uint32_t l = len - 3u;
  if (len == 258u) { sym = 285u; nb = 0; ev = 0; }
  else if (l < 8u) { sym = 257u + l; nb = 0; ev = 0; }
  else {
    nb = (31u - (uint32_t)__clz((int)l)) - 2u;
    sym = 261u + 4u * nb + ((l >> nb) & 3u);
    ev = l & ((1u << nb) - 1u);
  }
}
// distance 1..32768 -> (symbol 0..29, extra bits, extra value)
__device__ __forceinline__ void deflate_dist_code(uint32_t d, uint32_t& sym, uint32_t& nb, uint32_t& ev) {
  const uint32_t x = d - 1u;
  if (x < 4u) { sym = x; nb = 0; ev = 0; }
  else {
    const uint32_t b = 31u - (uint32_t)__clz((int)x);
    nb = b - 1u;
    sym = 2u * b + ((x >> nb) & 1u);
    ev = x & ((1u << nb) - 1u);
  }
}
__device__ __forceinline__ uint32_t deflate_len_extra(uint32_t sym) {   // 257..285
  return (sym < 265u || sym == 285u) ? 0u : (sym - 261u) >> 2;
}
__device__ __forceinline__ uint32_t deflate_dist_extra(uint32_t sym) { return sym < 4u ? 0u : (sym >> 1) - 1u; }
__device__ __forceinline__ uint32_t deflate_fixed_lit_len(uint32_t s) {
  return s < 144u ? 8u : s < 256u ? 9u : s < 280u ? 7u : 8u;
}

// ---------------------------------------------------------------------------
// Pass A: histograms
// ---------------------------------------------------------------------------
struct DeflateHist {
  uint32_t* hist;
  __device__ __forceinline__ void literals(const uint8_t* lit, uint32_t ll, int lane) {
    for (uint32_t i = lane; i < ll; i += kWarp) atomicAdd(&hist[lit[i]], 1u);
  }
  __device__ __forceinline__ void sequence(const uint8_t* lit, uint32_t ll, uint32_t off, uint32_t ml, int lane) {
    literals(lit, ll, lane);
    if (lane == 0) {
      uint32_t s, nb, ev;
      deflate_len_code(ml, s, nb, ev);
      atomicAdd(&hist[s], 1u);
      deflate_dist_code(off, s, nb, ev);
      atomicAdd(&hist[kDeflateDistBase + s], 1u);
    }
  }
  __device__ __forceinline__ void finish(const uint8_t* lit, uint32_t ll, int lane) { literals(lit, ll, lane); }
};

// ---------------------------------------------------------------------------
// Bit output: a warp-uniform bit position in a shared window, OR-ed into by atomics, flushed as whole words
// ---------------------------------------------------------------------------
struct DeflateBits {
  uint32_t* stage;
  uint32_t* code;
  uint8_t* out;
  uint32_t bitpos;    // bits in the window (warp-uniform)
  uint32_t flushed;   // bytes already written to out

  __device__ __forceinline__ void clear(int lane) {
    for (int i = lane; i < kDeflateStageWords; i += kWarp) stage[i] = 0;
    __syncwarp();
  }
  __device__ __forceinline__ void or_at(uint32_t q, uint32_t v, uint32_t n) {   // v < 2^n, n <= 32
    const uint32_t w = q >> 5, sh = q & 31u;
    atomicOr(&stage[w], v << sh);
    if (sh != 0u && sh + n > 32u) atomicOr(&stage[w + 1], v >> (32u - sh));
  }
  __device__ __forceinline__ void flush(int lane) {
    __syncwarp();
    const uint32_t nw = bitpos >> 5;
    for (uint32_t j = lane; j < 4u * nw; j += kWarp) out[flushed + j] = (uint8_t)(stage[j >> 2] >> (8u * (j & 3u)));
    const uint32_t carry = stage[nw];
    __syncwarp();
    for (int i = lane; i < kDeflateStageWords; i += kWarp) stage[i] = i == 0 ? carry : 0u;
    __syncwarp();
    flushed += 4u * nw;
    bitpos &= 31u;
  }
  __device__ __forceinline__ void put(uint32_t v, uint32_t n, int lane) {   // warp-uniform v, n <= 32
    if (bitpos >= kDeflateFlushBits) flush(lane);
    if (lane == 0 && n) or_at(bitpos, v, n);
    bitpos += n;
  }
  __device__ __forceinline__ void put_lanes(uint32_t v, uint32_t n, int lane) {   // each lane's own (v, n), lane order
    if (bitpos >= kDeflateFlushBits) flush(lane);
    uint32_t incl = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(kFull, incl, d);
      if (lane >= d) incl += o;
    }
    if (n) or_at(bitpos + incl - n, v, n);
    bitpos += __shfl_sync(kFull, incl, 31);
  }
  __device__ __forceinline__ void put_sym(uint32_t idx, int lane) {
    const uint32_t c = code[idx];
    put(c & 0xffffu, c >> 16, lane);
  }
  // pass B emitter
  __device__ __forceinline__ void literals(const uint8_t* lit, uint32_t ll, int lane) {
    for (uint32_t base = 0; base < ll; base += kWarp) {
      const uint32_t i = base + lane;
      const uint32_t c = i < ll ? code[lit[i]] : 0u;
      put_lanes(c & 0xffffu, c >> 16, lane);
    }
  }
  __device__ __forceinline__ void sequence(const uint8_t* lit, uint32_t ll, uint32_t off, uint32_t ml, int lane) {
    literals(lit, ll, lane);
    uint32_t s, nb, ev;
    deflate_len_code(ml, s, nb, ev);
    uint32_t c = code[s];
    put((c & 0xffffu) | (ev << (c >> 16)), (c >> 16) + nb, lane);
    deflate_dist_code(off, s, nb, ev);
    c = code[kDeflateDistBase + s];
    put((c & 0xffffu) | (ev << (c >> 16)), (c >> 16) + nb, lane);
  }
  __device__ __forceinline__ void finish(const uint8_t* lit, uint32_t ll, int lane) { literals(lit, ll, lane); }
  // pad the last byte and write what is left; returns the stream's length
  __device__ __forceinline__ uint32_t close(int lane) {
    __syncwarp();
    const uint32_t nb = (bitpos + 7u) >> 3;
    for (uint32_t j = lane; j < nb; j += kWarp) out[flushed + j] = (uint8_t)(stage[j >> 2] >> (8u * (j & 3u)));
    __syncwarp();
    return flushed + nb;
  }
};

// ---------------------------------------------------------------------------
// Length-limited code lengths by package-merge (rules in the file header).  freq[0..nsym) -> code[s] = length << 16.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void pm_lengths(const uint32_t* freq, int nsym, int limit, uint32_t* code, uint32_t* ws,
                                           int lane) {
  uint32_t* lw = ws;                         // leaf weights, sorted
  uint32_t* ls = ws + kDeflateLitSyms;       // their symbols
  uint32_t* cur = ws + 2 * kDeflateLitSyms;
  uint32_t* nxt = cur + 572;
  uint32_t* flags = nxt + 572;               // level d, item i is a leaf: bit i of flags[d * 18 ..]
  uint32_t cnt = 0;
  for (int s = lane; s < nsym; s += kWarp) {
    cnt += freq[s] != 0u;
    code[s] = 0;
  }
  const uint32_t n = __reduce_add_sync(kFull, cnt);
  __syncwarp();
  if (n <= 1u) {
    for (int s = lane; s < nsym; s += kWarp)
      if (freq[s]) code[s] = 1u << 16;
    __syncwarp();
    return;
  }
  for (int s = lane; s < nsym; s += kWarp) {
    const uint32_t f = freq[s];
    if (!f) continue;
    uint32_t r = 0;
    for (int t = 0; t < nsym; ++t) {
      const uint32_t ft = freq[t];
      r += (ft != 0u) && (ft < f || (ft == f && t < s));
    }
    lw[r] = f;
    ls[r] = (uint32_t)s;
  }
  for (int j = lane; j < limit * kPmFlagWords; j += kWarp) flags[j] = 0;
  __syncwarp();
  // deepest level: the leaves alone
  for (uint32_t i = lane; i < n; i += kWarp) {
    cur[i] = lw[i];
    atomicOr(&flags[(limit - 1) * kPmFlagWords + (i >> 5)], 1u << (i & 31u));
  }
  __syncwarp();
  uint32_t m = n;
  for (int d = limit - 2; d >= 0; --d) {
    const uint32_t np = m >> 1;   // packages: pairs of consecutive items of the level below
    for (uint32_t i = lane; i < n; i += kWarp) {
      const uint32_t w = lw[i];
      uint32_t lo = 0, hi = np;     // packages lighter than the leaf go first
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (cur[2 * mid] + cur[2 * mid + 1] < w) lo = mid + 1; else hi = mid;
      }
      const uint32_t pos = i + lo;
      nxt[pos] = w;
      atomicOr(&flags[d * kPmFlagWords + (pos >> 5)], 1u << (pos & 31u));
    }
    for (uint32_t k = lane; k < np; k += kWarp) {
      const uint32_t w = cur[2 * k] + cur[2 * k + 1];
      uint32_t lo = 0, hi = n;      // leaves of equal or lower weight go first
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (lw[mid] <= w) lo = mid + 1; else hi = mid;
      }
      nxt[k + lo] = w;
    }
    __syncwarp();
    uint32_t* t = cur; cur = nxt; nxt = t;
    m = n + np;
  }
  // the top level's first 2n - 2 items are selected; each selected package selects two items one level down.  A
  // leaf's code length is the number of levels whose selection contains it.
  uint32_t len[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  uint32_t k = 2u * n - 2u;
  for (int d = 0; d < limit; ++d) {
    const uint32_t word = lane < kPmFlagWords ? flags[d * kPmFlagWords + lane] : 0u;
    const uint32_t lo = 32u * (uint32_t)lane;
    const uint32_t mask = k >= lo + 32u ? 0xffffffffu : k > lo ? (1u << (k - lo)) - 1u : 0u;
    const uint32_t leaves = __reduce_add_sync(kFull, (uint32_t)__popc(word & mask));
#pragma unroll
    for (int j = 0; j < 9; ++j) len[j] += (uint32_t)lane + 32u * j < leaves;
    k = 2u * (k - leaves);
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    const uint32_t r = (uint32_t)lane + 32u * j;
    if (r < n) code[ls[r]] = len[j] << 16;
  }
  __syncwarp();
}

// lengths (code[s] >> 16) -> canonical codes, bit-reversed for the LSB-first stream
__device__ __forceinline__ void canonical_codes(uint32_t* code, int nsym, int lane) {
  if (lane == 0) {
    uint32_t count[16], next[16];
    for (int b = 0; b < 16; ++b) count[b] = 0;
    for (int s = 0; s < nsym; ++s) count[code[s] >> 16]++;
    count[0] = 0;
    uint32_t c = 0;
    for (int b = 1; b < 16; ++b) {
      c = (c + count[b - 1]) << 1;
      next[b] = c;
    }
    for (int s = 0; s < nsym; ++s) {
      const uint32_t l = code[s] >> 16;
      if (l) code[s] = (__brev(next[l]++) >> (32u - l)) | (l << 16);
    }
  }
  __syncwarp();
}

// The HLIT + HDIST code lengths as code-length symbols (greedy run-length rules in the file header); every lane
// walks the same sequence and calls f(symbol, extra value, extra bits).
template <class F>
__device__ __forceinline__ void rle_lengths(const uint32_t* code, uint32_t hlit, uint32_t hdist, F&& f) {
  auto L = [&](uint32_t i) { return code[i < hlit ? i : kDeflateDistBase + i - hlit] >> 16; };
  const uint32_t total = hlit + hdist;
  uint32_t i = 0;
  while (i < total) {
    const uint32_t v = L(i);
    uint32_t run = 1;
    while (i + run < total && L(i + run) == v) ++run;
    uint32_t r = run;
    if (v == 0) {
      while (r >= 3u) {
        const uint32_t k = min(r, 138u);
        if (k >= 11u) f(18u, k - 11u, 7u); else f(17u, k - 3u, 3u);
        r -= k;
      }
    } else {
      f(v, 0u, 0u);
      r -= 1;
      while (r >= 3u) {
        const uint32_t k = min(r, 6u);
        f(16u, k - 3u, 2u);
        r -= k;
      }
    }
    for (; r; --r) f(v, 0u, 0u);
    i += run;
  }
}

template <int kAlgo, class Em>
__device__ __forceinline__ void deflate_parse(const uint8_t* in, uint32_t n, Em& em, uint16_t* table, int lane) {
  if constexpr (DeflateAlgo<kAlgo>::kParse)
    lz77_compress_chunk<Em, DeflateAlgo<kAlgo>>(in, n, em, table, 1u, 0u, 4u, lane);
  else
    em.finish(in, n, lane);
}

// Compress one chunk of n <= 64 KB bytes into out (room for n + 5 * (n / 65535 + 1) bytes); returns the stream length.
template <int kAlgo>
__device__ __forceinline__ uint32_t deflate_compress_chunk(const uint8_t* __restrict__ in, uint32_t n,
                                                          uint8_t* __restrict__ out, const DeflateWarp& ws, int lane) {
  uint32_t* hist = ws.hist;
  uint32_t* code = ws.code;
  // --- pass A
  for (int i = lane; i < kDeflateSymWords; i += kWarp) hist[i] = i == 256 ? 1u : 0u;   // one end-of-block code
  __syncwarp();
  {
    DeflateHist h{hist};
    deflate_parse<kAlgo>(in, n, h, ws.table, lane);
  }
  __syncwarp();
  // --- costs
  uint32_t fixed_part = 0, extra_part = 0;
  for (int s = lane; s < kDeflateLitSyms + kDeflateDistSyms; s += kWarp) {
    const uint32_t f = hist[s];
    if (s < kDeflateLitSyms) {
      fixed_part += f * deflate_fixed_lit_len((uint32_t)s);
      if (s > 256) extra_part += f * deflate_len_extra((uint32_t)s);
    } else {
      fixed_part += f * 5u;
      extra_part += f * deflate_dist_extra((uint32_t)(s - kDeflateDistBase));
    }
  }
  const uint32_t extra_bits = __reduce_add_sync(kFull, extra_part);
  const uint32_t fixed_bits = 3u + __reduce_add_sync(kFull, fixed_part) + extra_bits;
  const uint32_t blocks = n == 0 ? 1u : (n + kStoredMax - 1u) / kStoredMax;
  const uint32_t stored_bits = 8u * (n + 5u * blocks);

  uint32_t* pm = (uint32_t*)ws.table;
  pm_lengths(hist, kDeflateLitSyms, 15, code, pm, lane);
  pm_lengths(hist + kDeflateDistBase, kDeflateDistSyms, 15, code + kDeflateDistBase, pm, lane);
  uint32_t last_lit = 0, last_dist = 0;
  for (int s = lane; s < kDeflateLitSyms + kDeflateDistSyms; s += kWarp)
    if (code[s]) {
      if (s < kDeflateLitSyms) last_lit = (uint32_t)s; else last_dist = (uint32_t)(s - kDeflateDistBase) + 1u;
    }
  const uint32_t hlit = max(257u, __reduce_max_sync(kFull, last_lit) + 1u);
  uint32_t hdist = __reduce_max_sync(kFull, last_dist);
  if (hdist == 0) {                      // no matches: one distance code of length 1
    if (lane == 0) code[kDeflateDistBase] = 1u << 16;
    __syncwarp();
    hdist = 1;
  }
  uint32_t body_part = 0;
  for (int s = lane; s < kDeflateLitSyms + kDeflateDistSyms; s += kWarp) body_part += hist[s] * (code[s] >> 16);
  const uint32_t body_bits = __reduce_add_sync(kFull, body_part) + extra_bits;
  uint32_t rle_extra = 0;
  rle_lengths(code, hlit, hdist, [&](uint32_t sym, uint32_t, uint32_t nb) {
    if (lane == 0) hist[kDeflateClenBase + sym]++;
    rle_extra += nb;
  });
  __syncwarp();
  pm_lengths(hist + kDeflateClenBase, kDeflateClenSyms, 7, code + kDeflateClenBase, pm, lane);
  constexpr int kOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  uint32_t hclen = 4, clen_part = 0, clen_used = 0;
  for (int i = 0; i < kDeflateClenSyms; ++i) {
    const uint32_t c = code[kDeflateClenBase + kOrder[i]];
    if (c) { hclen = max(hclen, (uint32_t)i + 1u); ++clen_used; }
    clen_part += hist[kDeflateClenBase + kOrder[i]] * (c >> 16);
  }
  const bool dyn_ok = clen_used >= 2u;
  const uint32_t dyn_bits = 3u + 14u + 3u * hclen + clen_part + rle_extra + body_bits;

  if (stored_bits <= fixed_bits && (!dyn_ok || stored_bits <= dyn_bits)) {
    uint32_t o = 0, p = 0;
    for (uint32_t b = 0; b < blocks; ++b) {
      const uint32_t len = min(n - p, kStoredMax);
      const uint32_t hdr[5] = {b + 1u == blocks ? 1u : 0u, len & 255u, len >> 8, ~len & 255u, (~len >> 8) & 255u};
      if (lane < 5) out[o + lane] = (uint8_t)hdr[lane];
      if (len) warp_copy<true>(out + o + 5u, in + p, len, lane);
      o += 5u + len;
      p += len;
    }
    __syncwarp();
    return o;
  }
  const bool fixed = fixed_bits <= dyn_bits || !dyn_ok;
  if (fixed) {
    // RFC 1951 3.2.6 (the canonical code over all 288 literal/length symbols: 286 and 287 take 8-bit codes before
    // the 9-bit ones, so it cannot be rebuilt from the 286 used lengths)
    for (int s = lane; s < kDeflateLitSyms + kDeflateDistSyms; s += kWarp) {
      const uint32_t u = (uint32_t)s;
      const uint32_t l = s < kDeflateLitSyms ? deflate_fixed_lit_len(u) : 5u;
      const uint32_t c = s >= kDeflateLitSyms ? u - kDeflateDistBase
                         : u < 144u ? 0x30u + u : u < 256u ? 0x190u + u - 144u : u < 280u ? u - 256u : 0xc0u + u - 280u;
      code[s] = (__brev(c) >> (32u - l)) | (l << 16);
    }
    __syncwarp();
  } else {
    canonical_codes(code, kDeflateLitSyms, lane);
    canonical_codes(code + kDeflateDistBase, kDeflateDistSyms, lane);
  }
  DeflateBits bo{ws.stage, code, out, 0u, 0u};
  bo.clear(lane);
  bo.put(fixed ? 3u : 5u, 3u, lane);     // BFINAL, BTYPE 01 / 10
  if (!fixed) {
    canonical_codes(code + kDeflateClenBase, kDeflateClenSyms, lane);
    bo.put((hlit - 257u) | ((hdist - 1u) << 5) | ((hclen - 4u) << 10), 14u, lane);
    for (uint32_t i = 0; i < hclen; ++i) bo.put(code[kDeflateClenBase + kOrder[i]] >> 16, 3u, lane);
    rle_lengths(code, hlit, hdist, [&](uint32_t sym, uint32_t ev, uint32_t nb) {
      const uint32_t c = code[kDeflateClenBase + sym];
      bo.put((c & 0xffffu) | (ev << (c >> 16)), (c >> 16) + nb, lane);
    });
  }
  // --- pass B
  deflate_parse<kAlgo>(in, n, bo, ws.table, lane);
  bo.put_sym(256, lane);
  return bo.close(lane);
}

}  // namespace detail
}  // namespace deflate
}  // namespace device
}  // namespace nvcomp
