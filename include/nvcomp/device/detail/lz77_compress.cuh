// nvcomp/device/detail/lz77_compress.cuh -- warp-per-chunk LZ77 matcher shared by the LZ4, Snappy and Deflate
// batched compressors.
//
// One warp owns one chunk.  Each round the 32 lanes hash 32 consecutive
// candidate positions, probe a shared-memory hash table (uint16 positions,
// 4096 entries = 8 KB per warp by default), vote with a ballot for the first verified
// match, extend it cooperatively (32 bytes per compare round) and hand the
// (literal run, offset, length) sequence to the format-specific Emitter.
//
// The compressor feeds the decoder (the graded path); it is written to be
// correct and reasonably parallel, not ratio-optimal: greedy parse, no
// back-extension.  Matches are >= 4 bytes (the hash covers 4 bytes).
//
// Hash inserts are deterministic: when several lanes of a round insert into one bucket, the highest lane's position
// is the one kept.  A same-address shared store from several lanes has no defined winner on the GPU, so without
// this a stream would depend on the hardware as well as on its input; every encoder's stream is pinned byte for
// byte to the host emulator.
//
// Compile-time parameters (LzParams): LZ4 and Snappy use the defaults.  Deflate sets a 32 768-byte window, a
// 258-byte match limit (cooperative extension stops there) and, for its high-compression mode, a 2^15-entry table
// and one-position lazy evaluation.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

constexpr int kHashLog = 12;             // 4096 entries (LZ4's default table size for 64 KB blocks)
constexpr int kHashEntries = 1 << kHashLog;           // uint16 entries
constexpr int kHashBytesPerWarp = kHashEntries * 2;   // 8 KB

template <int kLog = kHashLog>
__device__ __forceinline__ uint32_t hash4(uint32_t v) {
  return (v * 2654435761u) >> (32 - kLog);
}

struct LzParams {
  static constexpr int kHashLog = detail::kHashLog;
  static constexpr uint32_t kMaxDist = 65535u;
  static constexpr uint32_t kMaxLen = 0;        // 0: no limit
  // after a match starting at p is found, if position p + 1 (the next lane, stride 1 only) has a longer verified
  // match at a distance no larger, p becomes a literal and that match is taken instead (one step, not chained).
  // Without the distance condition a Deflate stream of float columns grows: the longer match is often far back,
  // and its distance code costs more than the byte gained.
  static constexpr bool kLazy = false;
};

// Insert position p into bucket h for every lane with `ins`; among lanes with the same bucket the highest one wins.
__device__ __forceinline__ void det_insert(uint16_t* table, uint32_t h, uint32_t p, bool ins, int lane) {
  const unsigned writers = __ballot_sync(kFull, ins);
  const unsigned peers = __match_any_sync(kFull, h) & writers;
  if (ins && lane == 31 - __clz((int)peers)) table[h] = (uint16_t)p;
}

// Cooperative forward extension of a verified 4-byte match at sp against sc: its length, at most
// match_end_limit - sp (and P::kMaxLen).
template <class P>
__device__ __forceinline__ uint32_t lz_extend(const uint8_t* __restrict__ in, uint32_t sp, uint32_t sc,
                                              uint32_t match_end_limit, int lane) {
  uint32_t len = 4;
  uint32_t max_len = match_end_limit - sp;
  if constexpr (P::kMaxLen != 0) max_len = min(max_len, P::kMaxLen);
  while (len < max_len) {
    const uint32_t j = len + lane;
    const bool differs = (j >= max_len) || (in[sp + j] != in[sc + j]);
    const unsigned d = __ballot_sync(kFull, differs);
    if (d) { len += __ffs(d) - 1; break; }
    len += 32;
  }
  if (len > max_len) len = max_len;
  return len;
}

// Emitter concept:
//   void begin(uint8_t* out, uint32_t n_in, int lane)       -- stream preamble
//   void sequence(const uint8_t* lit, uint32_t lit_len, uint32_t off, uint32_t match_len, int lane)
//   void finish(const uint8_t* lit, uint32_t lit_len, int lane)   -- trailing literals
//   uint32_t size()                                         -- bytes produced
//
// step: candidate stride in bytes (1, 2 or 4: the data_type hint).
// min_tail_lit: bytes at the end of the chunk that must stay literals
// match_start_limit: a match may not start within this many bytes of the end.
template <class Emitter, class P = LzParams>
__device__ __forceinline__ void lz77_compress_chunk(
    const uint8_t* __restrict__ in, uint32_t n, Emitter& em, uint16_t* table,
    uint32_t step, uint32_t min_tail_lit, uint32_t match_start_limit, int lane) {
  // clear the table (all candidates point at position 0; verified by compare)
  {
    uint32_t* t32 = (uint32_t*)table;
    for (int i = lane; i < (1 << P::kHashLog) / 2; i += kWarp) t32[i] = 0;
  }
  __syncwarp();

  uint32_t anchor = 0;
  uint32_t pos = 0;
  const uint32_t mstart_end = (n > match_start_limit) ? n - match_start_limit : 0;  // p < mstart_end
  const uint32_t match_end_limit = (n > min_tail_lit) ? n - min_tail_lit : 0;       // match end <= this
  uint32_t misses = 0;

  while (pos < mstart_end) {
    // Skip acceleration on incompressible data: after many empty rounds the
    // stride between probe groups grows (same idea as LZ4's skip strength).
    const uint32_t accel = 1u + (misses >> 3);
    const uint32_t p = pos + (uint32_t)lane * step * accel;
    const bool valid = p < mstart_end;   // guarantees p + 4 <= n
    uint32_t v = 0, h = 0, cand = 0;
    if (valid) {
      v = load_u32(in + p);
      h = hash4<P::kHashLog>(v);
      cand = table[h];
    }
    bool is_match = false;
    uint32_t cpos = 0;
    if (valid) {
      // rebuild the full candidate position from its low 16 bits
      cpos = (p & 0xffff0000u) | cand;
      if (cpos >= p) cpos = (cpos >= 0x10000u) ? cpos - 0x10000u : p;  // -> invalid when cpos == p
      if (cpos < p && (p - cpos) <= P::kMaxDist) is_match = (load_u32(in + cpos) == v);
    }
    // Intra-group candidates: the hash table cannot yet contain positions of this same
    // round, so short-period repeats (typed run-length data: period 1/2/4/8 elements)
    // are caught by comparing against the lanes d positions below.
    {
      const uint32_t stride = step * accel;
#pragma unroll
      for (int d = 1; d <= 8; d <<= 1) {
        const uint32_t vo = __shfl_up_sync(kFull, v, d);
        const bool vvalid = __shfl_up_sync(kFull, valid ? 1 : 0, d) != 0;
        if (!is_match && valid && vvalid && lane >= d && vo == v && (uint32_t)d * stride <= P::kMaxDist) {
          is_match = true;
          cpos = p - (uint32_t)d * stride;
        }
      }
    }
    unsigned m = __ballot_sync(kFull, is_match);
    if (m == 0) {
      det_insert(table, h, p, valid, lane);
      __syncwarp();
      pos += 32u * step * accel;
      if (misses < 64) ++misses;
      continue;
    }
    misses = 0;
    // Every verified candidate of this round stays valid, so the round emits as many matches as fit
    // left to right (greedy): after a match ends, the next candidate at or beyond its end is taken
    // without re-hashing.  Hash entries are inserted for the positions a match consumes up to its
    // start; positions beyond the last match are probed again next round.
    const uint32_t stride = step * accel;
    int prev_first = -1;
    uint32_t new_pos = pos;
    while (m) {
      const int first0 = __ffs(m) - 1;
      uint32_t mp = __shfl_sync(kFull, p, first0);
      uint32_t mc = __shfl_sync(kFull, cpos, first0);
      uint32_t len = lz_extend<P>(in, mp, mc, match_end_limit, lane);
      int lazy = 0;
      if constexpr (P::kLazy) {
        if (stride == 1u && first0 < 31 && ((m >> (first0 + 1)) & 1u)) {
          const uint32_t mp2 = __shfl_sync(kFull, p, first0 + 1);
          const uint32_t mc2 = __shfl_sync(kFull, cpos, first0 + 1);
          const uint32_t len2 = lz_extend<P>(in, mp2, mc2, match_end_limit, lane);
          if (len2 > len && mp2 - mc2 <= mp - mc) { lazy = 1; mp = mp2; mc = mc2; len = len2; }
        }
      }
      const int first = first0 + lazy;
      if (step > 1) len &= ~(step - 1);   // keep candidate positions element-aligned
      prev_first = first;
      if (len < 4) {                       // too short after limits: not a match after all
        m &= ~(1u << first);
        if (new_pos <= mp) new_pos = mp + step;
        continue;
      }
      em.sequence(in + anchor, mp - anchor, mp - mc, len, lane);
      new_pos = mp + len;
      anchor = new_pos;
      const uint32_t skip = (new_pos - pos + stride - 1) / stride;   // lanes whose position is consumed
      if (skip >= 32u) break;
      m &= ~((1u << skip) - 1u);
    }
    // the table is read only at the start of a round, so the inserts can wait for its end
    det_insert(table, h, p, valid && lane <= prev_first, lane);
    __syncwarp();
    pos = (new_pos > pos) ? new_pos : pos + 32u * stride;
  }
  em.finish(in + anchor, n - anchor, lane);
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
