// nvcomp/device/detail/zstd_decode.cuh -- Zstandard (RFC 8878) decode of one chunk by one warp.  The batched kernels
// of zstd.cu (nvcomp_b200/csrc/zstd_decode.cuh re-exports these names) and the device API (nvcomp/device/zstd.cuh)
// share it.  Everything here is a device function taking a lane, with all inline PTX in nvcomp/device/detail/ptx.cuh
// and every shared-memory access through lds_* / sts_*, so tests/emu runs these functions unchanged on the host.
//
// A chunk is what libzstd 1.5.5's one-shot ZSTD_decompress accepts: zero or more Zstandard frames and skippable
// frames, back to back, filling the chunk exactly.  Where libzstd is stricter or looser than the RFC its behaviour is
// followed (the tests pin every rule to it): a compressed block of 128 KB or more is rejected, Huffman codes may be 12
// bits long, a sequence stream may end with the final state update reading past its first byte, the reserved bits of
// the symbol-compression modes byte are ignored, a truncated content checksum is a checksum error.
//
// Shape (DESIGN §3.2):
//   * Frame, block, literals and sequences headers are parsed warp-uniformly.  Raw and RLE blocks are copied / filled
//     straight to the output by the whole warp.
//   * Bit reader (ZBits): the backward reader of FSE and Huffman streams, kept state-for-state equal to libzstd's
//     BIT_DStream_t (64-bit container, bits consumed, reload rules), so that a corrupted stream that reads past its
//     first byte decodes to the same values and the same verdict.  Loads are aligned 32-bit words that hold at least
//     one byte of the stream, so they stay inside the 16-byte granules of the input (the warp_copy contract).
//   * Tables live in the warp's shared memory and persist across the blocks of a frame (Repeat / Treeless modes);
//     what a block may reuse is reset at each frame.  Huffman: one level, 2^12 u16 entries (symbol | nbBits << 8).
//     FSE (LL, ML 2^9, OF 2^8 entries): u32 entries newState | nbBits << 16 | symbol << 24; a symbol's baseline and
//     extra bits come from the per-CTA info tables.  The predefined LL / OF / ML tables and the info tables are built
//     once per CTA (zstd_build_predefined) and only read afterwards.
//   * Every table is built lane-parallel.  FSE spread: cell j (in symbol order) of the normal-probability cells goes
//     to the j-th position of k * step mod size (k = 0, 1, ...) at or below highThreshold -- a ballot compacts that
//     sequence.  A cell's state is its symbol's count plus the cells of the same symbol before it.
//   * Literals: Raw literals are read from the input and RLE literals are a fill.  Huffman literals are decoded by
//     lanes 0-3 (one lane per stream; lane 0 alone for the single-stream form), each ending exactly on its stream's
//     first bit.
//   * Sequences are decoded warp-uniformly; lane k keeps sequence k of a group of 32.  The group then executes in
//     order: each literal run, then each match (warp_match_copy) by the whole warp.
//
// Where Huffman literals are staged.  A block's literals (up to 128 KB) must exist before its sequences consume them.
// They do not fit in shared memory, staging them past `actual` would write outside the decoded bytes, and a per-warp
// global workspace would cost 128 KB per resident warp.  So each compressed block runs two passes:
//   pass 1  decode the sequences without executing them: this validates every literal length and offset and gives
//           the block's output size B = literals + sum of match lengths.  The block is rejected if produced + B > cap.
//   stage   decode the Huffman literals into the block's own output tail [produced + B - lit, produced + B).
//   pass 2  decode the sequences again and execute them.
// Why this is safe: before sequence k runs, L_k / M_k are the literal / match bytes of sequences 0..k-1.  Sequence k
// writes [produced + L_k + M_k, produced + L_{k+1} + M_{k+1}) and reads its literals at produced + M + L_k ..., where
// M = B - lit is the total match length.  Since M_{k+1} <= M, every write ends at or before the next unread literal,
// so nothing unread is overwritten -- provided a copy whose source lies ahead of its destination by less than its
// length loads before it stores (zs_move_fwd).  The last literal run is already in place.  The size query is pass 1
// plus the literal decode with stores off.  Pass 2 keeps every bounds check: a disagreement between the passes is a
// rejected chunk, never a stray write.
// The out-of-line (__noinline__) functions of this header are declared inline: the header is included by every
// translation unit that uses the device API, and inline linkage lets several of them be linked into one program.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"
#include "nvcomp/device/detail/xxhash64.cuh"

namespace nvcomp {
namespace device {
namespace zstd {
namespace detail {

using lz::detail::kWarp;
using lz::detail::kFull;
using lz::detail::warp_copy;
using lz::detail::warp_match_copy;
using lz::detail::ldg_u32;
using lz::detail::lds_u8;
using lz::detail::lds_u16;
using lz::detail::lds_u32;
using lz::detail::sts_u8;
using lz::detail::sts_u16;
using lz::detail::sts_u32;
using lz::detail::st_v4;

enum ZstdResult : int { kZstdOk = 0, kZstdBad = 1, kZstdBadChecksum = 2 };

constexpr uint32_t kZsBlockMax = 1u << 17;            // Block_Maximum_Size
constexpr uint32_t kZsHufMaxLog = 12;                 // libzstd's HUF_TABLELOG_MAX
// per-warp shared memory layout (byte offsets)
constexpr uint32_t kZsHufOff = 0;                     // u16[4096] Huffman decode table
constexpr uint32_t kZsLLOff = kZsHufOff + 2 * 4096;   // u32[512]  literal-length FSE table
constexpr uint32_t kZsOFOff = kZsLLOff + 4 * 512;     // u32[256]  offset-code FSE table
constexpr uint32_t kZsMLOff = kZsOFOff + 4 * 256;     // u32[512]  match-length FSE table
constexpr uint32_t kZsWtOff = kZsMLOff + 4 * 512;     // u32[64]   FSE table of the Huffman weights
constexpr uint32_t kZsNormOff = kZsWtOff + 4 * 64;    // s16[256]  normalized counts
constexpr uint32_t kZsWeightOff = kZsNormOff + 512;   // u8[256]   Huffman weights
constexpr uint32_t kZsSymOff = kZsWeightOff + 256;    // u8[512]   FSE build: symbol of each cell
constexpr uint32_t kZsSeqOff = kZsSymOff + 512;       // u8[512]   FSE build: symbols in spread order
constexpr uint32_t kZsNextOff = kZsSeqOff + 512;      // u16[256]  FSE build: next state of each symbol
constexpr uint32_t kZsWarpSmem = kZsNextOff + 512;    // 15 872 bytes
// per-CTA predefined tables (built once, read-only)
constexpr uint32_t kZsPreLLOff = 0;                   // u32[64]  predefined LL table (accuracy log 6)
constexpr uint32_t kZsPreOFOff = 256;                 // u32[32]  predefined OF table (accuracy log 5)
constexpr uint32_t kZsPreMLOff = 384;                 // u32[64]  predefined ML table (accuracy log 6)
constexpr uint32_t kZsLLInfoOff = 640;                // u32[36]  LL code -> baseline | extra bits << 24
constexpr uint32_t kZsMLInfoOff = 784;                // u32[53]  ML code -> baseline | extra bits << 24
constexpr uint32_t kZsPreSmem = 1024;

struct ZstdWarp {
  uint32_t smem;     // this warp's tables and scratch (kZsWarpSmem bytes)
  uint32_t predef;   // the CTA's predefined tables (kZsPreSmem bytes)
};

__device__ __forceinline__ uint32_t zs_highbit(uint32_t v) { return 31u - (uint32_t)__clz((int)v); }   // v > 0
__device__ __forceinline__ uint32_t zs_le16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
__device__ __forceinline__ uint32_t zs_le24(const uint8_t* p) { return zs_le16(p) | ((uint32_t)p[2] << 16); }
__device__ __forceinline__ uint32_t zs_le32(const uint8_t* p) { return zs_le24(p) | ((uint32_t)p[3] << 24); }

// 8 little-endian bytes at p from the aligned words that hold them
__device__ __forceinline__ uint64_t zs_ld64(const uint8_t* p) {
  const uint32_t a = (uint32_t)((uintptr_t)p & 3u);
  const uint8_t* w = p - a;
  const uint32_t w0 = ldg_u32<0>(w), w1 = ldg_u32<4>(w);
  if (a == 0) return (uint64_t)w0 | ((uint64_t)w1 << 32);
  const uint32_t w2 = ldg_u32<8>(w);
  return (uint64_t)__funnelshift_r(w0, w1, 8u * a) | ((uint64_t)__funnelshift_r(w1, w2, 8u * a) << 32);
}

// ---------------------------------------------------------------------------
// Backward bit reader, state-for-state libzstd's BIT_DStream_t
// ---------------------------------------------------------------------------
enum ZsReload : uint32_t { kZsUnfinished = 0, kZsEndOfBuffer = 1, kZsCompleted = 2, kZsOverflow = 3 };

struct ZBits {
  const uint8_t* base;   // first byte of the stream
  uint64_t c;            // container: stream bytes [ptr, ptr + 8), read from the top bit down
  uint32_t ptr;          // offset of the container's first byte
  uint32_t consumed;     // bits of the container already read

  // false for an empty stream or one whose last byte (the one holding the sentinel bit) is zero
  __device__ __forceinline__ bool init(const uint8_t* src, uint32_t size) {
    base = src;
    ptr = 0;
    c = 0;
    consumed = 0;
    if (size == 0) return false;
    const uint32_t last = src[size - 1];
    if (last == 0) return false;
    if (size >= 8) {
      ptr = size - 8;
      c = zs_ld64(src + ptr);
      consumed = 8u - zs_highbit(last);
    } else {
      for (uint32_t i = 0; i < size; ++i) c |= (uint64_t)src[i] << (8 * i);
      consumed = 8u - zs_highbit(last) + 8u * (8u - size);
    }
    return true;
  }
  __device__ __forceinline__ uint32_t look(uint32_t n) const {       // BIT_lookBits, n <= 32
    return (uint32_t)(((c << (consumed & 63u)) >> 1) >> ((63u - n) & 63u));
  }
  __device__ __forceinline__ uint32_t read(uint32_t n) {
    const uint32_t v = look(n);
    consumed += n;
    return v;
  }
  __device__ __forceinline__ uint32_t reload() {
    if (consumed > 64u) return kZsOverflow;
    if (ptr >= 8u) {
      ptr -= consumed >> 3;
      consumed &= 7u;
      c = zs_ld64(base + ptr);
      return kZsUnfinished;
    }
    if (ptr == 0u) return consumed < 64u ? kZsEndOfBuffer : kZsCompleted;
    uint32_t nb = consumed >> 3, r = kZsUnfinished;
    if (nb > ptr) {
      nb = ptr;
      r = kZsEndOfBuffer;
    }
    ptr -= nb;
    consumed -= 8u * nb;
    c = zs_ld64(base + ptr);
    return r;
  }
  __device__ __forceinline__ bool finished() const { return ptr == 0u && consumed == 64u; }
};

// exclusive warp scan; *total = sum over the warp
__device__ __forceinline__ uint32_t zs_scan_excl(uint32_t v, uint32_t* total, int lane) {
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(kFull, inc, d);
    if (lane >= d) inc += t;
  }
  *total = __shfl_sync(kFull, inc, 31);
  return inc - v;
}

// ---------------------------------------------------------------------------
// FSE table description (libzstd FSE_readNCount, step for step: the clamped reads near the end of the header and the
// zero padding of a header shorter than 8 bytes decide the verdict of truncated headers).  Writes norm[0, *max_sv]
// (s16) and returns the header's size in bytes, or -1.
// ---------------------------------------------------------------------------
inline __device__ __noinline__ int zs_read_ncount(const uint8_t* src, uint32_t hb, uint32_t norm_a, uint32_t* max_sv,
                                                  uint32_t* table_log, int lane) {
  const int iend = hb < 8u ? 8 : (int)hb;
  auto rd32 = [&](int i) -> uint32_t {
    uint32_t v = 0;
    for (int k = 0; k < 4; ++k) {
      const uint32_t j = (uint32_t)(i + k);
      v |= (j < hb ? (uint32_t)src[j] : 0u) << (8 * k);
    }
    return v;
  };
  const uint32_t max_sv1 = *max_sv + 1u;
  for (uint32_t s = (uint32_t)lane; s < max_sv1; s += 32u) sts_u16(norm_a + 2u * s, 0u);
  __syncwarp();
  int ip = 0;
  uint32_t bits = rd32(0);
  int nb = (int)(bits & 15u) + 5;
  if (nb > 15) return -1;
  bits >>= 4;
  int bit_count = 4;
  *table_log = (uint32_t)nb;
  int remaining = (1 << nb) + 1;
  int threshold = 1 << nb;
  ++nb;
  uint32_t charnum = 0;
  bool previous0 = false;
  auto advance = [&]() {
    if (ip <= iend - 7 || ip + (bit_count >> 3) <= iend - 4) {
      ip += bit_count >> 3;
      bit_count &= 7;
    } else {
      bit_count -= 8 * (iend - 4 - ip);
      bit_count &= 31;
      ip = iend - 4;
    }
    bits = rd32(ip) >> bit_count;
  };
  for (;;) {
    if (previous0) {
      int repeats = (__ffs((int)(~bits | 0x80000000u)) - 1) >> 1;
      while (repeats >= 12) {
        charnum += 36u;
        if (ip <= iend - 7) {
          ip += 3;
        } else {
          bit_count -= 8 * (iend - 7 - ip);
          bit_count &= 31;
          ip = iend - 4;
        }
        bits = rd32(ip) >> bit_count;
        repeats = (__ffs((int)(~bits | 0x80000000u)) - 1) >> 1;
      }
      charnum += 3u * (uint32_t)repeats;
      bits >>= 2 * repeats;
      bit_count += 2 * repeats;
      charnum += bits & 3u;
      bit_count += 2;
      if (charnum >= max_sv1) break;
      advance();
    }
    const int maxv = (2 * threshold - 1) - remaining;
    int count;
    if ((int)(bits & (uint32_t)(threshold - 1)) < maxv) {
      count = (int)(bits & (uint32_t)(threshold - 1));
      bit_count += nb - 1;
    } else {
      count = (int)(bits & (uint32_t)(2 * threshold - 1));
      if (count >= threshold) count -= maxv;
      bit_count += nb;
    }
    --count;
    if (count >= 0) remaining -= count;
    else remaining += count;
    if (lane == 0) sts_u16(norm_a + 2u * charnum, (uint32_t)count & 0xffffu);
    ++charnum;
    previous0 = count == 0;
    if (remaining < threshold) {
      if (remaining <= 1) break;
      nb = (int)zs_highbit((uint32_t)remaining) + 1;
      threshold = 1 << (nb - 1);
    }
    if (charnum >= max_sv1) break;
    advance();
  }
  __syncwarp();
  if (remaining != 1 || charnum > max_sv1 || bit_count > 32) return -1;
  *max_sv = charnum - 1u;
  ip += (bit_count + 7) >> 3;
  if (hb < 8u && (uint32_t)ip > hb) return -1;
  return ip;
}

// ---------------------------------------------------------------------------
// FSE decode table from norm[0, max_sv] (accuracy log `log`, 5..9) into tab_a: entry = newState | nbBits << 16 |
// symbol << 24.
// ---------------------------------------------------------------------------
inline __device__ __noinline__ void zs_build_fse(uint32_t norm_a, uint32_t max_sv, uint32_t log, uint32_t tab_a,
                                                 uint32_t smem, int lane) {
  const uint32_t ul = (uint32_t)lane;
  const unsigned below = (1u << ul) - 1u;
  const uint32_t size = 1u << log;
  const uint32_t sym_a = smem + kZsSymOff, seq_a = smem + kZsSeqOff, next_a = smem + kZsNextOff;
  // low-probability symbols take the cells from size - 1 down; the others are listed in spread order
  uint32_t lows = 0, cum = 0;
  for (uint32_t s0 = 0; s0 <= max_sv; s0 += 32u) {
    const uint32_t s = s0 + ul;
    const int n = s <= max_sv ? (int)(int16_t)lds_u16(norm_a + 2u * s) : 0;
    const unsigned m = __ballot_sync(kFull, n == -1);
    const uint32_t w = n > 0 ? (uint32_t)n : 0u;
    uint32_t tot;
    const uint32_t ex = zs_scan_excl(w, &tot, lane);
    if (n == -1) sts_u8(sym_a + size - 1u - (lows + (uint32_t)__popc(m & below)), s);
    if (s <= max_sv) sts_u16(next_a + 2u * s, n == -1 ? 1u : w);
    for (uint32_t j = 0; j < w; ++j) sts_u8(seq_a + cum + ex + j, s);
    lows += (uint32_t)__popc(m);
    cum += tot;
  }
  __syncwarp();
  // spread: the j-th normal cell goes to the j-th position k * step (mod size) at or below highThreshold
  const uint32_t high = size - 1u - lows, step = (size >> 1) + (size >> 3) + 3u, mask = size - 1u;
  uint32_t placed = 0;
  for (uint32_t k0 = 0; k0 < size; k0 += 32u) {
    const uint32_t p = ((k0 + ul) * step) & mask;
    const bool ok = p <= high;
    const unsigned m = __ballot_sync(kFull, ok);
    if (ok) sts_u8(sym_a + p, lds_u8(seq_a + placed + (uint32_t)__popc(m & below)));
    placed += (uint32_t)__popc(m);
  }
  __syncwarp();
  // states: cell u of symbol s gets next[s]++ in cell order
  for (uint32_t u0 = 0; u0 < size; u0 += 32u) {
    const uint32_t u = u0 + ul;
    const uint32_t s = lds_u8(sym_a + u);
    uint32_t rank = 0;
    bool last = true;
    for (int r = 0; r < 32; ++r) {
      const uint32_t o = __shfl_sync(kFull, s, r);
      if (o == s && r < lane) ++rank;
      if (o == s && r > lane) last = false;
    }
    const uint32_t ns = lds_u16(next_a + 2u * s) + rank;
    __syncwarp();
    if (last) sts_u16(next_a + 2u * s, ns + 1u);
    const uint32_t nbits = log - zs_highbit(ns);
    sts_u32(tab_a + 4u * u, ((ns << nbits) - size) | (nbits << 16) | (s << 24));
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// Predefined tables and code info (once per CTA)
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t zs_ll_info(uint32_t c) {
  if (c < 16u) return c;
  if (c >= 25u) return (1u << (c - 19u)) | ((c - 19u) << 24);
  uint32_t base = 16u, bits = 1u;
  for (uint32_t i = 0; i <= c - 16u; ++i) {
    bits = i < 4u ? 1u : i >> 1;
    if (i < c - 16u) base += 1u << bits;
  }
  return base | (bits << 24);
}
__device__ __forceinline__ uint32_t zs_ml_info(uint32_t c) {
  if (c < 32u) return c + 3u;
  if (c >= 43u) return ((1u << (c - 36u)) + 3u) | ((c - 36u) << 24);
  uint32_t base = 35u, bits = 1u;
  for (uint32_t i = 0; i <= c - 32u; ++i) {
    bits = i < 4u ? 1u : i >> 1;
    if (i < c - 32u) base += 1u << bits;
  }
  return base | (bits << 24);
}

// builds the CTA's predefined tables at predef, using the scratch of the warp at smem
inline __device__ __noinline__ void zstd_build_predefined(uint32_t predef, uint32_t smem, int lane) {
  const int8_t ll[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                         2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
  const int8_t ml[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                         1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
  const int8_t of[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
  const uint32_t norm_a = smem + kZsNormOff, ul = (uint32_t)lane;
  for (uint32_t s = ul; s < 36u; s += 32u) sts_u16(norm_a + 2u * s, (uint32_t)(int)ll[s] & 0xffffu);
  __syncwarp();
  zs_build_fse(norm_a, 35, 6, predef + kZsPreLLOff, smem, lane);
  for (uint32_t s = ul; s < 53u; s += 32u) sts_u16(norm_a + 2u * s, (uint32_t)(int)ml[s] & 0xffffu);
  __syncwarp();
  zs_build_fse(norm_a, 52, 6, predef + kZsPreMLOff, smem, lane);
  for (uint32_t s = ul; s < 29u; s += 32u) sts_u16(norm_a + 2u * s, (uint32_t)(int)of[s] & 0xffffu);
  __syncwarp();
  zs_build_fse(norm_a, 28, 5, predef + kZsPreOFOff, smem, lane);
  for (uint32_t c = ul; c < 53u; c += 32u) {
    if (c < 36u) sts_u32(predef + kZsLLInfoOff + 4u * c, zs_ll_info(c));
    sts_u32(predef + kZsMLInfoOff + 4u * c, zs_ml_info(c));
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------
// Huffman tree description (libzstd HUF_readStats) -> the warp's single-level decode table.  Returns the
// description's size in bytes, or -1; *log = the code's table log.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t zs_fse_symbol(uint32_t& state, uint32_t tab_a, ZBits& br) {
  const uint32_t e = lds_u32(tab_a + 4u * state);
  state = (e & 0xffffu) + br.read((e >> 16) & 0xffu);
  return e >> 24;
}

// FSE-compressed weights (libzstd FSE_decompress_wksp, two interleaved states, at most 255 weights); returns the
// number of weights or -1
inline __device__ __noinline__ int zs_fse_weights(const uint8_t* src, uint32_t n, uint32_t smem, int lane) {
  const uint32_t norm_a = smem + kZsNormOff, tab_a = smem + kZsWtOff, w_a = smem + kZsWeightOff;
  uint32_t max_sv = 255, log = 0;
  const int hs = zs_read_ncount(src, n, norm_a, &max_sv, &log, lane);
  if (hs < 0 || log > 6u) return -1;
  zs_build_fse(norm_a, max_sv, log, tab_a, smem, lane);
  ZBits br;
  if (!br.init(src + hs, n - (uint32_t)hs)) return -1;
  uint32_t s1 = br.read(log);
  br.reload();
  uint32_t s2 = br.read(log);
  br.reload();
  uint32_t op = 0;
  auto put = [&](uint32_t v) {
    if (lane == 0) sts_u8(w_a + op, v);
    ++op;
  };
  while ((br.reload() == kZsUnfinished) & (op < 252u)) {
    put(zs_fse_symbol(s1, tab_a, br));
    put(zs_fse_symbol(s2, tab_a, br));
    put(zs_fse_symbol(s1, tab_a, br));
    put(zs_fse_symbol(s2, tab_a, br));
  }
  while (true) {
    if (op > 253u) return -1;
    put(zs_fse_symbol(s1, tab_a, br));
    if (br.reload() == kZsOverflow) {
      put(zs_fse_symbol(s2, tab_a, br));
      break;
    }
    if (op > 253u) return -1;
    put(zs_fse_symbol(s2, tab_a, br));
    if (br.reload() == kZsOverflow) {
      put(zs_fse_symbol(s1, tab_a, br));
      break;
    }
  }
  __syncwarp();
  return (int)op;
}

inline __device__ __noinline__ int zs_read_huffman(const uint8_t* src, uint32_t n, uint32_t smem, uint32_t* log_out,
                                                   int lane) {
  const uint32_t ul = (uint32_t)lane;
  const unsigned below = (1u << ul) - 1u;
  const uint32_t w_a = smem + kZsWeightOff, tab_a = smem + kZsHufOff;
  if (n == 0) return -1;
  uint32_t isize = src[0], osize;
  if (isize >= 128u) {
    osize = isize - 127u;
    isize = (osize + 1u) / 2u;
    if (isize + 1u > n) return -1;
    for (uint32_t i = ul; i < osize; i += 32u) {
      const uint32_t b = src[1u + i / 2u];
      sts_u8(w_a + i, (i & 1u) ? b & 15u : b >> 4);
    }
    __syncwarp();
  } else {
    if (isize + 1u > n) return -1;
    const int r = zs_fse_weights(src + 1, isize, smem, lane);
    if (r < 0) return -1;
    osize = (uint32_t)r;
  }
  // weight statistics: every weight <= 12, the implied last weight completes a power of two
  uint32_t total = 0;
  bool bad = false;
  for (uint32_t i0 = 0; i0 < osize; i0 += 32u) {
    const uint32_t i = i0 + ul;
    const uint32_t w = i < osize ? lds_u8(w_a + i) : 0u;
    bad |= w > kZsHufMaxLog;
    total += w ? 1u << (w - 1u) : 0u;
  }
  if (__any_sync(kFull, bad)) return -1;
  total = __reduce_add_sync(kFull, total);
  if (total == 0u) return -1;
  const uint32_t log = zs_highbit(total) + 1u;
  if (log > kZsHufMaxLog) return -1;
  const uint32_t rest = (1u << log) - total;
  if ((1u << zs_highbit(rest)) != rest) return -1;
  if (lane == 0) sts_u8(w_a + osize, zs_highbit(rest) + 1u);
  __syncwarp();
  const uint32_t nsym = osize + 1u;
  // codes per weight (lane w counts weight w) and each symbol's rank among the symbols of its weight
  uint32_t cnt = 0;
  for (uint32_t s0 = 0; s0 < nsym; s0 += 32u) {
    const uint32_t s = s0 + ul;
    const uint32_t w = s < nsym ? lds_u8(w_a + s) : 0u;
    unsigned present = __reduce_or_sync(kFull, w ? 1u << w : 0u);
    while (present) {
      const uint32_t q = (uint32_t)__ffs((int)present) - 1u;
      present &= present - 1u;
      const unsigned m = __ballot_sync(kFull, w == q);
      if (ul == q) cnt += (uint32_t)__popc(m);
    }
  }
  const uint32_t c1 = __shfl_sync(kFull, cnt, 1);
  if (c1 < 2u || (c1 & 1u)) return -1;
  // first entry of weight w: the entries of the lighter weights come first
  uint32_t tot;
  const uint32_t start = zs_scan_excl((ul >= 1u && ul <= log) ? cnt << (ul - 1u) : 0u, &tot, lane);
  uint32_t next = start;       // lane w: next entry of weight w
  for (uint32_t s0 = 0; s0 < nsym; s0 += 32u) {
    const uint32_t s = s0 + ul;
    const uint32_t w = s < nsym ? lds_u8(w_a + s) : 0u;
    const uint32_t base = __shfl_sync(kFull, next, (int)w);
    uint32_t rk = 0;
    unsigned present = __reduce_or_sync(kFull, w ? 1u << w : 0u);
    while (present) {
      const uint32_t q = (uint32_t)__ffs((int)present) - 1u;
      present &= present - 1u;
      const unsigned m = __ballot_sync(kFull, w == q);
      if (w == q) rk = (uint32_t)__popc(m & below);
      if (ul == q) next += (uint32_t)__popc(m) << (q - 1u);
    }
    if (w) {
      const uint32_t len = 1u << (w - 1u), e = s | ((log + 1u - w) << 8);
      const uint32_t first = base + (rk << (w - 1u));
      for (uint32_t i = 0; i < len; ++i) sts_u16(tab_a + 2u * (first + i), e);
    }
  }
  __syncwarp();
  *log_out = log;
  return (int)isize + 1;
}

// ---------------------------------------------------------------------------
// Huffman literal streams -> dst[0, lit) (nothing is written with kCount).  Lane k < streams decodes stream k.
// ---------------------------------------------------------------------------
template <bool kCount>
__device__ __noinline__ bool zs_huffman_literals(const uint8_t* src, uint32_t n, bool single, uint32_t lit,
                                                 uint8_t* dst, uint32_t log, uint32_t smem, int lane) {
  uint32_t so = 0, sl = n, lo = 0, hi = lit;
  const uint32_t streams = single ? 1u : 4u;
  if (!single) {
    if (n < 10u) return false;
    const uint32_t l1 = zs_le16(src), l2 = zs_le16(src + 2), l3 = zs_le16(src + 4);
    if (l1 + l2 + l3 + 6u > n) return false;
    const uint32_t seg = (lit + 3u) / 4u;
    if (3u * seg > lit) return false;
    const uint32_t k = (uint32_t)lane & 3u;
    so = 6u + (k > 0 ? l1 : 0u) + (k > 1 ? l2 : 0u) + (k > 2 ? l3 : 0u);
    sl = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : n - (l1 + l2 + l3 + 6u);
    lo = k * seg;
    hi = k == 3 ? lit : lo + seg;
  }
  bool ok = true;
  if ((uint32_t)lane < streams) {
    const uint32_t tab_a = smem + kZsHufOff;
    ZBits br;
    ok = br.init(src + so, sl);
    for (uint32_t i = lo; ok && i < hi; ++i) {
      if (br.consumed > 64u - kZsHufMaxLog && br.reload() == kZsOverflow) ok = false;
      const uint32_t e = lds_u16(tab_a + 2u * br.look(log));
      br.consumed += e >> 8;
      if (!kCount) dst[i] = (uint8_t)e;
    }
    if (ok) {
      br.reload();
      ok = br.finished();
    }
  }
  const bool all = __all_sync(kFull, ok);
  __syncwarp();
  return all;
}

// ---------------------------------------------------------------------------
// Sequences
// ---------------------------------------------------------------------------
// Decoder state that persists across the blocks of a frame
struct ZsFrame {
  uint32_t rep[3];
  bool fse_entropy;         // a block of this frame has decoded sequences (Repeat mode allowed)
  bool lit_entropy;         // a block of this frame has decoded Huffman literals (Treeless mode allowed)
  uint32_t huf_log;
  uint32_t tab[3], log[3];  // current LL, OF, ML tables (shared-memory address, accuracy log)
};

enum : int { kZsLL = 0, kZsOF = 1, kZsML = 2 };

// one symbol-compression mode of the sequences header; returns the bytes it reads, or -1
__device__ __forceinline__ int zs_seq_table(int which, uint32_t mode, const uint8_t* src, uint32_t avail, ZsFrame& f,
                                            const ZstdWarp& ws, int lane) {
  const uint32_t max = which == kZsLL ? 35u : which == kZsOF ? 31u : 52u;
  const uint32_t max_log = which == kZsOF ? 8u : 9u;
  const uint32_t own = ws.smem + (which == kZsLL ? kZsLLOff : which == kZsOF ? kZsOFOff : kZsMLOff);
  if (mode == 0u) {                                    // Predefined
    f.tab[which] = ws.predef + (which == kZsLL ? kZsPreLLOff : which == kZsOF ? kZsPreOFOff : kZsPreMLOff);
    f.log[which] = which == kZsOF ? 5u : 6u;
    return 0;
  }
  if (mode == 1u) {                                    // RLE: a one-cell table
    if (avail == 0u) return -1;
    const uint32_t sym = src[0];
    if (sym > max) return -1;
    if (lane == 0) sts_u32(own, sym << 24);
    __syncwarp();
    f.tab[which] = own;
    f.log[which] = 0;
    return 1;
  }
  if (mode == 2u) {                                    // FSE_Compressed
    uint32_t max_sv = max, log = 0;
    const int hs = zs_read_ncount(src, avail, ws.smem + kZsNormOff, &max_sv, &log, lane);
    if (hs < 0 || log > max_log) return -1;
    zs_build_fse(ws.smem + kZsNormOff, max_sv, log, own, ws.smem, lane);
    f.tab[which] = own;
    f.log[which] = log;
    return hs;
  }
  return f.fse_entropy ? 0 : -1;                       // Repeat
}

struct ZsSeq {
  uint32_t sll, sof, sml;
  uint32_t rep0, rep1, rep2;
};

// libzstd ZSTD_initFseState x 3 (LL, OF, ML)
__device__ __forceinline__ void zs_seq_init(ZsSeq& q, ZBits& br, const ZsFrame& f) {
  q.sll = br.read(f.log[kZsLL]);
  br.reload();
  q.sof = br.read(f.log[kZsOF]);
  br.reload();
  q.sml = br.read(f.log[kZsML]);
  br.reload();
  q.rep0 = f.rep[0];
  q.rep1 = f.rep[1];
  q.rep2 = f.rep[2];
}

// libzstd 1.5.5 ZSTD_decodeSequence (64-bit): offset bits, match-length bits, literal-length bits, then the LL, ML, OF
// state updates (after every sequence, the last one included)
__device__ __forceinline__ void zs_seq_decode(ZsSeq& q, ZBits& br, const ZsFrame& f, uint32_t predef, uint32_t& ll,
                                              uint32_t& ml, uint32_t& off) {
  const uint32_t ell = lds_u32(f.tab[kZsLL] + 4u * q.sll);
  const uint32_t eml = lds_u32(f.tab[kZsML] + 4u * q.sml);
  const uint32_t eof = lds_u32(f.tab[kZsOF] + 4u * q.sof);
  const uint32_t lli = lds_u32(predef + kZsLLInfoOff + 4u * (ell >> 24));
  const uint32_t mli = lds_u32(predef + kZsMLInfoOff + 4u * (eml >> 24));
  const uint32_t ofc = eof >> 24;
  const uint32_t llb = lli >> 24, mlb = mli >> 24, ofb = ofc;
  const uint32_t llbase = lli & 0xffffffu;
  if (ofb > 1u) {
    off = ((1u << ofc) - 3u) + br.read(ofb);
    q.rep2 = q.rep1;
    q.rep1 = q.rep0;
    q.rep0 = off;
  } else {
    const uint32_t ll0 = llbase == 0u;
    if (ofb == 0u) {
      off = ll0 ? q.rep1 : q.rep0;
      q.rep1 = ll0 ? q.rep0 : q.rep1;
      q.rep0 = off;
    } else {
      const uint32_t o = 1u + ll0 + br.read(1);
      uint32_t t = o == 3u ? q.rep0 - 1u : o == 1u ? q.rep1 : q.rep2;
      t += t == 0u;
      if (o != 1u) q.rep2 = q.rep1;
      q.rep1 = q.rep0;
      q.rep0 = t;
      off = t;
    }
  }
  ml = (mli & 0xffffffu) + (mlb ? br.read(mlb) : 0u);
  if (llb + mlb + ofb >= 31u) br.reload();
  ll = llbase + (llb ? br.read(llb) : 0u);
  q.sll = (ell & 0xffffu) + br.read((ell >> 16) & 0xffu);
  q.sml = (eml & 0xffffu) + br.read((eml >> 16) & 0xffu);
  q.sof = (eof & 0xffffu) + br.read((eof >> 16) & 0xffu);
}

// ---------------------------------------------------------------------------
// Output helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ void zs_fill(uint8_t* dst, uint32_t b, uint32_t n, int lane) {
  const uint32_t ul = (uint32_t)lane;
  const uint32_t head = min((16u - (uint32_t)((uintptr_t)dst & 15u)) & 15u, n);
  if (ul < head) dst[ul] = (uint8_t)b;
  const uint32_t nvec = (n - head) >> 4;
  const uint32_t w = b * 0x01010101u;
  const uint4 v = make_uint4(w, w, w, w);
  uint4* d16 = (uint4*)(dst + head);
  for (uint32_t i = ul; i < nvec; i += 32u) st_v4(d16 + i, v);
  const uint32_t done = head + (nvec << 4);
  if (done + ul < n) dst[done + ul] = (uint8_t)b;
}

// dst[0, n) = src[0, n) where src = dst + d for some d >= 0 (a forward move inside the output).  Every span loads
// before it stores.
__device__ __forceinline__ void zs_move_fwd(uint8_t* dst, const uint8_t* src, uint32_t n, int lane) {
  const uint32_t d = (uint32_t)(src - dst);
  if (d == 0u || n == 0u) return;
  if (d >= n) {
    warp_copy<false>(dst, src, n, lane);
    return;
  }
  if (d >= 512u) {
    for (uint32_t o = 0; o < n; o += d) {
      warp_copy<false>(dst + o, src + o, min(d, n - o), lane);
      __syncwarp();
    }
    return;
  }
  for (uint32_t o = 0; o < n; o += 32u) {
    const uint32_t i = o + (uint32_t)lane;
    const uint32_t v = i < n ? src[i] : 0u;
    __syncwarp();
    if (i < n) dst[i] = (uint8_t)v;
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// One compressed block in[bp, bp + bsize).  produced: the chunk's bytes so far (this frame started at frame_start).
// ---------------------------------------------------------------------------
template <bool kCount>
__device__ __forceinline__ bool zs_compressed_block(const uint8_t* in, uint32_t bp, uint32_t bsize, uint8_t* out,
                                                    uint32_t cap, uint32_t& produced, uint32_t frame_start,
                                                    ZsFrame& f, const ZstdWarp& ws, int lane) {
  if (bsize >= kZsBlockMax || bsize < 2u) return false;
  const uint8_t* b = in + bp;
  const uint32_t b0 = b[0], ltype = b0 & 3u, lhl = (b0 >> 2) & 3u;
  const uint32_t room = min(kZsBlockMax, cap - produced);
  uint32_t lit = 0, lit_sec = 0, raw_off = 0, rle = 0, huf_off = 0, huf_len = 0;
  bool single = true;
  // literals section header
  if (ltype < 2u) {
    uint32_t lh;
    if (lhl == 1u) {
      if (ltype == 1u && bsize < 3u) return false;
      lh = 2;
      lit = zs_le16(b) >> 4;
    } else if (lhl == 3u) {
      if (bsize < (ltype == 1u ? 4u : 3u)) return false;
      lh = 3;
      lit = zs_le24(b) >> 4;
    } else {
      lh = 1;
      lit = b0 >> 3;
    }
    if (lit > room) return false;
    if (ltype == 0u) {
      if (lh + lit > bsize) return false;
      raw_off = bp + lh;
      lit_sec = lh + lit;
    } else {
      rle = b[lh];
      lit_sec = lh + 1u;
    }
  } else {
    if (ltype == 3u && !f.lit_entropy) return false;
    if (bsize < 5u) return false;
    const uint32_t lhc = zs_le32(b);
    uint32_t lh, csz;
    if (lhl < 2u) {
      single = lhl == 0u;
      lh = 3;
      lit = (lhc >> 4) & 0x3ffu;
      csz = (lhc >> 14) & 0x3ffu;
    } else if (lhl == 2u) {
      single = false;
      lh = 4;
      lit = (lhc >> 4) & 0x3fffu;
      csz = lhc >> 18;
    } else {
      single = false;
      lh = 5;
      lit = (lhc >> 4) & 0x3ffffu;
      csz = (lhc >> 22) + ((uint32_t)b[4] << 10);
    }
    if (lit > kZsBlockMax) return false;
    if (!single && lit < 6u) return false;
    if (csz + lh > bsize) return false;
    if (room < lit) return false;
    huf_off = bp + lh;
    huf_len = csz;
    if (ltype == 2u) {
      const int hs = zs_read_huffman(in + huf_off, huf_len, ws.smem, &f.huf_log, lane);
      if (hs < 0 || (uint32_t)hs >= huf_len) return false;
      huf_off += (uint32_t)hs;
      huf_len -= (uint32_t)hs;
    }
    f.lit_entropy = true;
    lit_sec = lh + csz;
  }
  // sequences section header
  const uint32_t bend = bp + bsize;
  uint32_t sp = bp + lit_sec;
  if (sp >= bend) return false;
  // Only a first byte of 0 ends the section.  The 2-byte form can also spell a count of 0 (0x80 0x00); the modes
  // byte and the table descriptions still follow it and are built (a later block may repeat them), and the bytes
  // after them are ignored, as libzstd does.
  const uint32_t nb0 = in[sp++];
  uint32_t nseq = nb0;
  if (nb0 == 0u) {
    if (sp != bend) return false;
  } else if (nb0 == 255u) {
    if (sp + 2u > bend) return false;
    nseq = zs_le16(in + sp) + 0x7f00u;
    sp += 2u;
  } else if (nb0 >= 128u) {
    if (sp >= bend) return false;
    nseq = ((nb0 - 128u) << 8) + in[sp++];
  }
  if (nb0) {
    if (sp + 1u > bend) return false;
    const uint32_t modes = in[sp++];                  // libzstd 1.5.5 ignores the two reserved bits
    int r = zs_seq_table(kZsLL, modes >> 6, in + sp, bend - sp, f, ws, lane);
    if (r < 0) return false;
    sp += (uint32_t)r;
    r = zs_seq_table(kZsOF, (modes >> 4) & 3u, in + sp, bend - sp, f, ws, lane);
    if (r < 0) return false;
    sp += (uint32_t)r;
    r = zs_seq_table(kZsML, (modes >> 2) & 3u, in + sp, bend - sp, f, ws, lane);
    if (r < 0) return false;
    sp += (uint32_t)r;
    if (nseq) f.fse_entropy = true;                   // libzstd: set once sequences are decoded
  }
  // pass 1: validate the sequences, measure the block
  const uint32_t fpos0 = produced - frame_start;     // frame-local position of the block
  uint64_t mtotal = 0;
  ZsSeq q1{};
  if (nseq) {
    ZBits br;
    if (!br.init(in + sp, bend - sp)) return false;
    zs_seq_init(q1, br, f);
    uint32_t lit_left = lit;
    uint64_t pos = fpos0;
    for (uint32_t k = 0;;) {
      uint32_t ll, ml, off;
      zs_seq_decode(q1, br, f, ws.predef, ll, ml, off);
      if (ll > lit_left) return false;
      lit_left -= ll;
      pos += ll;
      if (off > pos) return false;                    // the match reaches back before the frame
      pos += ml;
      mtotal += ml;
      if ((uint64_t)produced + lit + mtotal > cap) return false;
      if (++k == nseq) break;
      br.reload();
    }
    if (br.reload() < kZsCompleted) return false;     // the stream is not consumed
  }
  const uint64_t bout64 = (uint64_t)lit + mtotal;
  if ((uint64_t)produced + bout64 > cap) return false;
  const uint32_t bout = (uint32_t)bout64, tail = (uint32_t)mtotal;
  uint8_t* bo = kCount ? nullptr : out + produced;
  // stage the Huffman literals in the block's output tail
  if (ltype >= 2u && !zs_huffman_literals<kCount>(in + huf_off, huf_len, single, lit, kCount ? nullptr : bo + tail,
                                                  f.huf_log, ws.smem, lane))
    return false;
  if (kCount) {
    f.rep[0] = q1.rep0;
    f.rep[1] = q1.rep1;
    f.rep[2] = q1.rep2;
    produced += bout;
    return true;
  }
  // pass 2: decode again and execute
  uint32_t used = 0, w = 0;                           // literals consumed, block bytes written
  auto literals = [&](uint32_t n) {
    if (ltype == 0u) warp_copy<true>(bo + w, in + raw_off + used, n, lane);
    else if (ltype == 1u) zs_fill(bo + w, rle, n, lane);
    else zs_move_fwd(bo + w, bo + tail + used, n, lane);
    __syncwarp();
  };
  if (nseq) {
    ZBits br;
    if (!br.init(in + sp, bend - sp)) return false;
    ZsSeq q;
    zs_seq_init(q, br, f);
    for (uint32_t done = 0; done < nseq; done += 32u) {
      const uint32_t cnt = min(32u, nseq - done);
      uint32_t mll = 0, mml = 0, moff = 0;
      for (uint32_t k = 0; k < cnt; ++k) {
        uint32_t ll, ml, off;
        zs_seq_decode(q, br, f, ws.predef, ll, ml, off);
        if ((uint32_t)lane == k) {
          mll = ll;
          mml = ml;
          moff = off;
        }
        if (done + k + 1u < nseq) br.reload();
      }
      for (uint32_t k = 0; k < cnt; ++k) {
        const uint32_t ll = __shfl_sync(kFull, mll, (int)k), ml = __shfl_sync(kFull, mml, (int)k);
        const uint32_t off = __shfl_sync(kFull, moff, (int)k);
        if (ll > lit - used || (uint64_t)w + ll + ml > bout || off > fpos0 + w + ll) return false;
        literals(ll);
        w += ll;
        used += ll;
        warp_match_copy(bo + w, off, ml, lane);
        __syncwarp();
        w += ml;
      }
    }
    f.rep[0] = q.rep0;
    f.rep[1] = q.rep1;
    f.rep[2] = q.rep2;
  }
  if (w + (lit - used) != bout) return false;
  literals(lit - used);
  produced += bout;
  return true;
}

// ---------------------------------------------------------------------------
// One chunk.  Returns a ZstdResult; on success *produced = bytes written to out[0, produced).  kCount walks the chunk
// without writing (out may be null; content checksums cannot be checked).  Every byte written lies in [0, produced).
// ---------------------------------------------------------------------------
template <bool kCount>
__device__ __forceinline__ int zstd_chunk(const uint8_t* in, uint32_t n, uint8_t* out, uint32_t cap,
                                          uint32_t* produced_out, const ZstdWarp& ws, int lane) {
  uint32_t pos = 0, produced = 0;
  *produced_out = 0;
  while (n - pos >= 5u) {
    const uint32_t magic = zs_le32(in + pos);
    if ((magic & 0xfffffff0u) == 0x184d2a50u) {          // skippable frame
      if (n - pos < 8u) return kZstdBad;
      const uint64_t sz = (uint64_t)zs_le32(in + pos + 4) + 8u;
      if (sz > n - pos) return kZstdBad;
      pos += (uint32_t)sz;
      continue;
    }
    if (magic != 0xfd2fb528u) return kZstdBad;
    // frame header
    if (n - pos < 9u) return kZstdBad;
    const uint32_t fhd = in[pos + 4];
    const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1u, checksum = (fhd >> 2) & 1u, did_flag = fhd & 3u;
    const uint32_t did_size = did_flag == 3u ? 4u : did_flag;
    const uint32_t fcs_size = fcs_flag == 0u ? single : 1u << fcs_flag;
    const uint32_t hsize = 5u + (single ^ 1u) + did_size + fcs_size;
    if (n - pos < hsize + 3u) return kZstdBad;
    if (fhd & 8u) return kZstdBad;                        // reserved bit
    uint32_t p = pos + 5u;
    if (!single) {
      if ((in[p] >> 3) + 10u > 31u) return kZstdBad;     // window over 2^31
      ++p;
    }
    uint32_t did = 0;
    for (uint32_t i = 0; i < did_size; ++i) did |= (uint32_t)in[p + i] << (8 * i);
    if (did) return kZstdBad;                            // needs a dictionary
    p += did_size;
    uint64_t fcs = ~0ull;
    if (fcs_size == 1u) fcs = in[p];
    else if (fcs_size == 2u) fcs = zs_le16(in + p) + 256u;
    else if (fcs_size == 4u) fcs = zs_le32(in + p);
    else if (fcs_size == 8u) fcs = (uint64_t)zs_le32(in + p) | ((uint64_t)zs_le32(in + p + 4) << 32);
    p += fcs_size;
    // blocks
    const uint32_t frame_start = produced;
    ZsFrame f;
    f.rep[0] = 1;
    f.rep[1] = 4;
    f.rep[2] = 8;
    f.fse_entropy = false;
    f.lit_entropy = false;
    f.huf_log = 0;
    for (int i = 0; i < 3; ++i) {
      f.tab[i] = ws.predef;
      f.log[i] = 0;
    }
    while (true) {
      if (n - p < 3u) return kZstdBad;
      const uint32_t bh = zs_le24(in + p);
      const uint32_t last = bh & 1u, type = (bh >> 1) & 3u, bsize = bh >> 3;
      if (type == 3u) return kZstdBad;
      p += 3u;
      const uint32_t csize = type == 1u ? 1u : bsize;
      if (csize > n - p) return kZstdBad;
      if (type == 0u) {
        if ((uint64_t)produced + bsize > cap) return kZstdBad;
        if (!kCount) warp_copy<true>(out + produced, in + p, bsize, lane);
        produced += bsize;
      } else if (type == 1u) {
        if ((uint64_t)produced + bsize > cap) return kZstdBad;
        if (!kCount) zs_fill(out + produced, in[p], bsize, lane);
        produced += bsize;
      } else if (!zs_compressed_block<kCount>(in, p, bsize, out, cap, produced, frame_start, f, ws, lane)) {
        return kZstdBad;
      }
      __syncwarp();
      p += csize;
      if (last) break;
    }
    if (fcs != ~0ull && (uint64_t)(produced - frame_start) != fcs) return kZstdBad;
    if (checksum) {
      if (n - p < 4u) {
        if (!kCount) return kZstdBadChecksum;
        *produced_out = produced;                        // decoding stops here, at the checksum
        return kZstdOk;
      }
      if (!kCount) {
        const uint64_t h = xxh64_warp(out + frame_start, produced - frame_start, lane);
        if ((uint32_t)h != zs_le32(in + p)) return kZstdBadChecksum;
      }
      p += 4u;
    }
    pos = p;
  }
  if (pos != n) return kZstdBad;
  *produced_out = produced;
  return kZstdOk;
}

}  // namespace detail
}  // namespace zstd
}  // namespace device
}  // namespace nvcomp
