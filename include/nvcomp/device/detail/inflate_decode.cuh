// nvcomp/device/detail/inflate_decode.cuh -- Deflate (RFC 1951) and Gzip (RFC 1952) decode of one chunk by one warp.
// The batched kernels of deflate.cu (nvcomp_b200/csrc/inflate_decode.cuh re-exports these names) and the device API
// (nvcomp/device/deflate.cuh, gzip.cuh) share it.  Everything here is a device function taking a lane, with all
// inline PTX in nvcomp/device/detail/ptx.cuh and every shared-memory access through lds_* / sts_*, so tests/emu runs
// these functions unchanged on the host.
//
// Shape (DESIGN §3.2):
//   * Header parsing is warp-uniform: every lane reads the same bits and takes the same branches.
//   * Bit reader: a 64-bit buffer refilled from aligned 32-bit loads.  A load touches only words that hold at least
//     one input byte (so it stays inside the 16-byte granules of the input, the warp_copy contract); bits past the
//     end read as zero, and a stream that consumes them is rejected as truncated.
//   * Decode tables (one per Huffman code, in the warp's shared memory): 16-bit entries, a root table indexed by the
//     next `root` stream bits plus second-level tables for the longer codes.  Leaf = symbol | length << 9 (length 0:
//     no code); link = 0x8000 | sub-table bits << 12 | offset.  Lane l fills the entries of symbols s = l (mod 32).
//   * Decode: all lanes decode the same symbols in lockstep (table lookups are broadcasts); lane k keeps token k of a
//     group of up to 32 (a literal, or a length/distance pair).  The group then executes: an exclusive scan of the
//     token lengths gives each token its output offset, the literals are stored, and the matches run in token order,
//     each by the whole warp (warp_match_copy).  Output goes straight to global memory.
//
// Table size bound.  A second-level table of 2^d entries serves a root prefix whose subtree is a full binary tree
// of depth d (every accepted code with a second level is complete), so it holds at least d + 1 symbols of its own.
// d <= 15 - root, and 2^d / (d + 1) grows with d, so the second-level entries are at most n * 2^dmax / (dmax + 1):
//   literal/length (root 10, n <= 288, dmax 5):  1024 + 288 * 32 / 6  = 2560 entries
//   distance       (root 8,  n <= 30,  dmax 7):   256 +  30 * 128 / 8 =  736 entries
//   code lengths   (root 7, lengths <= 7):         128 entries, no second level
// The builder still checks the total against the capacity and rejects the code rather than overflow.
// The out-of-line (__noinline__) functions of this header are declared inline: the header is included by every
// translation unit that uses the device API, and inline linkage lets several of them be linked into one program.
#pragma once

#include "nvcomp/device/detail/crc32.cuh"
#include "nvcomp/device/detail/lz_common.cuh"

namespace nvcomp {
namespace device {
namespace deflate {
namespace detail {

using lz::detail::kWarp;
using lz::detail::kFull;
using lz::detail::warp_copy;
using lz::detail::warp_match_copy;
using lz::detail::ldg_u32;
using lz::detail::lds_u8;
using lz::detail::lds_u16;
using lz::detail::sts_u8;
using lz::detail::sts_u16;
using crc::detail::crc0_warp;
using crc::detail::crc_finish;

enum InflateResult : int { kInflateOk = 0, kInflateBad = 1, kInflateBadChecksum = 2 };

constexpr uint32_t kInfLitRoot = 10, kInfDistRoot = 8, kInfClenRoot = 7;
constexpr uint32_t kInfLitEntries = 2560, kInfDistEntries = 736, kInfClenEntries = 128;
constexpr uint32_t kInfFixLitEntries = 1u << kInfLitRoot, kInfFixDistEntries = 1u << kInfDistRoot;
// per-warp shared memory layout (byte offsets)
constexpr uint32_t kInfLitOff = 0;                                        // dynamic literal/length table
constexpr uint32_t kInfDistOff = kInfLitOff + 2 * kInfLitEntries;         // dynamic distance table
constexpr uint32_t kInfFixLitOff = kInfDistOff + 2 * kInfDistEntries;     // fixed literal/length table
constexpr uint32_t kInfFixDistOff = kInfFixLitOff + 2 * kInfFixLitEntries;  // fixed distance table
constexpr uint32_t kInfClenOff = kInfFixDistOff + 2 * kInfFixDistEntries;   // code-length code table
constexpr uint32_t kInfRankOff = kInfClenOff + 2 * kInfClenEntries;       // u16 per symbol: rank among its length
constexpr uint32_t kInfLensOff = kInfRankOff + 2 * 320;                   // u8 per symbol: code lengths
constexpr uint32_t kInfWarpSmem = kInfLensOff + 320;                      // 10 368 bytes

// Per-warp decoder state that outlives a chunk: the warp's shared memory and whether the fixed-code tables in it are
// built (they are built on the first fixed block the warp meets, then kept).
struct InflateWarp {
  uint32_t smem;
  bool fixed_ready;
};

// ---------------------------------------------------------------------------
// Bit reader (warp-uniform: every lane holds the same state)
// ---------------------------------------------------------------------------
struct InfBits {
  const uint8_t* base;   // 4-byte aligned address at or before the first input byte
  uint32_t nwords;       // aligned words holding at least one input byte
  uint32_t wi;           // next word to load
  uint32_t skew;         // bits of word 0 in front of the first input byte
  uint32_t bits;         // valid bits in buf
  uint64_t buf;
  uint64_t limit;        // input bits

  __device__ __forceinline__ void init(const uint8_t* in, uint32_t n) {
    const uint32_t a = (uint32_t)((uintptr_t)in & 3u);
    base = in - a;
    skew = 8u * a;
    nwords = n ? (uint32_t)(((uint64_t)a + n + 3u) >> 2) : 0u;
    limit = 8ull * n;
    seek_byte(0);
  }
  __device__ __forceinline__ void refill() {
    while (bits <= 32u) {
      const uint32_t w = wi < nwords ? ldg_u32<0>(base + 4 * (size_t)wi) : 0u;
      buf |= (uint64_t)w << bits;
      bits += 32u;
      ++wi;
    }
  }
  // restart at input byte bp (after a stored block)
  __device__ __forceinline__ void seek_byte(uint64_t bp) {
    const uint64_t b = (skew >> 3) + bp;
    wi = (uint32_t)(b >> 2);
    buf = 0;
    bits = 0;
    refill();
    drop(8u * (uint32_t)(b & 3u));
  }
  __device__ __forceinline__ uint64_t consumed() const { return (uint64_t)wi * 32u - skew - bits; }
  __device__ __forceinline__ uint32_t peek() const { return (uint32_t)buf; }
  __device__ __forceinline__ void drop(uint32_t k) { buf >>= k; bits -= k; }
  __device__ __forceinline__ uint32_t get(uint32_t k) {     // k <= 16, at least k bits buffered
    const uint32_t v = (uint32_t)buf & ((1u << k) - 1u);
    drop(k);
    return v;
  }
};

// exclusive warp scan; *total = sum over the warp
__device__ __forceinline__ uint32_t inf_scan_excl(uint32_t v, uint32_t* total, int lane) {
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(kFull, inc, d);
    if (lane >= d) inc += t;
  }
  *total = __shfl_sync(kFull, inc, 31);
  return inc - v;
}

__device__ __forceinline__ uint32_t inf_brev(uint32_t code, uint32_t len) { return __brev(code) >> (32u - len); }

// ---------------------------------------------------------------------------
// Table build.  lens_a: n code lengths (u8, 0..15) in shared memory; tab_a: the table (cap entries).  A complete code
// is accepted; with `lenient` (literal/length and distance codes) also a single code of length 1 and an empty code.
// Returns false for a code the decoder rejects (over-subscribed, incomplete, or over the table bound).
// ---------------------------------------------------------------------------
inline __device__ __noinline__ bool inflate_build_table(uint32_t lens_a, uint32_t n, uint32_t tab_a, uint32_t root,
                                                        uint32_t cap, uint32_t rank_a, bool lenient, int lane) {
  const uint32_t ul = (uint32_t)lane;
  const unsigned below = (1u << ul) - 1u;
  // 1. codes per length (lane L counts length L) and each symbol's rank among the codes of its length
  uint32_t cnt = 0;
  for (uint32_t s0 = 0; s0 < n; s0 += 32u) {
    const uint32_t s = s0 + ul;
    const uint32_t L = s < n ? lds_u8(lens_a + s) : 0u;
    const uint32_t before = __shfl_sync(kFull, cnt, (int)L);
    unsigned present = __reduce_or_sync(kFull, L ? 1u << L : 0u);
    uint32_t rk = 0;
    while (present) {
      const uint32_t q = (uint32_t)__ffs((int)present) - 1u;
      present &= present - 1u;
      const unsigned m = __ballot_sync(kFull, L == q);
      if (ul == q) cnt += (uint32_t)__popc(m);
      if (L == q) rk = (uint32_t)__popc(m & below);
    }
    if (L) sts_u16(rank_a + 2u * s, before + rk);
  }
  // 2. canonical first codes from a prefix over the lengths: codes of length L start at 15-bit position S[L]
  const uint32_t w = (ul >= 1u && ul <= 15u) ? cnt << (15u - ul) : 0u;
  uint32_t total;
  const uint32_t S = inf_scan_excl(w, &total, lane);
  const uint32_t next_code = (ul >= 1u && ul <= 15u) ? S >> (15u - ul) : 0u;
  if (total > 32768u) return false;                                  // over-subscribed
  const uint32_t rsize = 1u << root;
  if (total < 32768u) {                                              // incomplete
    const uint32_t c1 = __shfl_sync(kFull, cnt, 1);
    if (!lenient || !(total == 0u || (total == 16384u && c1 == 1u))) return false;
    for (uint32_t i = ul; i < rsize; i += 32u) sts_u16(tab_a + 2u * i, 0u);
    __syncwarp();
  } else {
    // 3. second-level tables: the long codes (length > root) occupy the root prefixes from y0 on, in canonical
    // order; the deepest code under prefix P is the one that covers P's last position
    const uint32_t y0 = __shfl_sync(kFull, S, (int)(root + 1u));
    uint32_t used = rsize;
    for (uint32_t pb = y0 >> (15u - root); pb < rsize; pb += 32u) {
      const uint32_t P = pb + ul;
      const uint32_t xend = ((P + 1u) << (15u - root)) - 1u;
      uint32_t ml = root + 1u;
      for (uint32_t q = root + 2u; q <= 15u; ++q)
        if (__shfl_sync(kFull, S, (int)q) <= xend) ml = q;
      const uint32_t size = P < rsize ? 1u << (ml - root) : 0u;
      uint32_t sum;
      const uint32_t off = used + inf_scan_excl(size, &sum, lane);
      if (P < rsize && off < 4096u) sts_u16(tab_a + 2u * inf_brev(P, root), 0x8000u | ((ml - root) << 12) | off);
      used += sum;
    }
    if (used > cap) return false;
    __syncwarp();
  }
  // 4. fill: lane l writes the entries of its symbols
  for (uint32_t s0 = 0; s0 < n; s0 += 32u) {
    const uint32_t s = s0 + ul;
    const uint32_t L = s < n ? lds_u8(lens_a + s) : 0u;
    const uint32_t nc = __shfl_sync(kFull, next_code, (int)L);
    if (L) {
      const uint32_t rc = inf_brev(nc + lds_u16(rank_a + 2u * s), L);
      const uint32_t leaf = s | (L << 9);
      if (L <= root) {
        for (uint32_t i = rc; i < rsize; i += 1u << L) sts_u16(tab_a + 2u * i, leaf);
      } else {
        const uint32_t link = lds_u16(tab_a + 2u * (rc & (rsize - 1u)));
        const uint32_t off = link & 0xfffu, d = (link >> 12) & 7u;
        for (uint32_t i = rc >> root; i < (1u << d); i += 1u << (L - root)) sts_u16(tab_a + 2u * (off + i), leaf);
      }
    }
  }
  __syncwarp();
  return true;
}

// next symbol's table entry (at least 15 bits buffered); the caller drops the entry's length
__device__ __forceinline__ uint32_t inf_lookup(const InfBits& br, uint32_t tab_a, uint32_t root) {
  const uint32_t lo = br.peek();
  uint32_t e = lds_u16(tab_a + 2u * (lo & ((1u << root) - 1u)));
  if (e & 0x8000u) {
    const uint32_t d = (e >> 12) & 7u;
    e = lds_u16(tab_a + 2u * ((e & 0xfffu) + ((lo >> root) & ((1u << d) - 1u))));
  }
  return e;
}

// position of code-length code i in the header's order 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15
__device__ __forceinline__ uint32_t inf_clen_order(uint32_t i) {
  if (i < 3u) return 16u + i;
  if (i == 3u) return 0u;
  const uint32_t j = i - 4u;
  return (j & 1u) ? 7u - (j >> 1) : 8u + (j >> 1);
}

inline __device__ __noinline__ void inflate_build_fixed(uint32_t smem, int lane) {
  const uint32_t lens_a = smem + kInfLensOff;
  for (uint32_t s = (uint32_t)lane; s < 320u; s += 32u)
    sts_u8(lens_a + s, s < 144u ? 8u : s < 256u ? 9u : s < 280u ? 7u : s < 288u ? 8u : 5u);
  __syncwarp();
  inflate_build_table(lens_a, 288, smem + kInfFixLitOff, kInfLitRoot, kInfFixLitEntries, smem + kInfRankOff, false,
                      lane);
  inflate_build_table(lens_a + 288, 32, smem + kInfFixDistOff, kInfDistRoot, kInfFixDistEntries, smem + kInfRankOff,
                      false, lane);
}

// dynamic block header -> the warp's dynamic literal/length and distance tables (inlined: the bit reader stays in
// registers)
__device__ __forceinline__ bool inflate_read_dynamic(InfBits& br, const InflateWarp& ws, int lane) {
  const uint32_t lens_a = ws.smem + kInfLensOff, rank_a = ws.smem + kInfRankOff, clen_a = ws.smem + kInfClenOff;
  br.refill();
  const uint32_t hlit = br.get(5) + 257u, hdist = br.get(5) + 1u, hclen = br.get(4) + 4u;
  if (hlit > 286u || hdist > 30u) return false;
  uint32_t mine = 0;
  for (uint32_t i = 0; i < hclen; ++i) {
    br.refill();
    const uint32_t v = br.get(3);
    if ((uint32_t)lane == i) mine = v;
  }
  if (lane < 19) sts_u8(lens_a + inf_clen_order((uint32_t)lane), (uint32_t)lane < hclen ? mine : 0u);
  __syncwarp();
  if (!inflate_build_table(lens_a, 19, clen_a, kInfClenRoot, kInfClenEntries, rank_a, false, lane)) return false;
  // literal/length and distance code lengths as one sequence (a repeat may cross from one into the other)
  const uint32_t total = hlit + hdist;
  uint32_t i = 0, prev = 0;
  while (i < total) {
    br.refill();
    const uint32_t e = inf_lookup(br, clen_a, kInfClenRoot);
    const uint32_t len = (e >> 9) & 15u, sym = e & 511u;
    if (len == 0u) return false;
    br.drop(len);
    uint32_t val = 0, rep = 1;
    if (sym < 16u) {
      val = sym;
    } else if (sym == 16u) {
      if (i == 0u) return false;                                     // repeat with no previous length
      val = prev;
      rep = 3u + br.get(2);
    } else if (sym == 17u) {
      rep = 3u + br.get(3);
    } else {
      rep = 11u + br.get(7);
    }
    if (i + rep > total) return false;
    for (uint32_t j = (uint32_t)lane; j < rep; j += 32u) sts_u8(lens_a + i + j, val);
    prev = val;
    i += rep;
  }
  __syncwarp();
  if (br.consumed() > br.limit) return false;
  if (lds_u8(lens_a + 256u) == 0u) return false;                     // no end-of-block code
  if (!inflate_build_table(lens_a, hlit, ws.smem + kInfLitOff, kInfLitRoot, kInfLitEntries, rank_a, true, lane))
    return false;
  return inflate_build_table(lens_a + hlit, hdist, ws.smem + kInfDistOff, kInfDistRoot, kInfDistEntries, rank_a, true,
                             lane);
}

// one fixed or dynamic block, from its first symbol to its end-of-block code
template <bool kCount>
__device__ __forceinline__ bool inflate_huffman_block(InfBits& br, uint32_t lit_a, uint32_t dist_a, uint8_t* out,
                                                      uint32_t cap, uint32_t& produced, int lane) {
  const uint32_t ul = (uint32_t)lane;
  while (true) {
    // decode a group of up to 32 tokens; lane k keeps token k
    uint32_t tl = 0, td = 0, tb = 0, k = 0;
    bool eob = false, bad = false;
    while (k < 32u) {
      br.refill();
      const uint32_t e = inf_lookup(br, lit_a, kInfLitRoot);
      const uint32_t len = (e >> 9) & 15u, sym = e & 511u;
      if (len == 0u) { bad = true; break; }
      br.drop(len);
      if (sym < 256u) {
        if (ul == k) { tl = 1u; tb = sym; }
        ++k;
        continue;
      }
      if (sym == 256u) { eob = true; break; }
      if (sym > 285u) { bad = true; break; }                         // 286, 287: fixed code only, never valid
      const uint32_t li = sym - 257u;
      uint32_t ml;
      if (li < 8u) {
        ml = li + 3u;
      } else if (li == 28u) {
        ml = 258u;
      } else {
        const uint32_t x = (li - 4u) >> 2;
        ml = ((4u + (li & 3u)) << x) + 3u + br.get(x);
      }
      br.refill();
      const uint32_t de = inf_lookup(br, dist_a, kInfDistRoot);
      const uint32_t dlen = (de >> 9) & 15u, ds = de & 511u;
      if (dlen == 0u || ds > 29u) { bad = true; break; }             // no code, or 30 / 31 of the fixed code
      br.drop(dlen);
      uint32_t dist;
      if (ds < 4u) {
        dist = ds + 1u;
      } else {
        const uint32_t x = (ds >> 1) - 1u;
        dist = ((2u + (ds & 1u)) << x) + 1u + br.get(x);
      }
      if (ul == k) { tl = ml; td = dist; }
      ++k;
    }
    if (bad || br.consumed() > br.limit) return false;
    // execute the group
    uint32_t total;
    const uint32_t off = inf_scan_excl(tl, &total, lane);
    if ((uint64_t)produced + total > cap) return false;
    if (__any_sync(kFull, td > produced + off)) return false;        // distance beyond the output so far
    if (!kCount) {
      uint8_t* dst = out + produced;
      if (tl == 1u && td == 0u) dst[off] = (uint8_t)tb;
      __syncwarp();
      unsigned m = __ballot_sync(kFull, td != 0u);
      while (m) {
        const int j = __ffs((int)m) - 1;
        m &= m - 1u;
        const uint32_t L = __shfl_sync(kFull, tl, j), D = __shfl_sync(kFull, td, j), O = __shfl_sync(kFull, off, j);
        warp_match_copy(dst + O, D, L, lane);
        __syncwarp();
      }
    }
    produced += total;
    if (eob) return true;
  }
}

// A raw RFC 1951 stream at in[0, n): decodes until the end of the final block (later bytes are not read).
// *end_bits = bits consumed.  With kCount nothing is written and out may be null.
template <bool kCount>
__device__ __forceinline__ bool inflate_stream(const uint8_t* in, uint32_t n, uint8_t* out, uint32_t cap,
                                               uint32_t& produced, uint64_t& end_bits, InflateWarp& ws, int lane) {
  InfBits br;
  br.init(in, n);
  produced = 0;
  while (true) {
    br.refill();
    const uint32_t hdr = br.get(3);
    const uint32_t btype = hdr >> 1;
    if (btype == 0u) {
      // stored: skip to a byte boundary, LEN, NLEN, LEN bytes
      br.drop((0u - (uint32_t)br.consumed()) & 7u);
      br.refill();
      const uint32_t len = br.get(16), nlen = br.get(16);
      if ((len ^ 0xffffu) != nlen) return false;
      const uint64_t bp = br.consumed() >> 3;
      if (bp + len > n || (uint64_t)produced + len > cap) return false;
      if (!kCount) {
        warp_copy<true>(out + produced, in + bp, len, lane);
        __syncwarp();
      }
      produced += len;
      br.seek_byte(bp + len);
    } else if (btype == 1u) {
      if (!ws.fixed_ready) {
        inflate_build_fixed(ws.smem, lane);
        ws.fixed_ready = true;
      }
      if (!inflate_huffman_block<kCount>(br, ws.smem + kInfFixLitOff, ws.smem + kInfFixDistOff, out, cap, produced,
                                         lane))
        return false;
    } else if (btype == 2u) {
      if (!inflate_read_dynamic(br, ws, lane)) return false;
      if (!inflate_huffman_block<kCount>(br, ws.smem + kInfLitOff, ws.smem + kInfDistOff, out, cap, produced, lane))
        return false;
    } else {
      return false;                                                  // BTYPE 3
    }
    if (br.consumed() > br.limit) return false;                      // input ended inside the block
    if (hdr & 1u) break;                                             // BFINAL
  }
  end_bits = br.consumed();
  return true;
}

// skip a zero-terminated header field starting at pos; false when the input ends first
__device__ __forceinline__ bool inf_skip_zstring(const uint8_t* in, uint64_t n, uint64_t& pos, int lane) {
  while (pos < n) {
    const uint64_t i = pos + (uint64_t)lane;
    const unsigned m = __ballot_sync(kFull, i < n && in[i] == 0u);
    if (m) {
      pos += (uint64_t)__ffs((int)m);
      return true;
    }
    pos += 32u;
  }
  return false;
}

__device__ __forceinline__ uint32_t inf_le32(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// One chunk: a raw Deflate stream, or (kGzip) the first member of a Gzip stream.  Returns an InflateResult; on
// success *produced = bytes written to out[0, produced).  kCount walks the stream without writing (out may be null,
// and a Gzip CRC-32 cannot be checked; ISIZE is).  crc_table / crc_x2n: the CRC-32 tables (Gzip only).
template <bool kGzip, bool kCount>
__device__ __forceinline__ int inflate_chunk(const uint8_t* in, uint32_t n, uint8_t* out, uint32_t cap,
                                             uint32_t* produced, InflateWarp& ws, const uint32_t* crc_table,
                                             const uint32_t* crc_x2n, int lane) {
  uint32_t prod = 0;
  uint64_t end_bits = 0;
  *produced = 0;
  if (!kGzip) {
    if (!inflate_stream<kCount>(in, n, out, cap, prod, end_bits, ws, lane)) return kInflateBad;
    *produced = prod;
    return kInflateOk;
  }
  // RFC 1952 member header
  if (n < 10u) return kInflateBad;
  if (in[0] != 0x1fu || in[1] != 0x8bu || in[2] != 8u) return kInflateBad;
  const uint32_t flg = in[3];
  if (flg & 0xe0u) return kInflateBad;                               // reserved flag bits
  uint64_t pos = 10;
  if (flg & 4u) {                                                    // FEXTRA
    if (pos + 2u > n) return kInflateBad;
    pos += 2u + ((uint32_t)in[pos] | ((uint32_t)in[pos + 1] << 8));
    if (pos > n) return kInflateBad;
  }
  if ((flg & 8u) && !inf_skip_zstring(in, n, pos, lane)) return kInflateBad;    // FNAME
  if ((flg & 16u) && !inf_skip_zstring(in, n, pos, lane)) return kInflateBad;   // FCOMMENT
  if (flg & 2u) {                                                    // FHCRC: low 16 bits of the header's CRC-32
    if (pos + 2u > n) return kInflateBad;
    const uint32_t want = (uint32_t)in[pos] | ((uint32_t)in[pos + 1] << 8);
    const uint32_t got = crc_finish(crc_x2n, crc0_warp(crc_table, crc_x2n, in, pos, lane), pos) & 0xffffu;
    if (got != want) return kInflateBad;
    pos += 2u;
  }
  if (!inflate_stream<kCount>(in + pos, (uint32_t)(n - pos), out, cap, prod, end_bits, ws, lane)) return kInflateBad;
  // trailer: CRC-32 and ISIZE of the body, from the next byte boundary.  Checked in zlib's order: the CRC-32 as soon
  // as its 4 bytes are there, then ISIZE.
  const uint64_t tp = pos + ((end_bits + 7u) >> 3);
  if (!kCount) {
    if (tp + 4u > n) return kInflateBad;
    __syncwarp();
    const uint32_t crc = crc_finish(crc_x2n, crc0_warp(crc_table, crc_x2n, out, prod, lane), prod);
    if (crc != inf_le32(in + tp)) return kInflateBadChecksum;
  }
  if (tp + 8u > n) return kInflateBad;
  if (inf_le32(in + tp + 4) != prod) return kCount ? kInflateBad : kInflateBadChecksum;
  *produced = prod;
  return kInflateOk;
}

}  // namespace detail
}  // namespace deflate
}  // namespace device
}  // namespace nvcomp
