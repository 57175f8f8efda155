// nvcomp/device/detail/zstd_encode.cuh -- warp-per-chunk Zstandard (RFC 8878) encoder behind zstd::compress_warp
// (nvcomp/device/zstd.cuh).
//
// One warp owns one chunk (<= 64 KB) and writes one frame.  The matcher (lz77_compress.cuh) runs once over the whole
// chunk; its sequences are cut into blocks as they arrive.  A block's literals (copied from the input) and its
// sequence records share one buffer in the warp's region -- literals from the front, 6-byte records from the back --
// and the block is encoded when the parse passes its end.  No global scratch is used, and the output is a function of
// the input bytes alone, so the GPU and the host emulator write the same bytes.
//
// Stream rules:
//   * Frame: magic, Frame_Header_Descriptor with Single_Segment_Flag = 1, no Dictionary_ID, Content_Checksum_Flag =
//     0; Frame_Content_Size in 1 byte for n <= 255, else 2 bytes (n - 256).  The header is 6 or 7 bytes.
//   * Blocks: kZstdBlockBytes (16 KB) of input each, the last one shorter and flagged Last_Block; an empty chunk is one
//     empty Raw block.  Each block is Raw, RLE or Compressed, whichever is smallest; ties go Raw, then RLE.  (16 KB:
//     the literals and records of a block must fit in the region next to the hash table; libzstd level 1 loses
//     0.2-3 % of its ratio on the datagen tables when it cuts 64 KB chunks into independent 16 KB frames, and 21 % on
//     run-length int32, whose matches span blocks -- here blocks share history, so the loss is lower.)
//   * Parse: lz77_compress_chunk with the default LzParams -- greedy, deterministic hash inserts, distance <= 65 535,
//     matches >= 4 bytes, as the matcher finds them; matches may reach into earlier blocks.  A match that crosses a
//     block end is split there; a piece shorter than 4 bytes becomes literals.
//   * Repeat offsets (RFC 8878 3.1.2.5): the history starts at (1, 4, 8) per frame and is updated by every
//     Compressed block, as the decoder updates it.  A match with literals uses code 1, 2 or 3 when its offset equals
//     rep[0], rep[1] or rep[2] (checked in that order); without literals, code 1 for rep[1] and 2 for rep[2].  Every
//     other offset is coded as Offset_Value = offset + 3.
//   * Literals section: Raw, RLE (exactly one distinct byte) or Compressed, whichever is smallest (ties: Raw, RLE).
//     Header Size_Format: the smallest that fits.  Compressed: a Huffman code of at most 11 bits (package-merge, the
//     Deflate encoder's pm_lengths with the limit 11); weight w = maxBits + 1 - length, codes assigned as the
//     decoder's table expects (by weight, then symbol).  The weights are written directly (4 bits each) when the
//     highest literal is below 128, FSE-compressed (accuracy log <= 6, two interleaved states as RFC 8878 4.2.1.2)
//     when the weights take two or more distinct values and fit in 127 bytes; the smaller is used, ties direct.  One
//     stream for fewer than 256 literals, four otherwise (segments of (lit + 3) / 4).  Each stream is written from its
//     last literal back to its first and closed with a 1 bit, so it ends exactly on its final bit.  Treeless literals
//     are not used.
//   * Sequences section: Number_of_Sequences in the shortest form.  LL, OF and ML each take Predefined, RLE (one
//     distinct code) or FSE_Compressed, whichever has the lowest cost: sum over codes of count * (log - log2(p))
//     bits, with log2 taken as highbit + linear mantissa in 1/256 bit, plus 8 bits for RLE or 8 bits per header
//     byte for FSE; ties Predefined, then RLE.  Repeat_Mode is not used.  FSE counts: accuracy log libzstd's
//     FSE_optimalTableLog(max, nseq, max code) with max 9 (LL, ML) or 8 (OF); each used code gets
//     max(1, count * 2^log / nseq), and the difference to 2^log goes to the most frequent code (lowest code on
//     ties) or, when negative, is taken from the largest counts down to 1.  The counts are written as RFC 8878 4.1.1
//     (libzstd's FSE_writeNCount).  The bitstream follows the RFC's order; each state starts on the first cell (in
//     table order) of the last sequence's code, and the stream ends with a 1 bit, exactly on its final bit.
//   * Bound: the all-Raw frame, header + n + 3 bytes per block, which is within ZSTD_compressBound(n) for n <= 64 KB.
// The FSE tables are built by the decoder's own builder (zs_build_fse, and zstd_build_predefined for the predefined
// ones); an encoder state table is read off the decode table, so both sides agree on every cell.
#pragma once

#include "nvcomp/device/detail/deflate_compress.cuh"
#include "nvcomp/device/detail/zstd_decode.cuh"

namespace nvcomp {
namespace device {
namespace zstd {
namespace detail {

using lz::detail::lz77_compress_chunk;
using lz::detail::smem_addr;
using deflate::detail::pm_lengths;
using deflate::detail::DeflateBits;

constexpr uint32_t kZstdBlockBytes = 16384;
constexpr uint32_t kZstdMaxCompressChunk = 65536;
constexpr uint32_t kZeHufLimit = 11;

// Per-warp region (byte offsets).  ws is the package-merge workspace while the Huffman code is built, then the FSE
// state tables, one decode table and the decoder's table-builder scratch.
constexpr uint32_t kZeHashOff = 0;                                   // u16[4096] matcher hash table
constexpr uint32_t kZeBufOff = 2u << lz::detail::kHashLog;           // literals up, records (3 x u16) down
constexpr uint32_t kZeBufBytes = kZstdBlockBytes + kZstdBlockBytes / 2;   // lit + 4 * nseq <= block: fits
constexpr uint32_t kZeWsOff = kZeBufOff + kZeBufBytes;
constexpr uint32_t kZeStOff = 0;                                     // u16 state tables: LL [512], OF [256], ML [512]
constexpr uint32_t kZeTmpOff = 2560;                                 // u32[512] decode table being read off
constexpr uint32_t kZeScrOff = 4608;                                 // zs_build_fse scratch (sym, seq, next)
constexpr uint32_t kZeWsBytes = 7680;                                // >= package-merge's 7 656 at limit 11
constexpr uint32_t kZePreOff = kZeWsOff + kZeWsBytes;                // the decoder's predefined tables
constexpr uint32_t kZeHistOff = kZePreOff + kZsPreSmem;              // u32[256] literal histogram
constexpr uint32_t kZeCodeOff = kZeHistOff + 1024;                   // u32[256] code | length << 16
constexpr uint32_t kZeSlotOff = kZeCodeOff + 1024;                   // LL, OF, ML: hist, cnt, cum (u32[64]), norm
constexpr uint32_t kZeSlotBytes = 3 * 256 + 128;
constexpr uint32_t kZeTreeOff = kZeSlotOff + 3 * kZeSlotBytes;       // u8[128] Huffman tree description
constexpr uint32_t kZeWeightOff = kZeTreeOff + 128;                  // u8[256] Huffman weights
constexpr uint32_t kZeStageOff = kZeWeightOff + 256;                 // DeflateBits staging window
constexpr uint32_t kZstdEncWarpSmem = (kZeStageOff + 4u * 68u + 15u) & ~15u;

static_assert(kZeScrOff + 1536 <= kZeWsBytes && kZeScrOff >= kZsSymOff - kZsNormOff,
              "table-builder scratch fits in the workspace");
static_assert(2 * deflate::detail::kDeflateLitSyms + 2 * 572 + kZeHufLimit * deflate::detail::kPmFlagWords <=
                  kZeWsBytes / 4, "package-merge workspace fits");
static_assert(kZstdEncWarpSmem <= 49152, "four compressing warps fit on an SM");

__host__ __device__ constexpr uint32_t zstd_enc_bound(uint32_t n) {
  return (n <= 255u ? 6u : 7u) + n + 3u * (n == 0u ? 1u : (n + kZstdBlockBytes - 1u) / kZstdBlockBytes);
}

// Bit writer of one lane: LSB first, bytes past `lim` dropped (over = true), p == nullptr counts only.
struct ZsBitOut {
  uint8_t* p;
  uint32_t pos, lim;
  uint64_t acc;
  uint32_t nb;
  bool over;
  __device__ __forceinline__ void byte(uint32_t b) {
    if (pos < lim) { if (p) p[pos] = (uint8_t)b; }
    else over = true;
    ++pos;
  }
  __device__ __forceinline__ void add(uint32_t v, uint32_t n) {   // v < 2^n, n <= 32
    acc |= (uint64_t)v << nb;
    nb += n;
    while (nb >= 8u) { byte((uint32_t)acc & 255u); acc >>= 8; nb -= 8u; }
  }
  __device__ __forceinline__ void close() {
    add(1u, 1u);
    if (nb) byte((uint32_t)acc);
    acc = 0;
    nb = 0;
  }
};

// 1/256-bit cost of a symbol of probability c / 2^log
__device__ __forceinline__ uint32_t ze_cost(uint32_t c, uint32_t log) {
  const uint32_t hb = zs_highbit(c);
  return (log << 8) - ((hb << 8) + (((c << 8) >> hb) - 256u));
}

// libzstd FSE_optimalTableLog
__device__ __forceinline__ uint32_t ze_table_log(uint32_t max_log, uint32_t n, uint32_t max_sym) {
  const uint32_t src_bits = n > 1u ? zs_highbit(n - 1u) : 0u;
  uint32_t log = max_log;
  if (src_bits >= 2u && src_bits - 2u < log) log = src_bits - 2u;
  if (src_bits < 2u) log = 5u;
  const uint32_t min_bits = min(zs_highbit(max(n, 1u)) + 1u, zs_highbit(max(max_sym, 1u)) + 2u);
  if (log < min_bits) log = min_bits;
  return min(max(log, 5u), max_log);
}

// Normalized counts (lane 0; rules in the file header) of hist[0, max_sym] summing to total
__device__ __forceinline__ void ze_normalize(const uint32_t* hist, uint32_t max_sym, uint32_t total, uint32_t log,
                                             int16_t* norm) {
  const uint32_t size = 1u << log;
  int sum = 0;
  uint32_t big = 0;
  for (uint32_t s = 0; s <= max_sym; ++s) {
    const uint32_t h = hist[s];
    const int v = h ? max(1, (int)(((uint64_t)h << log) / total)) : 0;
    norm[s] = (int16_t)v;
    sum += v;
    if (h > hist[big]) big = s;
  }
  int diff = (int)size - sum;
  if (diff > 0) norm[big] = (int16_t)(norm[big] + diff);
  while (diff < 0) {
    uint32_t m = 0;
    for (uint32_t s = 1; s <= max_sym; ++s)
      if (norm[s] > norm[m]) m = s;
    const int take = min(-diff, norm[m] - 1);
    norm[m] = (int16_t)(norm[m] - take);
    diff += take;
  }
}

// RFC 8878 4.1.1 table description of norm[0, max_sym] (libzstd FSE_writeNCount), lane 0
__device__ __forceinline__ void ze_write_ncount(ZsBitOut& bo, const int16_t* norm, uint32_t max_sym, uint32_t log) {
  bo.add(log - 5u, 4u);
  int remaining = (1 << log) + 1;
  int threshold = 1 << log;
  uint32_t nbits = log + 1u;
  uint32_t s = 0;
  bool prev0 = false;
  while (s <= max_sym && remaining > 1) {
    if (prev0) {
      uint32_t start = s;
      while (norm[s] == 0) ++s;
      while (s >= start + 3u) { bo.add(3u, 2u); start += 3u; }
      bo.add(s - start, 2u);
    }
    int count = norm[s++];
    const int mx = (2 * threshold - 1) - remaining;
    remaining -= count < 0 ? -count : count;
    ++count;
    if (count >= threshold) count += mx;
    bo.add((uint32_t)count, nbits - (count < mx ? 1u : 0u));
    prev0 = count == 1;
    while (remaining < threshold) { --nbits; threshold >>= 1; }
  }
  if (bo.nb) bo.byte((uint32_t)bo.acc);
  bo.acc = 0;
  bo.nb = 0;
}

// Encoder view of the FSE decode table at tab_a (2^log cells, symbols <= max_sym): cnt[s] cells per symbol, cum[s]
// their first index in st, st[cum[s] + r] = the cell whose state is cnt[s] + r.
__device__ __forceinline__ void ze_enc_table(uint32_t tab_a, uint32_t log, uint32_t max_sym, uint32_t* cnt,
                                             uint32_t* cum, uint16_t* st, int lane) {
  const uint32_t size = 1u << log;
  for (uint32_t s = lane; s <= max_sym; s += kWarp) cnt[s] = 0;
  __syncwarp();
  for (uint32_t u = lane; u < size; u += kWarp) atomicAdd(&cnt[lds_u32(tab_a + 4u * u) >> 24], 1u);
  __syncwarp();
  if (lane == 0) {
    uint32_t c = 0;
    for (uint32_t s = 0; s <= max_sym; ++s) { cum[s] = c; c += cnt[s]; }
  }
  __syncwarp();
  for (uint32_t u = lane; u < size; u += kWarp) {
    const uint32_t e = lds_u32(tab_a + 4u * u), s = e >> 24, nb = (e >> 16) & 0xffu;
    const uint32_t ns = ((e & 0xffffu) + size) >> nb;
    st[cum[s] + ns - cnt[s]] = (uint16_t)u;
  }
  __syncwarp();
}

struct ZeFse {   // one FSE encoder state
  const uint32_t* cnt;
  const uint32_t* cum;
  const uint16_t* st;
  uint32_t log, x;
  __device__ __forceinline__ void init(uint32_t s) { x = (1u << log) + st[cum[s]]; }
  __device__ __forceinline__ void enc(ZsBitOut& bo, uint32_t s) {
    const uint32_t c = cnt[s], k = log - zs_highbit(c);
    const uint32_t nb = k - ((x >> k) < c ? 1u : 0u);
    bo.add(x & ((1u << nb) - 1u), nb);
    x = (1u << log) + st[cum[s] + (x >> nb) - c];
  }
  __device__ __forceinline__ void flush(ZsBitOut& bo) { bo.add(x - (1u << log), log); }
};

// code of a literal length / match length: the last code whose baseline (the decoder's info table) is <= v
__device__ __forceinline__ uint32_t ze_code(uint32_t info_a, uint32_t ncodes, uint32_t v) {
  uint32_t lo = 0, hi = ncodes - 1u;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1u) >> 1;
    if ((lds_u32(info_a + 4u * mid) & 0xffffffu) <= v) lo = mid; else hi = mid - 1u;
  }
  return lo;
}

struct ZstdEncWarp {
  uint8_t* base;
  uint32_t sa;    // shared address of base
  __device__ __forceinline__ uint16_t* table() const { return (uint16_t*)(base + kZeHashOff); }
  __device__ __forceinline__ uint8_t* buf() const { return base + kZeBufOff; }
  __device__ __forceinline__ uint8_t* ws() const { return base + kZeWsOff; }
  __device__ __forceinline__ uint32_t pre() const { return sa + kZePreOff; }
  // zs_build_fse / zstd_build_predefined address their scratch from a decoder region base: this one puts sym, seq
  // and next at ws + kZeScrOff (and the predefined builder's norm 768 bytes below).
  __device__ __forceinline__ uint32_t fake_base() const { return sa + kZeWsOff + kZeScrOff - kZsSymOff; }
  __device__ __forceinline__ uint32_t* hist() const { return (uint32_t*)(base + kZeHistOff); }
  __device__ __forceinline__ uint32_t* code() const { return (uint32_t*)(base + kZeCodeOff); }
  __device__ __forceinline__ uint32_t* slot(int t) const { return (uint32_t*)(base + kZeSlotOff + t * kZeSlotBytes); }
  __device__ __forceinline__ int16_t* norm(int t) const { return (int16_t*)(slot(t) + 192); }
  __device__ __forceinline__ uint16_t* st(int t) const {
    return (uint16_t*)(ws() + kZeStOff + (t == kZsLL ? 0u : t == kZsOF ? 1024u : 1536u));
  }
  __device__ __forceinline__ uint8_t* tree() const { return base + kZeTreeOff; }
  __device__ __forceinline__ uint8_t* weight() const { return base + kZeWeightOff; }
  __device__ __forceinline__ uint32_t* stage() const { return (uint32_t*)(base + kZeStageOff); }
};

// Huffman tree description of weight()[0, nw) FSE-compressed into tree()[1, ...) (lane 0).  Returns its size
// (without the header byte), or 0 when this form is not possible.
__device__ __forceinline__ uint32_t ze_fse_weights(const ZstdEncWarp& w, uint32_t nw, int lane) {
  uint32_t* h = w.slot(kZsLL);
  uint32_t* cnt = h + 64;
  uint32_t* cum = h + 128;
  int16_t* norm = w.norm(kZsLL);
  const uint8_t* wt = w.weight();
  uint32_t max_w = 0, distinct = 0, log = 0;
  if (lane == 0) {
    for (int s = 0; s < 16; ++s) h[s] = 0;
    for (uint32_t i = 0; i < nw; ++i) h[wt[i]]++;
    for (uint32_t s = 0; s < 16; ++s)
      if (h[s]) { max_w = s; ++distinct; }
    if (distinct >= 2u && nw >= 2u) {
      log = ze_table_log(6u, nw, max_w);
      ze_normalize(h, max_w, nw, log, norm);
    }
  }
  log = __shfl_sync(kFull, log, 0);
  max_w = __shfl_sync(kFull, max_w, 0);
  __syncwarp();
  if (log == 0u) return 0;
  const uint32_t tmp_a = w.sa + kZeWsOff + kZeTmpOff;
  zs_build_fse(smem_addr(norm), max_w, log, tmp_a, w.fake_base(), lane);
  ze_enc_table(tmp_a, log, max_w, cnt, cum, w.st(kZsLL), lane);
  uint32_t size = 0;
  if (lane == 0) {
    ZsBitOut bo{w.tree() + 1, 0u, 127u, 0ull, 0u, false};
    ze_write_ncount(bo, norm, max_w, log);
    ZeFse s1{cnt, cum, w.st(kZsLL), log, 0u}, s2 = s1;
    uint32_t i;
    if (nw & 1u) {
      s1.init(wt[nw - 1u]);
      s2.init(wt[nw - 2u]);
      if (nw >= 3u) s1.enc(bo, wt[nw - 3u]);
      i = nw >= 3u ? nw - 3u : 0u;
    } else {
      s2.init(wt[nw - 1u]);
      s1.init(wt[nw - 2u]);
      i = nw - 2u;
    }
    while (i > 0u) {
      s2.enc(bo, wt[--i]);
      s1.enc(bo, wt[--i]);
    }
    s2.flush(bo);
    s1.flush(bo);
    bo.close();
    size = bo.over ? 0u : bo.pos;
  }
  size = __shfl_sync(kFull, size, 0);
  __syncwarp();
  return size;
}

// The parse's emitter and the block encoder
struct ZstdEnc {
  const uint8_t* in;
  uint8_t* out;
  ZstdEncWarp w;
  uint32_t n;
  uint32_t o;         // frame bytes written
  uint32_t bstart;    // input offset of the open block
  uint32_t bend;
  uint32_t pos;       // input bytes taken into the open block
  uint32_t nlit, nseq, lit_mark;
  uint32_t rep[3];

  __device__ __forceinline__ uint16_t* rec(uint32_t k) const {
    return (uint16_t*)(w.buf() + kZeBufBytes) - 3u * (k + 1u);
  }
  __device__ __forceinline__ void take_literals(const uint8_t* p, uint32_t k, int lane) {
    uint8_t* b = w.buf() + nlit;
    uint32_t* h = w.hist();
    for (uint32_t i = lane; i < k; i += kWarp) {
      const uint32_t c = p[i];
      b[i] = (uint8_t)c;
      atomicAdd(&h[c], 1u);
    }
    nlit += k;
  }
  __device__ __forceinline__ void next_block(int lane) {
    if (pos == bend && pos < n) encode_block(false, lane);
  }
  __device__ __forceinline__ void literals(const uint8_t* p, uint32_t ll, int lane) {
    while (ll) {
      const uint32_t k = min(ll, bend - pos);
      take_literals(p, k, lane);
      p += k;
      pos += k;
      ll -= k;
      next_block(lane);
    }
  }
  __device__ __forceinline__ void sequence(const uint8_t* lit, uint32_t ll, uint32_t off, uint32_t ml, int lane) {
    literals(lit, ll, lane);
    while (ml) {
      const uint32_t k = min(ml, bend - pos);
      if (k >= 4u) {
        if (lane == 0) {
          uint16_t* r = rec(nseq);
          r[0] = (uint16_t)(nlit - lit_mark);
          r[1] = (uint16_t)k;
          r[2] = (uint16_t)off;
        }
        ++nseq;
        lit_mark = nlit;
      } else {
        take_literals(in + pos, k, lane);
      }
      pos += k;
      ml -= k;
      next_block(lane);
    }
  }
  __device__ __forceinline__ void finish(const uint8_t* lit, uint32_t ll, int lane) {
    literals(lit, ll, lane);
    encode_block(true, lane);
  }

  __device__ __forceinline__ void put_bytes(uint32_t at, uint32_t v, uint32_t nbytes, int lane) {
    if ((uint32_t)lane < nbytes) out[at + lane] = (uint8_t)(v >> (8 * lane));
  }

  __device__ void encode_block(bool last, int lane);
  __device__ uint32_t compressed_block(const uint8_t* b, uint32_t blen, uint8_t* dst, uint32_t* nrep, int lane);
  __device__ uint32_t literals_section(uint8_t* dst, uint32_t lim, int lane);
  __device__ uint32_t sequences_section(uint8_t* dst, uint32_t lim, uint32_t* nrep, int lane);
};

__device__ __forceinline__ void ZstdEnc::encode_block(bool last, int lane) {
  __syncwarp();
  const uint32_t blen = pos - bstart;
  const uint8_t* b = in + bstart;
  bool diff = false;
  for (uint32_t i = lane; i < blen; i += kWarp) diff |= b[i] != b[0];
  const bool same = blen >= 2u && !__any_sync(kFull, diff);
  uint32_t nrep[3] = {rep[0], rep[1], rep[2]};
  const uint32_t lastb = last ? 1u : 0u;
  if (same) {
    put_bytes(o, lastb | (1u << 1) | (blen << 3) | ((uint32_t)b[0] << 24), 4u, lane);
    o += 4u;
  } else {
    const uint32_t c = blen ? compressed_block(b, blen, out + o + 3u, nrep, lane) : 0u;
    if (c) {
      put_bytes(o, lastb | (2u << 1) | (c << 3), 3u, lane);
      o += 3u + c;
      rep[0] = nrep[0];
      rep[1] = nrep[1];
      rep[2] = nrep[2];
    } else {
      put_bytes(o, lastb | (blen << 3), 3u, lane);
      warp_copy<true>(out + o + 3u, b, blen, lane);
      o += 3u + blen;
    }
  }
  uint32_t* h = w.hist();
  for (int i = lane; i < 256; i += kWarp) h[i] = 0;
  bstart = pos;
  bend = min(pos + kZstdBlockBytes, n);
  nlit = nseq = lit_mark = 0;
  __syncwarp();
}

// Compressed form of the open block into dst; its size, or 0 when it is not smaller than blen
__device__ __forceinline__ uint32_t ZstdEnc::compressed_block(const uint8_t* b, uint32_t blen, uint8_t* dst,
                                                                  uint32_t* nrep, int lane) {
  const uint32_t ls = literals_section(dst, blen, lane);
  if (ls == 0u || ls + 1u >= blen) return 0;
  const uint32_t ss = sequences_section(dst + ls, blen - ls - 1u, nrep, lane);   // ls + ss < blen
  __syncwarp();
  return ss == 0u ? 0u : ls + ss;
}

// The literals section (rules in the file header) written to dst; its size, or 0 when it would not leave a byte
// of dst[0, lim) for the sequences.
__device__ __forceinline__ uint32_t ZstdEnc::literals_section(uint8_t* dst, uint32_t lim, int lane) {
  const uint32_t L = nlit;
  const uint8_t* lits = w.buf();
  uint32_t* h = w.hist();
  uint32_t* code = w.code();
  uint32_t nd = 0, maxsym = 0;
  for (int s = lane; s < 256; s += kWarp)
    if (h[s]) { ++nd; maxsym = (uint32_t)s; }
  nd = __reduce_add_sync(kFull, nd);
  maxsym = __reduce_max_sync(kFull, maxsym);
  const uint32_t lh_raw = L <= 31u ? 1u : L <= 4095u ? 2u : 3u;
  uint32_t best = lh_raw + L, mode = 0;       // 0 raw, 1 rle, 2 huffman
  if (nd == 1u && lh_raw + 1u < best) { best = lh_raw + 1u; mode = 1; }
  uint32_t tree_sz = 0, lh = 0, csz = 0, sbytes[4] = {0, 0, 0, 0};
  const bool single = L < 256u;
  bool direct = false;
  if (nd >= 2u) {
    pm_lengths(h, 256, (int)kZeHufLimit, code, (uint32_t*)w.ws(), lane);
    uint32_t mb = 0;
    for (int s = lane; s < 256; s += kWarp) mb = max(mb, code[s] >> 16);
    mb = __reduce_max_sync(kFull, mb);
    uint8_t* wt = w.weight();
    for (uint32_t s = lane; s <= maxsym; s += kWarp) {
      const uint32_t l = code[s] >> 16;
      wt[s] = (uint8_t)(l ? mb + 1u - l : 0u);
    }
    __syncwarp();
    if (lane == 0) {   // canonical codes in the decoder's table order: by weight, then symbol
      uint32_t start[16];
      for (int k = 0; k < 16; ++k) start[k] = 0;
      for (uint32_t s = 0; s <= maxsym; ++s)
        if (wt[s]) start[wt[s]] += 1u << (wt[s] - 1u);
      uint32_t acc = 0;
      for (uint32_t k = 1; k <= mb; ++k) { const uint32_t c = start[k]; start[k] = acc; acc += c; }
      for (uint32_t s = 0; s <= maxsym; ++s) {
        const uint32_t k = wt[s];
        if (k) {
          code[s] = (start[k] >> (k - 1u)) | ((mb + 1u - k) << 16);
          start[k] += 1u << (k - 1u);
        }
      }
    }
    __syncwarp();
    const uint32_t fse_sz = ze_fse_weights(w, maxsym, lane);
    const uint32_t direct_sz = maxsym < 128u ? (maxsym + 1u) / 2u : 0u;
    direct = direct_sz != 0u && (fse_sz == 0u || direct_sz <= fse_sz);
    tree_sz = 1u + (direct ? direct_sz : fse_sz);
    if (direct_sz != 0u || fse_sz != 0u) {
      // stream sizes: code bits per segment, plus the closing bit
      const uint32_t seg = (L + 3u) / 4u;
      uint32_t bits[4] = {0, 0, 0, 0};
      for (uint32_t i = lane; i < L; i += kWarp) {
        const uint32_t l = code[lits[i]] >> 16;
        const uint32_t k = single ? 0u : i / seg;
#pragma unroll
        for (uint32_t j = 0; j < 4; ++j) bits[j] += j == k ? l : 0u;
      }
      uint32_t streams = 0;
#pragma unroll
      for (uint32_t j = 0; j < 4; ++j) {
        sbytes[j] = (__reduce_add_sync(kFull, bits[j]) + 8u) >> 3;
        if (j == 0 || !single) streams += sbytes[j];
      }
      csz = tree_sz + (single ? 0u : 6u) + streams;
      lh = (single || max(L, csz) <= 1023u) ? 3u : max(L, csz) <= 16383u ? 4u : 5u;
      if (lh + csz < best) { best = lh + csz; mode = 2; }
    }
  }
  if (best + 1u >= lim) return 0;
  if (mode == 0u) {
    const uint32_t hv = lh_raw == 1u ? L << 3 : lh_raw == 2u ? (1u << 2) | (L << 4) : (3u << 2) | (L << 4);
    if ((uint32_t)lane < lh_raw) dst[lane] = (uint8_t)(hv >> (8 * lane));
    for (uint32_t i = lane; i < L; i += kWarp) dst[lh_raw + i] = lits[i];
  } else if (mode == 1u) {
    const uint32_t hv = 1u | (lh_raw == 1u ? L << 3 : lh_raw == 2u ? (1u << 2) | (L << 4) : (3u << 2) | (L << 4));
    if ((uint32_t)lane < lh_raw) dst[lane] = (uint8_t)(hv >> (8 * lane));
    if (lane == 0) dst[lh_raw] = lits[0];
  } else {
    const uint32_t sf = single ? 0u : lh == 3u ? 1u : lh == 4u ? 2u : 3u;
    const uint32_t fb = lh == 3u ? 10u : lh == 4u ? 14u : 18u;
    const uint64_t hv = 2ull | ((uint64_t)sf << 2) | ((uint64_t)L << 4) | ((uint64_t)csz << (4u + fb));
    if ((uint32_t)lane < lh) dst[lane] = (uint8_t)(hv >> (8 * lane));
    uint8_t* t = dst + lh;
    if (direct) {
      const uint8_t* wt = w.weight();
      if (lane == 0) t[0] = (uint8_t)(127u + maxsym);
      for (uint32_t i = lane; i < tree_sz - 1u; i += kWarp) {
        const uint32_t a = wt[2u * i], c = 2u * i + 1u < maxsym ? wt[2u * i + 1u] : 0u;
        t[1u + i] = (uint8_t)((a << 4) | c);
      }
    } else {
      // ze_fse_weights left the FSE form in tree()[1, tree_sz)
      if (lane == 0) t[0] = (uint8_t)(tree_sz - 1u);
      for (uint32_t i = 1u + lane; i < tree_sz; i += kWarp) t[i] = w.tree()[i];
    }
    uint8_t* s = t + tree_sz;
    if (!single) {
      if (lane < 6) s[lane] = (uint8_t)(sbytes[lane >> 1] >> (8 * (lane & 1)));
      s += 6;
    }
    const uint32_t seg = single ? L : (L + 3u) / 4u;
    const uint32_t nstreams = single ? 1u : 4u;
    for (uint32_t k = 0; k < nstreams; ++k) {
      const uint32_t lo = k * seg, hi = k + 1u == nstreams ? L : lo + seg;
      __syncwarp();
      DeflateBits bo{w.stage(), code, s, 0u, 0u};
      bo.clear(lane);
      for (uint32_t base = 0; base < hi - lo; base += kWarp) {
        const uint32_t j = base + (uint32_t)lane;
        const uint32_t c = j < hi - lo ? code[lits[hi - 1u - j]] : 0u;
        bo.put_lanes(c & 0xffffu, c >> 16, lane);
      }
      bo.put(1u, 1u, lane);
      bo.close(lane);
      s += sbytes[k];
    }
  }
  __syncwarp();
  return best;
}

// The sequences section written to dst (at most lim bytes); its size, or 0 when it does not fit.  nrep: the repeat
// offsets after the block.
__device__ __forceinline__ uint32_t ZstdEnc::sequences_section(uint8_t* dst, uint32_t lim, uint32_t* nrep,
                                                                   int lane) {
  if (nseq == 0u) {
    if (lane == 0) dst[0] = 0;
    __syncwarp();
    return 1;
  }
  const uint32_t pre = w.pre();
  // offset values with the repeat history (lane 0, in order), stored back into the records: the low 16 bits in
  // place of the offset, bit 16 in bit 15 of the literal length
  if (lane == 0) {
    for (uint32_t k = 0; k < nseq; ++k) {
      uint16_t* r = rec(k);
      const uint32_t ll = r[0], off = r[2];
      uint32_t ov;
      if (ll != 0u && off == nrep[0]) ov = 1;
      else if (off == nrep[1]) ov = ll ? 2u : 1u;
      else if (off == nrep[2]) ov = ll ? 3u : 2u;
      else ov = off + 3u;
      // the decoder's update, by the repeat slot the code names (not by value: two slots may hold the offset)
      const uint32_t slot = ov > 3u ? 3u : ov - 1u + (ll == 0u ? 1u : 0u);
      if (slot >= 2u) nrep[2] = nrep[1];
      if (slot >= 1u) { nrep[1] = nrep[0]; nrep[0] = off; }
      r[0] = (uint16_t)(ll | ((ov >> 16) << 15));
      r[2] = (uint16_t)ov;
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) nrep[i] = __shfl_sync(kFull, nrep[i], 0);
  // code histograms
  for (int t = 0; t < 3; ++t)
    for (int s = lane; s < 64; s += kWarp) w.slot(t)[s] = 0;
  __syncwarp();
  for (uint32_t k = lane; k < nseq; k += kWarp) {
    const uint16_t* r = rec(k);
    const uint32_t ov = r[2] | ((uint32_t)(r[0] >> 15) << 16);
    atomicAdd(&w.slot(kZsLL)[ze_code(pre + kZsLLInfoOff, 36u, r[0] & 0x7fffu)], 1u);
    atomicAdd(&w.slot(kZsOF)[zs_highbit(ov)], 1u);
    atomicAdd(&w.slot(kZsML)[ze_code(pre + kZsMLInfoOff, 53u, r[1])], 1u);
  }
  __syncwarp();
  // modes
  uint32_t modes[3], logs[3], maxs[3];
  const uint32_t tmp_a = w.sa + kZeWsOff + kZeTmpOff;
  for (int t = 0; t < 3; ++t) {
    uint32_t* h = w.slot(t);
    uint32_t* cnt = h + 64;
    uint32_t* cum = h + 128;
    const uint32_t plog = t == kZsOF ? 5u : 6u;
    const uint32_t pmax = t == kZsLL ? 35u : t == kZsOF ? 28u : 52u;
    const uint32_t ptab = pre + (t == kZsLL ? kZsPreLLOff : t == kZsOF ? kZsPreOFOff : kZsPreMLOff);
    ze_enc_table(ptab, plog, pmax, cnt, cum, w.st(t), lane);
    uint32_t nd = 0, mx = 0, pcost = 0;
    for (uint32_t s = lane; s < 64; s += kWarp)
      if (h[s]) {
        ++nd;
        mx = s;
        pcost += h[s] * ze_cost(cnt[s], plog);
      }
    nd = __reduce_add_sync(kFull, nd);
    mx = __reduce_max_sync(kFull, mx);
    pcost = __reduce_add_sync(kFull, pcost);
    const uint32_t log = ze_table_log(t == kZsOF ? 8u : 9u, nseq, mx);
    int16_t* norm = w.norm(t);
    uint32_t hdr = 0;
    if (lane == 0) {
      ze_normalize(h, mx, nseq, log, norm);
      ZsBitOut bo{nullptr, 0u, 0u, 0ull, 0u, false};
      ze_write_ncount(bo, norm, mx, log);
      hdr = bo.pos;
    }
    hdr = __shfl_sync(kFull, hdr, 0);
    __syncwarp();
    uint32_t fcost = 0;
    for (uint32_t s = lane; s <= mx; s += kWarp)
      if (h[s]) fcost += h[s] * ze_cost((uint32_t)norm[s], log);
    fcost = __reduce_add_sync(kFull, fcost) + (hdr << 11);
    uint32_t m = 0, best = pcost;
    if (nd == 1u && (8u << 8) < best) { m = 1; best = 8u << 8; }
    if (fcost < best) m = 2;
    modes[t] = m;
    maxs[t] = mx;
    logs[t] = m == 0u ? plog : m == 1u ? 0u : log;
    if (m == 2u) {
      zs_build_fse(smem_addr(norm), mx, log, tmp_a, w.fake_base(), lane);
      ze_enc_table(tmp_a, log, mx, cnt, cum, w.st(t), lane);
    }
  }
  // header, table descriptions, bitstream (lane 0)
  uint32_t size = 0;
  if (lane == 0) {
    ZsBitOut bo{dst, 0u, lim, 0ull, 0u, false};
    if (nseq < 128u) bo.byte(nseq);
    else { bo.byte((nseq >> 8) + 128u); bo.byte(nseq & 255u); }
    bo.byte((modes[0] << 6) | (modes[1] << 4) | (modes[2] << 2));
    for (int t = 0; t < 3; ++t) {
      if (modes[t] == 1u) bo.byte(maxs[t]);
      else if (modes[t] == 2u) ze_write_ncount(bo, w.norm(t), maxs[t], logs[t]);
    }
    ZeFse f[3];
    for (int t = 0; t < 3; ++t) f[t] = ZeFse{w.slot(t) + 64, w.slot(t) + 128, w.st(t), logs[t], 0u};
    for (uint32_t k = nseq; k-- > 0;) {
      const uint16_t* r = rec(k);
      const uint32_t ll = r[0] & 0x7fffu, ml = r[1];
      const uint32_t ov = r[2] | ((uint32_t)(r[0] >> 15) << 16);
      const uint32_t llc = ze_code(pre + kZsLLInfoOff, 36u, ll), mlc = ze_code(pre + kZsMLInfoOff, 53u, ml);
      const uint32_t ofc = zs_highbit(ov);
      const uint32_t lli = lds_u32(pre + kZsLLInfoOff + 4u * llc), mli = lds_u32(pre + kZsMLInfoOff + 4u * mlc);
      if (k + 1u == nseq) {
        if (modes[kZsLL] != 1u) f[kZsLL].init(llc);
        if (modes[kZsOF] != 1u) f[kZsOF].init(ofc);
        if (modes[kZsML] != 1u) f[kZsML].init(mlc);
      } else {
        if (modes[kZsOF] != 1u) f[kZsOF].enc(bo, ofc);
        if (modes[kZsML] != 1u) f[kZsML].enc(bo, mlc);
        if (modes[kZsLL] != 1u) f[kZsLL].enc(bo, llc);
      }
      bo.add(ll - (lli & 0xffffffu), lli >> 24);
      bo.add(ml - (mli & 0xffffffu), mli >> 24);
      bo.add(ov - (1u << ofc), ofc);
      if (bo.over) break;
    }
    if (modes[kZsML] != 1u) f[kZsML].flush(bo);
    if (modes[kZsOF] != 1u) f[kZsOF].flush(bo);
    if (modes[kZsLL] != 1u) f[kZsLL].flush(bo);
    bo.close();
    size = bo.over ? 0u : bo.pos;
  }
  size = __shfl_sync(kFull, size, 0);
  __syncwarp();
  return size;
}

// Compress one chunk of n <= 64 KB bytes into out (zstd_enc_bound(n) bytes) with the warp's region at smem
// (kZstdEncWarpSmem bytes); returns the frame's length.
__device__ __forceinline__ uint32_t zstd_compress_chunk(const uint8_t* __restrict__ in, uint32_t n,
                                                        uint8_t* __restrict__ out, uint8_t* smem, int lane) {
  ZstdEnc e;
  e.in = in;
  e.out = out;
  e.w = ZstdEncWarp{smem, smem_addr(smem)};
  e.n = n;
  const uint32_t hl = n <= 255u ? 6u : 7u;
  const uint64_t hv = 0xFD2FB528ull | ((uint64_t)(n <= 255u ? 0x20u : 0x60u) << 32) |
                      ((uint64_t)(n <= 255u ? n : n - 256u) << 40);
  if ((uint32_t)lane < hl) out[lane] = (uint8_t)(hv >> (8 * lane));
  e.o = hl;
  e.bstart = e.pos = 0;
  e.bend = min(kZstdBlockBytes, n);
  e.nlit = e.nseq = e.lit_mark = 0;
  e.rep[0] = 1;
  e.rep[1] = 4;
  e.rep[2] = 8;
  zstd_build_predefined(e.w.pre(), e.w.fake_base(), lane);
  uint32_t* h = e.w.hist();
  for (int i = lane; i < 256; i += kWarp) h[i] = 0;
  __syncwarp();
  lz77_compress_chunk(in, n, e, e.w.table(), 1u, 0u, 4u, lane);
  __syncwarp();
  return e.o;
}

}  // namespace detail
}  // namespace zstd
}  // namespace device
}  // namespace nvcomp
