/*
 * typed_oracle.c -- CPU restatement of this repo's Cascaded, Bitcomp and ANS streams
 * (test infrastructure; see oracle.h).  PARITY UNPINNED at the stream level: the
 * reference bitstreams are undocumented and no libnvcomp binary exists here (SURVEY.md 8c),
 * so these functions restate the stream definitions in DESIGN.md (and the headers of
 * nvcomp_b200/csrc/{cascaded,bitcomp,ans}.cu) as an independent scalar implementation.
 * The algorithms follow the reference's description: doc/cascaded_overview.md:7-42
 * (RLE / delta / bit-packing layers), benchmarks/benchmark_bitcomp_chunked.cu:32-33
 * (algorithm 0/1, typed), benchmarks/benchmark_ans_chunked.cu:39-47 (rANS).
 */
#include "oracle.h"
#include <stdlib.h>
#include <string.h>

/* Every rejection is a named rule (DESIGN.md lists them by format).  oracle_typed_skip_rules() is a test hook: the
 * rules it names (comma-separated; NULL: none) are not applied in the calling thread, so a test can show that a
 * malformed stream breaks exactly the rules it is built to break.  A skipped rule can make the oracle read or write past
 * the stream or the output: only for callers that leave room for that. */
static __thread const char* skip_rules;
void oracle_typed_skip_rules(const char* names) { skip_rules = names; }
static int broken(const char* rule, int cond)
{
  if (!cond || !skip_rules) return cond;
  size_t k = strlen(rule);
  for (const char* p = skip_rules; (p = strstr(p, rule)) != NULL; p += k)
    if ((p == skip_rules || p[-1] == ',') && (p[k] == ',' || p[k] == 0)) return 0;
  return 1;
}

static uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static void wr32(uint8_t* p, uint32_t v) { memcpy(p, &v, 4); }
static void wr64(uint8_t* p, uint64_t v) { memcpy(p, &v, 8); }

static unsigned type_size(unsigned t)
{
  switch (t) { case 0: case 1: return 1; case 2: case 3: return 2; case 4: case 5: return 4;
               case 6: case 7: return 8; default: return 0; }
}
static int type_signed(unsigned t) { return t == 0 || t == 2 || t == 4 || t == 6; }

static uint64_t get_bits(const uint8_t* words, size_t nbytes, uint64_t bitpos, unsigned bits, int* err)
{
  if (bits == 0) return 0;
  size_t w = (size_t)(bitpos >> 6);
  unsigned s = (unsigned)(bitpos & 63);
  if ((w + 1) * 8 > nbytes) { *err = 1; return 0; }
  uint64_t v = rd64(words + 8 * w) >> s;
  if (s + bits > 64) {
    if ((w + 2) * 8 > nbytes) { *err = 1; return 0; }
    v |= rd64(words + 8 * (w + 1)) << (64 - s);
  }
  if (bits < 64) v &= ((1ull << bits) - 1ull);
  return v;
}

static void put_bits(uint8_t* words, uint64_t bitpos, unsigned bits, uint64_t v)
{
  if (bits == 0) return;
  size_t w = (size_t)(bitpos >> 6);
  unsigned s = (unsigned)(bitpos & 63);
  wr64(words + 8 * w, rd64(words + 8 * w) | (v << s));
  if (s + bits > 64) wr64(words + 8 * (w + 1), rd64(words + 8 * (w + 1)) | (v >> (64 - s)));
}

static uint64_t trunc_ts(uint64_t v, unsigned ts) { return ts == 8 ? v : (v & ((1ull << (8 * ts)) - 1ull)); }
static uint64_t sext_ts(uint64_t v, unsigned ts)
{
  if (ts == 8) return v;
  unsigned sh = 64 - 8 * ts;
  return (uint64_t)(((int64_t)(v << sh)) >> sh);
}
static void store_ts(uint8_t* p, uint64_t v, unsigned ts) { memcpy(p, &v, ts); }   /* little endian host */
static uint64_t load_ts(const uint8_t* p, unsigned ts) { uint64_t v = 0; memcpy(&v, p, ts); return v; }

/* ------------------------------------------------------------------ Cascaded */
#define CSC_MAGIC 0x31435343u

typedef struct { uint32_t count, bits; uint64_t minv; const uint8_t* words; size_t nbytes; } stream_t;

static int read_stream(const uint8_t* p, size_t avail, stream_t* s, size_t* used)
{
  if (broken("csc_stream_header_truncated", avail < 16)) return -1;
  s->count = rd32(p); s->bits = rd32(p + 4); s->minv = rd64(p + 8);
  if (broken("csc_stream_bits_above_64", s->bits > 64)) return -1;
  size_t nwords = (size_t)(((uint64_t)s->count * s->bits + 63) / 64);
  if (broken("csc_stream_words_past_partition", 16 + 8 * nwords > avail)) return -1;
  s->words = p + 16; s->nbytes = 8 * nwords;
  *used = 16 + 8 * nwords;
  return 0;
}

static long casc_decode_part(const uint8_t* p, size_t nb, uint8_t* out, size_t n_out, unsigned ts, int R, int D,
                             size_t cap)
{
  size_t hdr = 8 * (size_t)D + ((4 * (size_t)D + 7) & ~(size_t)7);
  if (broken("csc_part_shorter_than_delta_header", nb < hdr)) return -1;
  const uint8_t* firsts = p;
  const uint8_t* cin = p + 8 * D;
  size_t off = hdr, used;
  stream_t runs[8], vals;
  for (int i = 0; i < R; ++i) {
    if (read_stream(p + off, nb - off, &runs[i], &used)) return -1;
    off += used;
  }
  if (read_stream(p + off, nb - off, &vals, &used)) return -1;
  if (broken("csc_value_count_above_partition", vals.count > cap)) return -1;
  uint64_t* cur = (uint64_t*)malloc(sizeof(uint64_t) * (cap + 1));
  uint64_t* nxt = (uint64_t*)malloc(sizeof(uint64_t) * (cap + 1));
  int err = 0;
  size_t count = vals.count;
  for (size_t k = 0; k < count; ++k)
    cur[k] = trunc_ts(get_bits(vals.words, vals.nbytes, (uint64_t)k * vals.bits, vals.bits, &err) + vals.minv, ts);
  int L = R > D ? R : D;
  for (int i = L - 1; i >= 0 && !err; --i) {
    if (i < D) {
      uint32_t c_in = rd32(cin + 4 * i);
      if (c_in == 0) { if (broken("csc_delta_count_zero_with_values", count != 0)) err = 1; }
      else {
        if (broken("csc_delta_count_not_values_plus_1", c_in != count + 1) ||
            broken("csc_delta_count_above_partition", c_in > cap)) { err = 1; break; }
        uint64_t acc = rd64(firsts + 8 * i);
        nxt[0] = trunc_ts(acc, ts);
        for (size_t k = 0; k < count; ++k) { acc += cur[k]; nxt[k + 1] = trunc_ts(acc, ts); }
        count += 1;
        uint64_t* t = cur; cur = nxt; nxt = t;
      }
    }
    if (i < R && !err) {
      if (broken("csc_run_count_not_value_count", runs[i].count != count)) { err = 1; break; }
      size_t total = 0;
      for (size_t k = 0; k < count && !err; ++k) {
        uint64_t len = get_bits(runs[i].words, runs[i].nbytes, (uint64_t)k * runs[i].bits, runs[i].bits, &err)
                       + runs[i].minv;
        /* len > cap - total, not total + len > cap: a length near 2^64 (raw + min wraps) must not wrap the sum */
        if (broken("csc_run_zero_length", len == 0) || broken("csc_runs_total_above_partition", len > cap - total)) {
          err = 1;
          break;
        }
        for (uint64_t j = 0; j < len; ++j) nxt[total + j] = cur[k];
        total += len;
      }
      count = total;
      uint64_t* t = cur; cur = nxt; nxt = t;
    }
  }
  if (!err && broken("csc_total_not_partition", count != n_out)) err = 1;
  if (!err) for (size_t k = 0; k < count; ++k) store_ts(out + k * ts, cur[k], ts);
  free(cur); free(nxt);
  return err ? -1 : (long)(count * ts);
}

long oracle_cascaded_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap)
{
  if (broken("csc_stream_shorter_than_header", n < 20) || broken("csc_magic", rd32(src) != CSC_MAGIC)) return -1;
  uint32_t cfg = rd32(src + 4);
  unsigned type = cfg & 0xff; int R = (cfg >> 8) & 0xff, D = (cfg >> 16) & 0xff;
  unsigned ts = type_size(type);
  uint32_t ulen = rd32(src + 8), P = rd32(src + 12), np = rd32(src + 16);
  if (broken("csc_type", !ts) || broken("csc_R_above_7", R > 7) || broken("csc_D_above_7", D > 7) ||
      broken("csc_part_size_below_512", P < 512) || broken("csc_part_size_above_16384", P > 16384) ||
      broken("csc_part_size_not_multiple_of_8", P % 8))
    return -1;
  if (!ts) ts = 1;
  uint32_t tail = ulen % ts, whole = ulen - tail;   /* partitions cover the whole elements */
  if (broken("csc_num_parts_too_small", (uint64_t)np * P < whole) ||
      broken("csc_num_parts_too_large", np && (uint64_t)(np - 1) * P >= whole))
    return -1;
  if (broken("csc_offset_table_beyond_stream", 20 + 4 * ((size_t)np + 1) > n) || broken("csc_n_above_capacity", ulen > cap))
    return -1;
  for (uint32_t p = 0; p < np; ++p) {
    uint32_t o0 = rd32(src + 20 + 4 * p), o1 = rd32(src + 20 + 4 * (p + 1));
    if (broken("csc_offset_misaligned", o0 & 7) || broken("csc_offset_decreasing", o0 > o1) ||
        broken("csc_offset_beyond_stream", o1 > n))
      return -1;
    uint32_t begin = p * P, nb = whole - begin < P ? whole - begin : P;
    if (casc_decode_part(src + o0, o1 - o0, dst + begin, nb / ts, ts, R, D, P / ts) < 0) return -1;
  }
  if (tail) {   /* trailing bytes: one verbatim word after the last partition */
    uint32_t to = rd32(src + 20 + 4 * np);
    if (broken("csc_tail_word_missing", (uint64_t)to + 8 > n)) return -1;
    memcpy(dst + whole, src + to, tail);
  }
  return (long)ulen;
}

long oracle_cascaded_decompressed_size(const uint8_t* src, size_t n)
{
  if (n < 20 || rd32(src) != CSC_MAGIC) return -1;
  return (long)rd32(src + 8);
}

static size_t pack_stream(uint8_t* dst, const uint64_t* v, size_t count, int use_bp, int is_signed, unsigned ts,
                          unsigned raw_bits)
{
  uint64_t mn = 0, mx = 0;
  unsigned bits = raw_bits;
  if (use_bp) {
    bits = 0;
    if (count) {
      uint64_t bias = is_signed ? (1ull << 63) : 0;
      uint64_t lo = ~0ull, hi = 0;
      for (size_t k = 0; k < count; ++k) {
        uint64_t x = (is_signed ? sext_ts(v[k], ts) : v[k]) ^ bias;
        if (x < lo) lo = x;
        if (x > hi) hi = x;
      }
      mn = lo ^ bias; mx = hi ^ bias;
      uint64_t range = mx - mn;
      while (range) { ++bits; range >>= 1; }
    }
  }
  size_t nwords = (size_t)(((uint64_t)count * bits + 63) / 64);
  wr32(dst, (uint32_t)count); wr32(dst + 4, bits); wr64(dst + 8, use_bp ? mn : 0);
  memset(dst + 16, 0, 8 * nwords);
  uint64_t mask = bits < 64 ? ((1ull << bits) - 1ull) : ~0ull;
  for (size_t k = 0; k < count; ++k) {
    uint64_t x = v[k];
    if (use_bp) x = (is_signed ? sext_ts(x, ts) : x) - mn;
    if (bits) put_bits(dst + 16, (uint64_t)k * bits, bits, x & mask);
  }
  return 16 + 8 * nwords;
}

/* opts: chunk_size (partition bytes), type, num_RLEs, num_deltas, use_bp */
long oracle_cascaded_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t P, unsigned type,
                              int R, int D, int use_bp)
{
  unsigned ts = type_size(type);
  if (!ts || P < 512 || P > 16384 || (P % 8)) return -1;
  size_t tail = n % ts, whole = n - tail;
  size_t np = (whole + P - 1) / P;
  size_t off = (20 + 4 * (np + 1) + 7) & ~(size_t)7;
  if (cap < off) return -1;
  wr32(dst, CSC_MAGIC);
  wr32(dst + 4, (type & 0xff) | ((uint32_t)R << 8) | ((uint32_t)D << 16) | ((uint32_t)(use_bp ? 1 : 0) << 24));
  wr32(dst + 8, (uint32_t)n); wr32(dst + 12, (uint32_t)P); wr32(dst + 16, (uint32_t)np);
  /* pad bytes are zero: an odd partition count leaves 4 between the offset table and the first partition */
  memset(dst + 20 + 4 * (np + 1), 0, off - (20 + 4 * (np + 1)));
  size_t cap_e = P / ts;
  uint64_t* cur = (uint64_t*)malloc(8 * (cap_e + 1));
  uint64_t* nxt = (uint64_t*)malloc(8 * (cap_e + 1));
  uint64_t* rl = (uint64_t*)malloc(8 * (cap_e + 1));
  for (size_t p = 0; p < np; ++p) {
    wr32(dst + 20 + 4 * p, (uint32_t)off);
    size_t begin = p * P, nb = whole - begin < P ? whole - begin : P;
    size_t count = nb / ts;
    for (size_t k = 0; k < count; ++k) cur[k] = load_ts(src + begin + k * ts, ts);
    uint8_t* q = dst + off;
    size_t hdr = 8 * (size_t)D + ((4 * (size_t)D + 7) & ~(size_t)7);
    /* worst case of this partition: R run streams at <= 16 bits + one value stream */
    if (off + hdr + (size_t)(R + 1) * 24 + (size_t)R * 2 * cap_e + P + 16 > cap) {
      free(cur); free(nxt); free(rl);
      return -1;
    }
    memset(q, 0, hdr);
    size_t o = hdr;
    int L = R > D ? R : D, had_delta = 0;
    for (int i = 0; i < L; ++i) {
      if (i < R) {
        size_t m = 0;
        for (size_t k = 0; k < count; ++k) {
          if (k == 0 || cur[k] != cur[k - 1]) { nxt[m] = cur[k]; rl[m] = 1; ++m; }
          else rl[m - 1] += 1;
        }
        o += pack_stream(q + o, rl, m, use_bp, 0, 2, 16);
        count = m;
        uint64_t* t = cur; cur = nxt; nxt = t;
      }
      if (i < D) {
        wr64(q + 8 * i, count ? cur[0] : 0);
        wr32(q + 8 * D + 4 * i, (uint32_t)count);
        for (size_t k = 0; k + 1 < count; ++k) nxt[k] = trunc_ts(cur[k + 1] - cur[k], ts);
        count = count ? count - 1 : 0;
        had_delta = 1;
        uint64_t* t = cur; cur = nxt; nxt = t;
      }
    }
    o += pack_stream(q + o, cur, count, use_bp, had_delta ? 1 : type_signed(type), ts, 8 * ts);
    off += (o + 7) & ~(size_t)7;
  }
  wr32(dst + 20 + 4 * np, (uint32_t)off);
  free(cur); free(nxt); free(rl);
  if (tail) {
    if (cap < off + 8) return -1;
    memset(dst + off, 0, 8);
    memcpy(dst + off, src + whole, tail);
    off += 8;
  }
  return (long)off;
}

/* ------------------------------------------------------------------- Bitcomp */
#define BTC_MAGIC 0x31435442u

static uint64_t unzigzag(uint64_t z) { return (z >> 1) ^ (0ull - (z & 1ull)); }
static uint64_t zigzag_ts(uint64_t d, unsigned ts)
{
  int64_t s = (int64_t)sext_ts(d, ts);
  return trunc_ts(((uint64_t)s << 1) ^ (uint64_t)(s >> 63), ts);
}

long oracle_bitcomp_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap)
{
  if (broken("btc_stream_shorter_than_header", n < 16) || broken("btc_magic", rd32(src) != BTC_MAGIC)) return -1;
  unsigned algo = rd32(src + 4) & 0xff, type = (rd32(src + 4) >> 8) & 0xff;
  unsigned ts = type_size(type);
  uint32_t ulen = rd32(src + 8), nblocks = rd32(src + 12);
  if (broken("btc_type", !ts) || broken("btc_algo_above_1", algo > 1) || broken("btc_n_above_capacity", ulen > cap))
    return -1;
  if (!ts) ts = 1;
  size_t ne = ulen / ts;
  if (broken("btc_nblocks_mismatch", nblocks != (ne + 127) / 128) ||
      broken("btc_desc_table_beyond_stream", 16 + 2 * (size_t)nblocks > n))
    return -1;
  size_t off = (16 + 2 * (size_t)nblocks + 7) & ~(size_t)7;
  for (uint32_t b = 0; b < nblocks; ++b) {
    unsigned desc = src[16 + 2 * b] | (src[17 + 2 * b] << 8);
    size_t e0 = (size_t)b * 128, nv = ne - e0 < 128 ? ne - e0 : 128;
    int err = 0;
    if (algo == 0) {
      unsigned bits = desc & 0xff;
      if (broken("btc_algo0_bits_above_64", bits > 64)) return -1;
      size_t bytes = 8 + 16 * (size_t)bits;
      if (broken("btc_payload_beyond_stream", off + bytes > n)) return -1;
      uint64_t acc = rd64(src + off);
      for (size_t k = 0; k < nv; ++k) {
        acc += unzigzag(get_bits(src + off + 8, bytes - 8, (uint64_t)k * bits, bits, &err));
        store_ts(dst + (e0 + k) * ts, acc, ts);
      }
      off += bytes;
    } else {
      unsigned nz = desc & 0xff, bits = desc >> 8;
      if (broken("btc_algo1_nz_above_128", nz > 128) || broken("btc_algo1_bits_above_64", bits > 64)) return -1;
      size_t bytes = 16 + 8 * (((size_t)nz * bits + 63) / 64);
      if (broken("btc_payload_beyond_stream", off + bytes > n)) return -1;
      uint64_t mlo = rd64(src + off), mhi = rd64(src + off + 8);
      if (broken("btc_algo1_popcount_not_nz", (unsigned)(__builtin_popcountll(mlo) + __builtin_popcountll(mhi)) != nz))
        return -1;
      unsigned rank = 0;
      for (size_t k = 0; k < nv; ++k) {
        int set = (int)(((k < 64 ? mlo >> k : mhi >> (k - 64))) & 1);
        uint64_t v = 0;
        if (set) { v = get_bits(src + off + 16, bytes - 16, (uint64_t)rank * bits, bits, &err); ++rank; }
        store_ts(dst + (e0 + k) * ts, v, ts);
      }
      off += bytes;
    }
    if (err) return -1;
  }
  /* trailing bytes of a chunk whose length is not a multiple of the element size: one verbatim word */
  size_t tail = ulen - ne * ts;
  if (tail) {
    if (broken("btc_tail_word_missing", off + 8 > n)) return -1;
    memcpy(dst + ne * ts, src + off, tail);
  }
  return (long)ulen;
}

long oracle_bitcomp_decompressed_size(const uint8_t* src, size_t n)
{
  if (n < 16 || rd32(src) != BTC_MAGIC) return -1;
  return (long)rd32(src + 8);
}

long oracle_bitcomp_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, unsigned algo, unsigned type)
{
  unsigned ts = type_size(type);
  if (!ts || algo > 1) return -1;
  size_t ne = n / ts, nblocks = (ne + 127) / 128;
  size_t off = (16 + 2 * nblocks + 7) & ~(size_t)7;
  if (cap < off + nblocks * (16 + 128 * (size_t)ts) + 8) return -1;
  wr32(dst, BTC_MAGIC); wr32(dst + 4, algo | (type << 8)); wr32(dst + 8, (uint32_t)n);
  wr32(dst + 12, (uint32_t)nblocks);
  memset(dst + 16, 0, off - 16);
  for (size_t b = 0; b < nblocks; ++b) {
    size_t e0 = b * 128, nv = ne - e0 < 128 ? ne - e0 : 128;
    uint64_t v[128], z[128];
    for (size_t k = 0; k < 128; ++k) v[k] = k < nv ? load_ts(src + (e0 + k) * ts, ts) : 0;
    unsigned desc;
    if (algo == 0) {
      uint64_t m = 0;
      for (size_t k = 0; k < 128; ++k) {
        z[k] = (k == 0 || k >= nv) ? 0 : zigzag_ts(trunc_ts(v[k] - v[k - 1], ts), ts);
        m |= z[k];
      }
      unsigned bits = 0;
      while (m) { ++bits; m >>= 1; }
      desc = bits;
      size_t bytes = 8 + 16 * (size_t)bits;
      memset(dst + off, 0, bytes);
      wr64(dst + off, v[0]);
      for (size_t k = 0; k < 128; ++k) put_bits(dst + off + 8, (uint64_t)k * bits, bits, z[k]);
      off += bytes;
    } else {
      uint64_t m = 0, mlo = 0, mhi = 0;
      unsigned nz = 0;
      for (size_t k = 0; k < 128; ++k) {
        m |= v[k];
        if (v[k]) { ++nz; if (k < 64) mlo |= 1ull << k; else mhi |= 1ull << (k - 64); }
      }
      unsigned bits = 0;
      while (m) { ++bits; m >>= 1; }
      desc = nz | (bits << 8);
      size_t bytes = 16 + 8 * (((size_t)nz * bits + 63) / 64);
      memset(dst + off, 0, bytes);
      wr64(dst + off, mlo); wr64(dst + off + 8, mhi);
      unsigned rank = 0;
      for (size_t k = 0; k < 128; ++k) if (v[k]) { put_bits(dst + off + 16, (uint64_t)rank * bits, bits, v[k]); ++rank; }
      off += bytes;
    }
    dst[16 + 2 * b] = (uint8_t)(desc & 255); dst[17 + 2 * b] = (uint8_t)(desc >> 8);
  }
  if (n - ne * ts) {
    memset(dst + off, 0, 8);
    memcpy(dst + off, src + ne * ts, n - ne * ts);
    off += 8;
  }
  return (long)off;
}

/* ----------------------------------------------------------------------- ANS */
#define ANS_MAGIC 0x31534e41u
#define ANS_SEG 16384u
#define ANS_M 4096u
#define ANS_L 65536u

long oracle_ans_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap)
{
  if (broken("ans_stream_shorter_than_header", n < 16) || broken("ans_magic", rd32(src) != ANS_MAGIC)) return -1;
  uint32_t ulen = rd32(src + 4), mode = rd32(src + 8), nseg = rd32(src + 12);
  if (broken("ans_n_above_capacity", ulen > cap)) return -1;
  if (mode == 1) {
    if (broken("ans_mode1_short", 16 + (size_t)ulen > n)) return -1;
    memcpy(dst, src + 16, ulen);
    return (long)ulen;
  }
  if (mode == 2) {
    if (broken("ans_mode2_short", n < 17)) return -1;
    memset(dst, src[16], ulen);
    return (long)ulen;
  }
  if (broken("ans_mode_above_2", mode != 0) || broken("ans_nseg_mismatch", nseg != (ulen + ANS_SEG - 1) / ANS_SEG))
    return -1;
  if (broken("ans_header_beyond_stream", 16 + 512 + 4 * ((size_t)nseg + 1) > n)) return -1;
  uint32_t cum[257];
  cum[0] = 0;
  for (int s = 0; s < 256; ++s) cum[s + 1] = cum[s] + (src[16 + 2 * s] | (src[17 + 2 * s] << 8));
  if (broken("ans_freq_sum_not_4096", cum[256] != ANS_M)) return -1;
  static __thread uint8_t sym_of[ANS_M];
  for (int s = 0; s < 256; ++s) {
    if (broken("ans_single_freq_4096", cum[s + 1] - cum[s] > 4095)) return -1;
    for (uint32_t k = cum[s]; k < cum[s + 1] && k < ANS_M; ++k) sym_of[k] = (uint8_t)s;
  }
  for (uint32_t sg = 0; sg < nseg; ++sg) {
    uint32_t o0 = rd32(src + 528 + 4 * sg), o1 = rd32(src + 528 + 4 * (sg + 1));
    if (broken("ans_seg_offset_misaligned", o0 & 3) || broken("ans_seg_offset_decreasing", o0 > o1) ||
        broken("ans_seg_offset_past_end", o1 > n) || broken("ans_seg_shorter_than_128", o1 - o0 < 128))
      return -1;
    uint32_t x[32];
    for (int l = 0; l < 32; ++l) x[l] = rd32(src + o0 + 4 * l);
    const uint8_t* words = src + o0 + 128;
    uint32_t nwords = (o1 - o0 - 128) / 2, wpos = 0;
    uint32_t begin = sg * ANS_SEG, ns = ulen - begin < ANS_SEG ? ulen - begin : ANS_SEG;
    /* symbol i belongs to lane i % 32; within a round lanes renormalise in lane order */
    for (uint32_t i = 0; i < ns; ++i) {
      uint32_t l = i & 31;
      uint32_t slot = x[l] & (ANS_M - 1);
      uint32_t s = sym_of[slot];
      dst[begin + i] = (uint8_t)s;
      x[l] = (cum[s + 1] - cum[s]) * (x[l] >> 12) + slot - cum[s];
      if (x[l] < ANS_L) {
        if (broken("ans_words_exhausted", wpos >= nwords)) return -1;
        x[l] = (x[l] << 16) | (uint32_t)(words[2 * wpos] | (words[2 * wpos + 1] << 8));
        ++wpos;
      }
    }
    if (broken("ans_two_leftover_words", nwords - wpos > 1)) return -1;
    for (int l = 0; l < 32; ++l) if (broken("ans_final_state_not_L", x[l] != ANS_L)) return -1;
  }
  return (long)ulen;
}

long oracle_ans_decompressed_size(const uint8_t* src, size_t n)
{
  if (n < 16 || rd32(src) != ANS_MAGIC) return -1;
  return (long)rd32(src + 4);
}

long oracle_ans_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap)
{
  uint32_t nseg = (uint32_t)((n + ANS_SEG - 1) / ANS_SEG);
  if (cap < 16 + 512 + 4 * ((size_t)nseg + 1) + n + 16) return -1;
  uint32_t hist[256] = {0}, freq[256], cum[257];
  for (size_t i = 0; i < n; ++i) hist[src[i]]++;
  uint32_t present = 0, sum = 0, best = 0, bestc = 0;
  for (int s = 0; s < 256; ++s) {
    uint32_t f = 0;
    if (hist[s]) {
      ++present;
      f = (uint32_t)(((uint64_t)hist[s] * ANS_M) / n);
      if (!f) f = 1;
      if (hist[s] > bestc) { bestc = hist[s]; best = s; }
    }
    freq[s] = f; sum += f;
  }
  wr32(dst, ANS_MAGIC); wr32(dst + 4, (uint32_t)n);
  if (n == 0) { wr32(dst + 8, 1); wr32(dst + 12, 0); return 16; }
  if (present <= 1) { wr32(dst + 8, 2); wr32(dst + 12, 0); dst[16] = src[0]; return 17; }
  if (sum < ANS_M) freq[best] += ANS_M - sum;
  while (sum > ANS_M) {
    uint32_t bi = 0, bf = 0;
    for (int s = 0; s < 256; ++s) if (freq[s] > bf) { bf = freq[s]; bi = s; }
    uint32_t dec = sum - ANS_M < bf - 1 ? sum - ANS_M : bf - 1;
    freq[bi] = bf - dec; sum -= dec;
  }
  cum[0] = 0;
  for (int s = 0; s < 256; ++s) cum[s + 1] = cum[s] + freq[s];
  uint32_t off = (16 + 512 + 4 * (nseg + 1) + 3) & ~3u;
  uint16_t* wbuf = (uint16_t*)malloc(2 * ANS_SEG);
  uint8_t* tmp = (uint8_t*)malloc(cap);
  for (uint32_t sg = 0; sg < nseg; ++sg) {
    uint32_t begin = sg * ANS_SEG, ns = (uint32_t)(n - begin < ANS_SEG ? n - begin : ANS_SEG);
    uint32_t x[32], wp = ANS_SEG;
    for (int l = 0; l < 32; ++l) x[l] = ANS_L;
    /* encode backwards; within a round emit in DEcreasing lane order so the forward
     * reader sees increasing lane order */
    for (uint32_t i = ns; i-- > 0;) {
      uint32_t l = i & 31, s = src[begin + i], f = freq[s];
      if (x[l] >= (f << 20)) { wbuf[--wp] = (uint16_t)(x[l] & 0xffff); x[l] >>= 16; }
      x[l] = ((x[l] / f) << 12) + (x[l] % f) + cum[s];
    }
    uint32_t nw = ANS_SEG - wp;
    wr32(tmp + 528 + 4 * sg, off);
    if ((size_t)off + 128 + 2 * (size_t)nw + 4 > cap) { free(wbuf); free(tmp); return -1; }
    for (int l = 0; l < 32; ++l) wr32(tmp + off + 4 * l, x[l]);
    memcpy(tmp + off + 128, wbuf + wp, 2 * (size_t)nw);
    if (nw & 1) { tmp[off + 128 + 2 * nw] = 0; tmp[off + 128 + 2 * nw + 1] = 0; }
    off += 128 + ((2 * nw + 3) & ~3u);
  }
  wr32(tmp + 528 + 4 * nseg, off);
  free(wbuf);
  if (off >= 16 + n) {
    free(tmp);
    wr32(dst + 8, 1); wr32(dst + 12, 0); memcpy(dst + 16, src, n);
    return (long)(16 + n);
  }
  memcpy(dst + 16, tmp + 16, off - 16);
  free(tmp);
  wr32(dst + 8, 0); wr32(dst + 12, nseg);
  for (int s = 0; s < 256; ++s) { dst[16 + 2 * s] = (uint8_t)(freq[s] & 255); dst[17 + 2 * s] = (uint8_t)(freq[s] >> 8); }
  return (long)off;
}
