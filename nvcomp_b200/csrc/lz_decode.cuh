// lz_decode.cuh -- block-parallel LZ77 (LZ4 / Snappy) chunk decoder for H100.
//
// One warp owns one chunk.  On tabular data a 64 KB chunk holds 10-15 thousand *short* tokens
// (4-8 output bytes each), so throughput is bounded by warp-instructions per token, not bytes.
//
//  * BLOCK PATH (lz_block): 1 KB of compressed input is staged in shared memory by a TMA bulk copy (the next
//    block is prefetched while this one executes); every lane finds the
//    token chain through its own 32-byte segment (exit table computed right to left, entries resolved
//    across lanes), the ~350-500 tokens of the block are listed in stream order and executed 32 per
//    step, one token per lane: literals from the staged block, matches in dependency rounds.
//  * The most recent 4 KB of output live in a per-warp shared-memory ring (explicit 32-bit shared
//    addressing), so match sources are read at shared-memory latency; completed 512-byte blocks are
//    flushed to HBM with 16-byte aligned vector stores (full-line writes, DRAM traffic == algorithmic
//    bytes).  Matches that reach further back than the ring read the flushed bytes from global memory.
//  * SERIAL PATH (P::serial_token + lz_emit_*): tokens with length-extension bytes / long lengths are
//    parsed once by the whole warp; up to 192 bytes they are executed inside the ring, longer runs go
//    straight to global memory as 16-byte vectors (periodic runs are built in registers, no
//    store->load round trip) and the ring restarts empty behind them.  A serial token looks at the token
//    behind it before it moves its bytes (lz_serial_lookahead): the block copy that follows is in flight
//    during the move and the driver does not peek at global memory in steady state.
//  * Chunks that compressed >= 4x (and incompressible ones) never enter this machinery: a classification
//    pass puts them on the light kernel's list (lz_sched.cuh), which decodes them with the direct
//    global-memory token loop of lz4_decode.cuh / snappy_decode.cuh.
//
// Format specifics (token grammar, stream end, size limits) come from a policy.
#pragma once

#include "common.cuh"

// counters for the host emulator's statistics build (tests/emu); nothing in the product
#ifndef B200_LZ_STAT
#define B200_LZ_STAT(slot, n) ((void)0)
#endif

namespace b200 {

constexpr uint32_t kRingBytes = 4096;
constexpr uint32_t kRingMask = kRingBytes - 1;
constexpr uint32_t kFlushBlock = 512;
// A match source is served from the ring only if it is younger than this many bytes
// (ring size minus the largest output one execution step can append, minus alignment slack).
constexpr uint32_t kRingReach = kRingBytes - 1024 - 16;

struct LzState {
  const uint8_t* in;
  uint32_t in_n;
  uint8_t* out;        // chunk output base (any alignment)
  uint64_t out_cap;    // capacity (LZ4) or exact size (Snappy)
  uint32_t ip;         // input cursor
  uint32_t op;         // output cursor (bytes produced)
  uint32_t flushed;    // output bytes already in global memory
  uint32_t ring_lo;    // lowest output offset whose bytes are valid in the ring
  uint32_t align;      // (uintptr_t)out & 15: ring index = (offset + align) & mask
  uint32_t ring;       // shared-window address of the kRingBytes ring (32-bit: LDS/STS with immediates)
  // compressed-input staging (lz_block): two block buffers filled by TMA bulk copies behind one mbarrier
  uint32_t cur;        // buffer that holds the block being parsed
  uint32_t pf_ip;      // input position whose block is being prefetched into the other buffer (kNoPrefetch: none)
  uint32_t parity;     // phase parity the next mbarrier wait uses
  uint32_t next;       // what the driver knows about the token at ip (kNext*)
};
constexpr uint32_t kNoPrefetch = 0xffffffffu;
constexpr uint32_t kNextUnknown = 0, kNextSerial = 1, kNextBlock = 2;

__device__ __forceinline__ uint32_t ring_idx(const LzState& s, uint32_t off) {
  return (off + s.align) & kRingMask;
}
__device__ __forceinline__ uint32_t ring_ld(const LzState& s, uint32_t off) { return lds_u8(s.ring + ring_idx(s, off)); }
__device__ __forceinline__ void ring_st(const LzState& s, uint32_t off, uint32_t v) { sts_u8(s.ring + ring_idx(s, off), v); }
// Write ring bytes [s.flushed, upto) to global memory.  Vector stores where the global
// address is 16-byte aligned, byte stores for ragged ends.
__device__ __forceinline__ void lz_flush(LzState& s, uint32_t upto, int lane) {
  uint32_t f = s.flushed;
  if (upto <= f) return;
  __syncwarp();
  // ragged head up to the next 16-byte boundary (in aligned space)
  uint32_t head = (16u - ((f + s.align) & 15u)) & 15u;
  if (head > upto - f) head = upto - f;
  if ((uint32_t)lane < head) s.out[f + lane] = (uint8_t)ring_ld(s, f + lane);
  f += head;
  const uint32_t nvec = (upto - f) >> 4;
  for (uint32_t v = lane; v < nvec; v += kWarp) {
    const uint32_t o = f + (v << 4);
    const uint4 d = lds_v4(s.ring + ring_idx(s, o));
    st_v4((uint4*)(s.out + o), d);
  }
  f += nvec << 4;
  const uint32_t tail = upto - f;
  if ((uint32_t)lane < tail) s.out[f + lane] = (uint8_t)ring_ld(s, f + lane);
  s.flushed = upto;
}

// Flush every completed 512-byte block (keeps global stores full-line).
__device__ __forceinline__ void lz_flush_blocks(LzState& s, int lane) {
  const uint32_t lim = ((s.op + s.align) & ~(kFlushBlock - 1));
  if (lim > s.flushed + s.align) lz_flush(s, lim - s.align, lane);
}

// ---------------------------------------------------------------------------
// Format policies.  A "token" is one LZ4 sequence (literals + match) or one Snappy element (literal
// OR copy).  Everything the block parser needs is a pure function of the token's first byte:
//   sizes4(w): for the four bytes of w, taken as token tags, the distance to the next token (1..32),
//              or kTokStop for a token the lane-parallel path does not take (length-extension
//              bytes, long literals / copies, copy-4) -- SIMD within a 32-bit register
// fields() extracts literal length / match length / offset for execution.
// ---------------------------------------------------------------------------
constexpr uint32_t kTokStop = 64;
constexpr uint32_t kTokExt = 0x80;      // sizes4 marker: the size depends on an extension byte (P::ext_size)
constexpr uint32_t kMaxTokOut = 32;     // output bytes of one fast token (32 tokens x 32 bytes = one step)

// 4 bytes at an arbitrary position of a shared-memory buffer (two aligned words + funnel shift)
__device__ __forceinline__ uint32_t lds_u32_any(uint32_t base, uint32_t pos) {
  const uint32_t a = base + (pos & ~3u);
  return __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (pos & 3u) * 8u);
}
// offset of byte p of a lane's 32-byte row in the lane-private bank layout (word (p >> 2) * 32 + lane)
__device__ __forceinline__ uint32_t lane_private(uint32_t p) { return (p >> 2) * 124u + p; }
// per-byte mask 0xff where the low bit of the byte of x is set (x has only bit 0 of every byte)
__device__ __forceinline__ uint32_t byte_mask(uint32_t x) { return (x << 8) - x; }

struct Lz4Policy {
  // sequence: token, L literals, 2-byte offset; fast when the literal nibble is < 15.  A match nibble of 15 is
  // followed by length-extension bytes: sizes4 marks it kTokExt | (size with one extension byte) and the chain
  // step (lz_block) looks at that byte -- one byte below 14 - L keeps the token fast (M = 19 + ext, L + M <= 32).
  static constexpr bool kHasExt = true;
  __device__ static __forceinline__ uint32_t sizes4(uint32_t w) {
    const uint32_t L = (w >> 4) & 0x0f0f0f0fu, Mn = w & 0x0f0f0f0fu;
    // nibble == 15  <=>  nibble + 1 carries into bit 4
    const uint32_t stop = byte_mask(((L + 0x01010101u) >> 4) & 0x01010101u);
    const uint32_t ext = ((Mn + 0x01010101u) >> 4) & 0x01010101u;
    const uint32_t sz = L + 0x03030303u + ext;                 // + 1 extension byte
    return ((sz | (ext << 7)) & ~stop) | (stop & 0x40404040u);
  }
  // size of a token sizes4 marked kTokExt: blk/pos locate the token, marked = kTokExt | (4 + L)
  __device__ static __forceinline__ uint32_t ext_size(uint32_t blk, uint32_t pos, uint32_t marked) {
    const uint32_t sz = marked & 0x7fu;                        // 4 + L
    const uint32_t ext = lds_u8(blk + pos + sz - 1u);
    return ext + sz < 18u ? sz : kTokStop;                     // ext < 14 - L
  }
  __device__ static __forceinline__ void fields(uint32_t blk, uint32_t pos, uint32_t& L, uint32_t& M,
                                                uint32_t& off, uint32_t& lit_at) {
    const uint32_t x = lds_u32_any(blk, pos);
    L = (x >> 4) & 15u;
    M = (x & 15u) + 4u;
    lit_at = pos + 1u;
    uint32_t y = x >> 8;                                       // offset (2 bytes), first extension byte
    if (L) y = lds_u32_any(blk, pos + 1u + L);
    off = y & 0xffffu;
    if (M == 19u) M += (y >> 16) & 0xffu;
  }
  // does the token at p need the serial path?  (p has at least kSegBytes readable bytes)
  __device__ static __forceinline__ bool is_stop(const uint8_t* __restrict__ p) {
    const uint32_t b0 = p[0], L = b0 >> 4;
    if (L == 15u) return true;
    return (b0 & 15u) == 15u && (uint32_t)p[3u + L] + L > 13u;
  }
};

struct SnappyPolicy {
  static constexpr bool kHasExt = false;
  __device__ static __forceinline__ uint32_t ext_size(uint32_t, uint32_t, uint32_t) { return kTokStop; }
  // literal (kind 0): 1 + (h+1) bytes, fast up to 31 literal bytes; copy-1: 2 bytes; copy-2: 3 bytes, fast up to
  // kMaxTokOut output bytes; copy-4: serial
  __device__ static __forceinline__ uint32_t sizes4(uint32_t w) {
    const uint32_t kind = w & 0x03030303u, h = (w >> 2) & 0x3f3f3f3fu;
    const uint32_t k1 = kind & 0x01010101u, k2 = (kind >> 1) & 0x01010101u;
    const uint32_t nz = byte_mask(k1 | k2);                       // 0xff where the element is a copy
    const uint32_t sz = ((kind + 0x01010101u) & nz) | ((h + 0x02020202u) & ~nz);
    // stops: kind 3; literal with h >= 31; copy-2 with h >= 32 (more than 32 output bytes)
    const uint32_t h31 = ((h + 0x61616161u) >> 7) & 0x01010101u;  // h >= 31
    const uint32_t h32 = (h >> 5) & 0x01010101u;                  // h >= 32
    const uint32_t stop = (k1 & k2) | (h31 & ~(k1 | k2)) | (h32 & k2);
    const uint32_t sm = byte_mask(stop);
    return (sz & ~sm) | (sm & 0x40404040u);
  }
  __device__ static __forceinline__ void fields(uint32_t blk, uint32_t pos, uint32_t& L, uint32_t& M,
                                                uint32_t& off, uint32_t& lit_at) {
    const uint32_t x = lds_u32_any(blk, pos);
    const uint32_t kind = x & 3u, h = (x >> 2) & 63u;
    lit_at = pos + 1u;
    const uint32_t len = kind == 1u ? 4u + (h & 7u) : h + 1u;
    L = kind == 0u ? len : 0u;
    M = kind == 0u ? 0u : len;
    off = kind == 1u ? ((x >> 5) & 7u) << 8 | ((x >> 8) & 255u) : (x >> 8) & 0xffffu;
  }
  __device__ static __forceinline__ bool is_stop(const uint8_t* __restrict__ p) {
    const uint32_t b0 = p[0];
    const uint32_t kind = b0 & 3u, h = b0 >> 2;
    return kind == 3u || (kind == 0u && h >= 31u) || (kind == 2u && h >= 32u);
  }
};

// ---------------------------------------------------------------------------
// Block path.  One call parses up to kBlkBytes of compressed input and executes its tokens.
//
//   1. stage   the block (16-byte aligned base, kBlkPad more bytes for tokens that start in the last
//              segment) arrives by cp.async.bulk; lane l reads its 32-byte segment and writes the token
//              size every byte would have as a tag (sizes4) into the other block buffer.
//   2. chain   every lane computes, right to left over its own 32 size bytes (in registers, fully
//              unrolled), where a token chain entering its segment at byte p leaves it: a 32-entry
//              exit table per lane.  The true entry of every segment is the fixpoint of
//              entry[l] = exit[l-1][entry[l-1]] with entry[0] known: one shuffle + one table lookup
//              per round, as many rounds as mis-guessed entries survive (streams re-synchronise
//              within a few tokens), at most 32.
//   3. walk    each lane walks the tokens of its segment (size bytes only): count, warp scan, then
//              the positions of all tokens of the block are listed in stream order.
//   4. execute 32 consecutive tokens per step, one per lane: a warp scan of the output lengths
//              places them, literals come from the staged block, matches run in dependency rounds:
//              a match runs as soon as the tokens of this step that produce its source bytes have
//              run (sources below the step are final; sources flushed long ago are read from global
//              memory as aligned words before the rounds).
// ---------------------------------------------------------------------------
constexpr uint32_t kSegBytes = 32;
constexpr uint32_t kBlkBytes = 32 * kSegBytes;
constexpr uint32_t kBlkPad = 32;
constexpr uint32_t kBlkStage = kBlkBytes + kBlkPad;
constexpr uint32_t kMaxStepOut = 32 * kMaxTokOut;   // output bytes one step may append (the ring reach depends on it)
constexpr uint32_t kSmemIn = kRingBytes;            // two block buffers: the staged block | its token sizes, then the
                                                    // next block prefetched over the (dead) sizes; roles swap per block
constexpr uint32_t kSmemRec = kSmemIn + 2 * kBlkStage;  // exit tables (1 B x 1024), then token positions (2 B x 512)
constexpr uint32_t kSmemMbar = kSmemRec + kBlkBytes;    // mbarrier of the TMA bulk copies
constexpr uint32_t kLzWarpSmem = kSmemMbar + 16;
static_assert(kRingReach + kMaxStepOut + 16 <= kRingBytes, "ring reach");
static_assert(kSmemRec % 16 == 0 && kSmemMbar % 8 == 0 && kBlkStage % 16 == 0, "alignment");

// Called once per warp before its first chunk (the barrier lives as long as the kernel).
__device__ __forceinline__ void lz_warp_init(uint32_t ring, int lane) {
  if (lane == 0) mbar_init(ring + kSmemMbar, 1);
  __syncwarp();
}
// wait for the bulk copy in flight (one is in flight whenever this is called)
__device__ __forceinline__ void lz_stage_wait(LzState& s) {
  mbar_wait(s.ring + kSmemMbar, s.parity);
  s.parity ^= 1u;
}
// lane 0 starts the bulk copy of `bytes` (multiple of 16) from the 16-byte aligned `src` into block buffer `buf`
__device__ __forceinline__ void lz_stage_issue(const LzState& s, uint32_t buf, const uint8_t* src, uint32_t bytes, int lane) {
  fence_proxy_async_smem();                         // every lane's generic-proxy accesses to the buffer are ordered
  __syncwarp();                                     // ... and done ...
  if (lane == 0) {
    fence_proxy_async_smem();                       // ... before the async proxy overwrites it
    mbar_expect_tx(s.ring + kSmemMbar, bytes);
    tma_bulk_g2s(s.ring + kSmemIn + kBlkStage * buf, src, bytes, s.ring + kSmemMbar);
  }
}

// Starts the copy of the block that begins at stream position next_ip into the idle buffer (at most one copy is in
// flight: the caller checks s.pf_ip).  False when too few bytes are left for the block path.
__device__ __forceinline__ bool lz_prefetch_block(LzState& s, uint32_t next_ip, int lane) {
  const uint32_t nmis = (uint32_t)((uintptr_t)(s.in + next_ip) & 15u);
  const uint32_t navail = s.in_n - next_ip + nmis;
  if (navail < kSegBytes + kBlkPad) return false;
  const uint32_t nnl = min((navail - kBlkPad) / kSegBytes, 32u);
  lz_stage_issue(s, s.cur ^ 1u, s.in + next_ip - nmis, kSegBytes * nnl + kBlkPad, lane);
  s.pf_ip = next_ip;
  return true;
}

// A serial token knows where it ends before it moves its bytes: look at the token behind it then (the load and, when
// the block path will take over there, the copy of that block overlap the byte moves) and leave the answer in s.next.
template <class P>
__device__ __forceinline__ void lz_serial_lookahead(LzState& s, uint32_t next_ip, int lane) {
  s.next = kNextUnknown;
  if (s.in_n - next_ip < kSegBytes + kBlkPad) return;
  if (P::is_stop(s.in + next_ip)) { s.next = kNextSerial; return; }
  s.next = kNextBlock;
  if (s.pf_ip == kNoPrefetch) lz_prefetch_block(s, next_ip, lane);
}

// Returns the number of tokens retired (0: nothing done, the caller takes the serial path), -1 on a
// malformed stream.
template <class P>
__device__ __forceinline__ int lz_block(LzState& s, int lane) {
  const uint32_t ul = (uint32_t)lane;
  const uint8_t* const ipp = s.in + s.ip;
  const uint32_t mis = (uint32_t)((uintptr_t)ipp & 15u);
  const uint32_t avail = s.in_n - s.ip + mis;                 // bytes from the aligned base to the stream end
  if (avail < kSegBytes + kBlkPad) return 0;
  uint32_t nl = (avail - kBlkPad) / kSegBytes;                // segments that lie (with the pad) inside the stream
  if (nl > 32u) nl = 32u;
  const uint8_t* const abase = ipp - mis;
  const uint32_t rec = s.ring + kSmemRec;

  // ---- 1. stage: TMA bulk copy of the block into shared memory -----------------------------------
  // The previous call already prefetched this block if its chain ended at a token boundary (below); otherwise
  // (first block of the chunk, after serial tokens) it is fetched now.  Either way exactly one copy is in flight.
  if (s.pf_ip != kNoPrefetch && s.pf_ip != s.ip) { lz_stage_wait(s); s.pf_ip = kNoPrefetch; }   // stale prefetch
  if (s.pf_ip == s.ip) s.cur ^= 1u;
  else lz_stage_issue(s, s.cur, abase, kSegBytes * nl + kBlkPad, lane);
  s.pf_ip = kNoPrefetch;
  lz_stage_wait(s);
  const uint32_t blk = s.ring + kSmemIn + kBlkStage * s.cur, szs = s.ring + kSmemIn + kBlkStage * (s.cur ^ 1u);
  uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
  if (ul < nl) {
    a0 = lds_v4(blk + kSegBytes * ul);
    a1 = lds_v4(blk + kSegBytes * ul + 16u);
  }
  // Per-lane byte arrays (token sizes, exit table) use a lane-private bank layout: byte p of lane l lives in
  // word (p >> 2) * 32 + l, i.e. every lane stays in its own shared-memory bank whatever p it indexes
  // (32-byte rows per lane would put eight lanes on one bank).
  uint32_t w[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
  const uint32_t my_sz = szs + 4u * ul, my_ex = rec + 4u * ul;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    w[i] = P::sizes4(w[i]);
    sts_u32(my_sz + 128u * i, w[i]);
  }
  // ---- 2. chain: exit table of this lane's segment (code >= 32: the chain ends in a stop token) ----
  // (a size that depends on an extension byte -- sizes4 marked it kTokExt -- counts with its one-byte form here; the
  // walk below looks at the byte for the tokens that are really on the chain and ends the block where it is not)
#pragma unroll
  for (int p = 31; p >= 0; --p) {
    const uint32_t q = (uint32_t)p + ((w[p >> 2] >> (8 * (p & 3))) & (P::kHasExt ? 0x7fu : 0xffu));
    const uint32_t code = (q >= kSegBytes) ? q - kSegBytes : lds_u8(my_ex + lane_private(q));
    sts_u8(my_ex + (uint32_t)(128 * (p >> 2) + (p & 3)), code);
  }
  __syncwarp();
  // entry of every segment: fixpoint of e[l] = exit[l-1][e[l-1]], e[0] = mis.  A stop exit hands the next
  // lane entry 0: lanes behind a stop are ignored below, this only keeps the iteration short.
  uint32_t e = ul == 0u ? mis : 0u;
  {
    const uint32_t prev = my_ex - 4u;
    while (true) {
      B200_LZ_STAT(7, 1);
      const uint32_t pe = __shfl_up_sync(kFull, e, 1);
      uint32_t ne = mis;
      if (ul != 0u) { ne = lds_u8(prev + lane_private(pe)); if (ne >= kSegBytes) ne = 0u; }
      const bool changed = ne != e;
      e = ne;
      if (!__any_sync(kFull, changed)) break;
    }
  }
  const uint32_t my_exit = lds_u8(my_ex + lane_private(e));
  const unsigned stopm = __ballot_sync(kFull, ul < nl && my_exit >= kSegBytes);
  uint32_t stop_lane = stopm ? (uint32_t)__ffs((int)stopm) - 1u : 32u;
  // ---- 3. walk: tokens of this lane's segment ------------------------------------------------------
  const bool active = ul < nl && ul <= stop_lane;
  uint32_t p = e, cnt = 0;
  bool ext_stop = false;
  if (active) {
    while (p < kSegBytes) {
      uint32_t sz = lds_u8(my_sz + lane_private(p));
      if (sz == kTokStop) break;
      if (P::kHasExt && (sz & kTokExt)) {
        sz = P::ext_size(blk, kSegBytes * ul + p, sz);
        if (sz == kTokStop) { ext_stop = true; break; }
      }
      ++cnt;
      p += sz;
    }
  }
  if (P::kHasExt) {
    // a token whose extension byte makes it long is a stop token after all: the block ends there
    const unsigned em = __ballot_sync(kFull, ext_stop);
    if (em) stop_lane = min(stop_lane, (uint32_t)__ffs((int)em) - 1u);
    if (ul > stop_lane) cnt = 0;
  }
  // block end: the stop token, or where the chain leaves the last segment
  const uint32_t end_pos = __shfl_sync(kFull, kSegBytes * ul + p, (int)(stop_lane < 32u ? stop_lane : nl - 1u));
  uint32_t incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += o;
  }
  const uint32_t N = __shfl_sync(kFull, incl, 31);
  if (N == 0u) return 0;
  __syncwarp();                                                 // exit tables are dead: positions overwrite them
  {
    uint32_t ra = rec + 2u * (incl - cnt), q = e;
    for (uint32_t j = 0; j < cnt; ++j) {
      sts_u16(ra, kSegBytes * ul + q);
      q += lds_u8(my_sz + lane_private(q)) & (P::kHasExt ? 0x7fu : 0xffu);
      ra += 2u;
    }
  }
  // the size bytes are dead: prefetch the next block over them while this one executes (only when this block
  // ends at a token boundary the block path will continue from)
  if (stop_lane == 32u) lz_prefetch_block(s, s.ip + end_pos - mis, lane);
  __syncwarp();

  // ---- 4. execute ------------------------------------------------------------------------------
  // Output positions are kept in "aligned space" (offset + s.align): the ring index is (pos & mask)
  // and (s.out - s.align)[pos] is the global address.  Every lane moves at most 8 literal and 8 match
  // bytes of its token itself; what a longer token has beyond that is moved by the whole warp, one
  // token at a time (a long token must not make 31 short ones loop).
  const uint32_t rbase = s.ring;
  const uint8_t* const outa = s.out - s.align;
  const uint32_t cap_left0 = (uint32_t)min(s.out_cap - s.op, (uint64_t)0xffffffffu);
  uint32_t produced = 0;
  B200_LZ_STAT(5, 1);
  for (uint32_t t0 = 0; t0 < N; t0 += 32u) {
    B200_LZ_STAT(0, 1);
    B200_LZ_STAT(1, min(N - t0, 32u));
    const bool valid = ul < N - t0;
    const uint32_t pos = lds_u16(rec + 2u * (t0 + (valid ? ul : 0u)));
    uint32_t L, M, off, lit_at;
    P::fields(blk, pos, L, M, off, lit_at);
    if (!valid) { L = 0; M = 0; }
    const uint32_t len = L + M;
    uint32_t run = len;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(kFull, run, d);
      if (lane >= d) run += o;
    }
    const uint32_t step_out = __shfl_sync(kFull, run, 31);
    if (step_out > cap_left0 - produced) return -1;
    const uint32_t step_lo = s.op + s.align;
    const uint32_t dst = step_lo + run - len;
    const uint32_t o_mat = dst + L;
    const bool has = M != 0u;
    // off == 0 or beyond the bytes produced so far: malformed (off - 1 wraps to 0xffffffff for off == 0)
    if (__any_sync(kFull, has && off - 1u >= o_mat - s.align)) return -1;
    // a token that crosses the end of the ring goes byte-wise with masked indices
    const uint32_t didx_l = dst & kRingMask;
    const bool wrap = didx_l + len > kRingBytes;
    // ---- literals
    const unsigned litm = __ballot_sync(kFull, L != 0u);
    if (litm) {
      const uint32_t la = blk + lit_at, ld = rbase + didx_l;
      if (L != 0u && !wrap) {
        const uint32_t x0 = lds_u8<0>(la), x1 = lds_u8<1>(la), x2 = lds_u8<2>(la), x3 = lds_u8<3>(la);
        sts_u8<0>(ld, x0);
        if (L > 1u) sts_u8<1>(ld, x1);
        if (L > 2u) sts_u8<2>(ld, x2);
        if (L > 3u) sts_u8<3>(ld, x3);
      }
      unsigned longl = __ballot_sync(kFull, L > 4u || (L != 0u && wrap));
      if (longl) {
        if (L > 4u && !wrap) {
          const uint32_t x0 = lds_u8<4>(la), x1 = lds_u8<5>(la), x2 = lds_u8<6>(la), x3 = lds_u8<7>(la);
          sts_u8<4>(ld, x0);
          if (L > 5u) sts_u8<5>(ld, x1);
          if (L > 6u) sts_u8<6>(ld, x2);
          if (L > 7u) sts_u8<7>(ld, x3);
        }
        longl = __ballot_sync(kFull, L > 8u || (L != 0u && wrap));
        while (longl) {                                        // whole warp: the rest of one long literal per round
          const int t = __ffs((int)longl) - 1;
          longl &= longl - 1u;
          const uint32_t tL = __shfl_sync(kFull, L, t), tla = __shfl_sync(kFull, la, t), td = __shfl_sync(kFull, dst, t);
          const uint32_t j0 = __shfl_sync(kFull, wrap ? 0u : 8u, t);
          const uint32_t j = j0 + ul;                          // L <= 31: one round
          if (j < tL) sts_u8(rbase + ((td + j) & kRingMask), lds_u8(tla + j));
        }
      }
    }
    __syncwarp();
    // ---- matches
    const unsigned hasm = __ballot_sync(kFull, has);
    if (hasm) {
      const uint32_t cur_op = s.op;
      const uint32_t ring_from = max(s.ring_lo, cur_op > kRingReach ? cur_op - kRingReach : 0u) + s.align;
      const uint32_t src = o_mat - off;
      const uint32_t src_end = src + min(M, off);              // exclusive end of the bytes this match reads
      // which tokens of this step produce my source bytes?  Token ranges are consecutive, so the
      // producers are the lanes from the one holding byte max(src, step_lo) to the one holding src_end-1
      // (own literals precede the own match in program order: the self bit is dropped).
      unsigned dep = 0;
      const bool inwin = has && src_end > step_lo;
      if (__any_sync(kFull, inwin)) {
        B200_LZ_STAT(3, 1);
        B200_LZ_STAT(6, __popc(__ballot_sync(kFull, inwin)));
        const uint32_t key = valid ? dst : 0xffffffffu;
        const uint32_t qa = max(src, step_lo), qb = src_end - 1u;
        uint32_t ja = 0, jb = 0;
#pragma unroll
        for (uint32_t st = 16; st; st >>= 1) {
          const uint32_t va = __shfl_sync(kFull, key, (int)(ja + st));
          const uint32_t vb = __shfl_sync(kFull, key, (int)(jb + st));
          if (va <= qa) ja += st;
          if (vb <= qb) jb += st;
        }
        if (inwin) dep = ((2u << jb) - 1u) & ~((1u << ja) - 1u) & ~(1u << ul);
      }
      const uint32_t sidx = src & kRingMask;
      const bool in_ring = src >= ring_from && sidx + M + 8u <= kRingBytes;
      // flushed long ago: read from the output buffer in global memory (whole words around the source: they must
      // lie below this step's first byte, i.e. inside what the chunk has produced)
      const bool far = src + M <= ring_from && (src & ~3u) + 12u <= step_lo;
      // groups of four bytes are loaded, then stored: needs off >= 4 and M >= 4 (shorter periods / copies
      // and anything that crosses the end of the ring take the byte loop)
      const bool simple = !wrap && off >= 4u && M >= 4u && (in_ring || far);
      const bool c_r0 = has && simple, c_r = c_r0 && !far, c_b = has && !simple;
      const uint32_t dp = rbase + (o_mat & kRingMask);
      const uint32_t sa = rbase + (sidx & ~3u), sh = (src & 3u) * 8u;    // aligned words around the source
      // sources flushed long ago are final: those matches run first, outside the rounds (their bytes may feed round 1)
      const bool c_g = c_r0 && far;
      const unsigned m_g = __ballot_sync(kFull, c_g);
      if (m_g) {
        if (c_g) {
          const uint8_t* const gp = outa + (src & ~3u);
          const uint32_t w0 = ldg_u32<0>(gp), w1 = ldg_u32<4>(gp);
          const uint32_t x = __funnelshift_r(w0, w1, sh);
          sts_u8<0>(dp, x);
          sts_u8<1>(dp, x >> 8);
          sts_u8<2>(dp, x >> 16);
          sts_u8<3>(dp, x >> 24);
          if (M > 4u) {
            const uint32_t y = __funnelshift_r(w1, ldg_u32<8>(gp), sh);
            sts_u8<4>(dp, y);
            if (M > 5u) sts_u8<5>(dp, y >> 8);
            if (M > 6u) sts_u8<6>(dp, y >> 16);
            if (M > 7u) sts_u8<7>(dp, y >> 24);
          }
        }
        unsigned lg = __ballot_sync(kFull, c_g && M > 8u);      // bytes 8.. of a long far match: whole warp
        while (lg) {
          const int t = __ffs((int)lg) - 1;
          lg &= lg - 1u;
          const uint32_t tM = __shfl_sync(kFull, M, t), tsrc = __shfl_sync(kFull, src, t), tdp = __shfl_sync(kFull, dp, t);
          const uint32_t j = 8u + ul;
          if (j < tM) sts_u8(tdp + j, (uint32_t)outa[tsrc + j]);
        }
        __syncwarp();
      }
      const unsigned m_b = __ballot_sync(kFull, c_b);
      const unsigned m_4 = __ballot_sync(kFull, c_r && M > 4u);
      const unsigned m_8 = __ballot_sync(kFull, c_r && M > 8u);
      unsigned done = ~__ballot_sync(kFull, c_r || c_b);
      bool pend = c_r || c_b;
      B200_LZ_STAT(4, __popc(__ballot_sync(kFull, has && far)));
      B200_LZ_STAT(8, __popc(m_b));
      while (done != kFull) {
        B200_LZ_STAT(2, 1);
        const bool ready = pend && (dep & ~done) == 0u;
        const unsigned rm = __ballot_sync(kFull, ready);
        const bool go = ready && c_r;
        if (go) {
          const uint32_t x = __funnelshift_r(lds_u32(sa), lds_u32(sa + 4u), sh);
          sts_u8<0>(dp, x);
          sts_u8<1>(dp, x >> 8);
          sts_u8<2>(dp, x >> 16);
          sts_u8<3>(dp, x >> 24);
        }
        if (rm & m_4) {
          if (go && M > 4u) {                                  // (reloaded: with off < 8 these are bytes stored just above)
            const uint32_t x = __funnelshift_r(lds_u32(sa + 4u), lds_u32(sa + 8u), sh);
            sts_u8<4>(dp, x);
            if (M > 5u) sts_u8<5>(dp, x >> 8);
            if (M > 6u) sts_u8<6>(dp, x >> 16);
            if (M > 7u) sts_u8<7>(dp, x >> 24);
          }
        }
        if (rm & m_b) {
          // short periods / copies, ring wrap-around, sources straddling the flushed boundary: byte by byte,
          // in order (a byte may read what this loop wrote off bytes earlier)
          if (ready && c_b) {
            for (uint32_t j = 0; j < M; ++j) {
              const uint32_t q = src + j;
              const uint32_t b = (q >= ring_from) ? lds_u8(rbase + (q & kRingMask)) : (uint32_t)outa[q];
              sts_u8(rbase + ((o_mat + j) & kRingMask), b);
            }
          }
        }
        __syncwarp();
        unsigned longm = rm & m_8;
        if (longm) {
          // bytes 8.. of the long matches that just ran: whole warp, one match per round (M <= 32).  Byte j of an
          // overlapping match (off < M) repeats byte j mod off.
          do {
            const int t = __ffs((int)longm) - 1;
            longm &= longm - 1u;
            const uint32_t tM = __shfl_sync(kFull, M, t), toff = __shfl_sync(kFull, off, t);
            const uint32_t tsp = __shfl_sync(kFull, sidx, t), tdp = __shfl_sync(kFull, dp, t);
            const uint32_t j = 8u + ul;
            if (j < tM) sts_u8(tdp + j, lds_u8(rbase + tsp + (toff < tM ? j % toff : j)));
          } while (longm);
          __syncwarp();
        }
        done |= rm;
        pend = pend && !ready;
      }
    }
    s.op += step_out;
    produced += step_out;
    lz_flush_blocks(s, lane);
  }
  s.ip += end_pos - mis;
  // what the caller meets at s.ip now: a stop token (the chain ended in one) or the next block (prefetched)
  s.next = stop_lane < 32u ? kNextSerial : kNextBlock;
  return (int)N;
}

// ---------------------------------------------------------------------------
// Medium tokens (too long for the lane-parallel path, L + M <= kMediumMax): executed by the
// whole warp one token at a time but still inside the ring, so the data stays at shared-memory
// latency and later short matches keep hitting the ring.
// ---------------------------------------------------------------------------
constexpr uint32_t kMediumMax = 192;

__device__ __forceinline__ void ring_put_literals(LzState& s, uint32_t dst, const uint8_t* __restrict__ src,
                                                  uint32_t n, int lane) {
  for (uint32_t i = lane; i < n; i += kWarp) ring_st(s, dst + i, src[i]);
}

// dst[0..n) = dst[-off..] with LZ77 semantics, all inside the ring (far sources from global).
__device__ __forceinline__ void ring_match(LzState& s, uint32_t dst, uint32_t off, uint32_t n,
                                           uint32_t ring_from, int lane) {
  const uint32_t src = dst - off;
  if (off >= 32u) {
    // bytes of round k only depend on bytes written in rounds < k
    for (uint32_t base = 0; base < n; base += kWarp) {
      const uint32_t j = base + lane;
      if (j < n) {
        const uint32_t sp = src + j;
        const uint32_t b = (sp >= ring_from) ? ring_ld(s, sp) : (uint32_t)s.out[sp];
        ring_st(s, dst + j, b);
      }
      __syncwarp();
    }
  } else {
    // short period: every byte is src[j mod off], all final before the copy starts
    uint32_t r = (uint32_t)lane % off;
    const uint32_t step = 32u % off;
    for (uint32_t j = lane; j < n; j += kWarp) {
      const uint32_t sp = src + r;
      const uint32_t b = (sp >= ring_from) ? ring_ld(s, sp) : (uint32_t)s.out[sp];
      ring_st(s, dst + j, b);
      r += step;
      if (r >= off) r -= off;
    }
  }
}

__device__ __forceinline__ uint32_t ring_from_of(const LzState& s) {
  return max(s.ring_lo, s.op > kRingReach ? s.op - kRingReach : 0u);
}

// one already-produced output byte, wherever it currently lives
__device__ __forceinline__ uint32_t lz_out_byte(const LzState& s, uint32_t pos, uint32_t ring_from) {
  return (pos >= ring_from) ? ring_ld(s, pos) : (uint32_t)s.out[pos];
}

// ---------------------------------------------------------------------------
// Serial (one token at a time, whole warp) emitters for tokens the lane-parallel path cannot
// take.  Up to kMediumMax bytes stay inside the ring; longer runs go straight to global
// memory as 16-byte vectors and the ring restarts empty behind them.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void lz_emit_literals(LzState& s, const uint8_t* __restrict__ src, uint32_t n, int lane) {
  if (n <= kMediumMax) {
    ring_put_literals(s, s.op, src, n, lane);
    s.op += n;
    return;
  }
  lz_flush(s, s.op, lane);
  warp_copy<true>(s.out + s.op, src, n, lane);
  s.op += n;
  s.flushed = s.op;
  s.ring_lo = s.op;
}

__device__ __forceinline__ void lz_emit_match(LzState& s, uint32_t off, uint32_t n, int lane) {
  __syncwarp();
  if (n <= kMediumMax) {
    ring_match(s, s.op, off, n, ring_from_of(s), lane);
    s.op += n;
    return;
  }
  const uint32_t dst = s.op;
  if (off <= 16u && (off & (off - 1u)) == 0u) {
    // Long run with a period that divides 16 (typed run-length data).  Every 16-byte aligned
    // vector of the run is the same: build it once in registers from the period bytes (ring or
    // global), no store->load round trip, then stream it out with vector stores.
    const uint32_t rf = ring_from_of(s);
    const uint32_t src = dst - off, m = off - 1u;
    const uint32_t head = (16u - ((dst + s.align) & 15u)) & 15u;
    uint32_t wv[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint32_t acc = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) acc |= lz_out_byte(s, src + ((head + 4u * q + i) & m), rf) << (8 * i);
      wv[q] = acc;
    }
    const uint32_t hb = lz_out_byte(s, src + ((uint32_t)lane & m), rf);
    lz_flush(s, dst, lane);                                   // everything before the run is now in global memory
    uint8_t* o = s.out + dst;
    if ((uint32_t)lane < head) o[lane] = (uint8_t)hb;
    const uint32_t nvec = (n - head) >> 4;
    uint4* d16 = (uint4*)(o + head);
    const uint4 pat = make_uint4(wv[0], wv[1], wv[2], wv[3]);
    for (uint32_t v = lane; v < nvec; v += kWarp) st_v4(d16 + v, pat);
    const uint32_t j = head + (nvec << 4) + lane;             // < 16 tail bytes
    if (j < n) {
      const uint32_t k = (j - head) & 15u;                    // position inside the pattern vector
      const uint32_t q = k >> 2;
      const uint32_t wsel = q == 0 ? wv[0] : q == 1 ? wv[1] : q == 2 ? wv[2] : wv[3];
      o[j] = (uint8_t)(wsel >> (8 * (k & 3u)));
    }
  } else {
    lz_flush(s, dst, lane);
    __syncwarp();
    warp_match_copy(s.out + dst, off, n, lane);
  }
  __syncwarp();
  s.op += n;
  s.flushed = s.op;
  s.ring_lo = s.op;
}

// Decode driver shared by LZ4 and Snappy.  P::serial_token(s, lane) executes exactly one token
// at s.ip with the emitters above and returns 1 (continue), 2 (stream finished) or -1 (malformed).
template <class P>
__device__ __forceinline__ bool lz_decode_loop(LzState& s, int lane) {
  while (true) {
    if (P::at_end(s)) break;
    // A token that needs the serial path is recognised from its first bytes: do not pay for a block parse that
    // would retire nothing.  The peek is a global load the whole warp waits for, so it is only made when the
    // previous step does not already tell: a block that ended in a stop token is followed by that token, a block that
    // ran to its end is followed by the next (prefetched) block.
    const uint32_t next = s.next;
    s.next = kNextUnknown;                              // (the block path and serial tokens that look ahead set it)
    if (next != kNextSerial && s.in_n - s.ip >= kSegBytes + kBlkPad && (next == kNextBlock || !P::is_stop(s.in + s.ip))) {
      const int r = lz_block<P>(s, lane);
      if (r < 0) return false;
      if (r > 0) continue;
    }
    B200_LZ_STAT(10, 1);
    const int r = P::serial_token(s, lane);
    if (r < 0) return false;
    lz_flush_blocks(s, lane);
    if (r == 2) break;
  }
  lz_flush(s, s.op, lane);
  return true;
}

template <class P>
__device__ __forceinline__ bool lz_decode_stream(LzState& s, int lane) {
  const bool ok = lz_decode_loop<P>(s, lane);
  if (s.pf_ip != kNoPrefetch) { lz_stage_wait(s); s.pf_ip = kNoPrefetch; }   // no copy may outlive the chunk
  return ok;
}

}  // namespace b200
