// nvcomp/device/detail/lz4_decode.cuh -- LZ4 block-format decode for one chunk owned by one warp: the format policy of
// the lane-parallel decoder (lz_decode.cuh), the serial sequence path, the direct loop for chunks that compressed >= 4x
// and the size-query walker.  The batched kernels are in nvcomp_b200/csrc/lz4.cu, the device API in
// nvcomp/device/lz4.cuh.
#pragma once

#include "nvcomp/device/detail/lz_common.cuh"
#include "nvcomp/device/detail/lz_decode.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

// ---------------------------------------------------------------------------
// Length-extension bytes (the 255,255,...,x tail of a 15 nibble): 32 bytes are
// examined per round with a ballot instead of a serial byte walk.
// Returns false on input overrun.
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool lz4_read_ext(const uint8_t* __restrict__ in, uint32_t in_n,
                                             uint32_t& ip, uint32_t& len, int lane) {
  while (true) {
    const uint32_t q = ip + lane;
    const uint32_t b = (q < in_n) ? in[q] : 0u;   // 0 terminates: overrun detected below
    const unsigned stop = __ballot_sync(kFull, b != 255u);
    if (stop == 0) { len += 255u * 32u; ip += 32; continue; }
    const int k = __ffs(stop) - 1;
    len += 255u * (uint32_t)k + __shfl_sync(kFull, b, k);
    ip += k + 1;
    return ip <= in_n;
  }
}

// Walk the sequences of one LZ4 block without copying (size query: LZ4 blocks carry no size header).
// Returns true on a well-formed block; *produced receives the decompressed size.
// kHist (LZ4 frames, lz4frame_decode.cuh): the block starts at output position op0 of its frame, and a match may reach
// back into those op0 earlier bytes; *produced is then the end position (op0 + the block's size).  Without kHist op0
// is ignored and the block starts at 0.
template <bool kHist = false>
__device__ __forceinline__ bool lz4_walk_chunk(const uint8_t* __restrict__ in, uint32_t in_n,
                                               uint32_t* produced, int lane, uint32_t op0 = 0) {
  uint32_t ip = 0;
  uint64_t op = kHist ? op0 : 0;
  if (in_n == 0) { *produced = (uint32_t)op; return true; }
  while (true) {
    if (ip >= in_n) return false;
    const uint32_t tok = in[ip++];
    uint32_t ll = tok >> 4;
    if (ll == 15) { if (!lz4_read_ext(in, in_n, ip, ll, lane)) return false; }
    if (ll > in_n - ip) return false;
    ip += ll; op += ll;
    if (ip >= in_n) break;                 // last sequence carries literals only
    if (in_n - ip < 2) return false;
    const uint32_t off = load_u16(in + ip);
    ip += 2;
    uint32_t ml = tok & 15u;
    if (ml == 15) { if (!lz4_read_ext(in, in_n, ip, ml, lane)) return false; }
    ml += 4;
    if (off == 0 || (uint64_t)off > op) return false;
    op += ml;
    if (op > 0xffffffffull) return false;
  }
  *produced = (uint32_t)op;
  return true;
}

// ---------------------------------------------------------------------------
// Direct decode for chunks that compressed >= 4x (long matches, typed run-length data).  One coalesced
// 32-byte load brings a whole sequence (token, short literals, offset, length-extension bytes) into a
// register window; fields are picked with shuffles / a ballot.  A match whose period (1, 2, 4 or 8 bytes) lies
// inside the literals of its own sequence -- the shape of typed run-length data -- is expanded from the
// window: the 8-byte period is rotated to the destination alignment and broadcast with 16-byte stores,
// no load from the output buffer.  Other matches are copied through memory (lz_common.cuh) with the fields
// already in registers; sequences that do not fit the window (long literal runs, far length
// extensions, the end of the block) take the generic field-by-field path below.
// kHist (LZ4 frames): `out` is the frame's first output byte, the block starts at position op0 with the op0 bytes
// before it final in global memory, matches may reach back into them, and out_cap64 and *produced are positions in
// the frame (end of the block's room, end of the block).  Without kHist op0 is ignored and the block starts at 0.
// ---------------------------------------------------------------------------
template <bool kHist = false>
__device__ __forceinline__ bool lz4_decode_chunk_direct(const uint8_t* __restrict__ in, uint32_t in_n,
                                                        uint8_t* out, uint64_t out_cap64,
                                                        uint32_t* produced, int lane, uint32_t op0 = 0) {
  if (in_n == 0) { *produced = kHist ? op0 : 0; return true; }
  const uint32_t cap = out_cap64 > 0xffffffffull ? 0xffffffffu : (uint32_t)out_cap64;
  const uint32_t ul = (uint32_t)lane;
  uint32_t ip = 0, op = kHist ? op0 : 0;
  while (true) {
    if (ip >= in_n) return false;
    if (ip + 32u <= in_n) {
      // ---- window path
      const uint32_t b = in[ip + ul];
      const uint32_t tok = __shfl_sync(kFull, b, 0);
      const uint32_t ll = tok >> 4;
      if (ll < 15u) {                                              // 15 = extended literal length: generic path
        uint32_t used = 3u + ll;                                   // token + literals + offset
        const uint32_t off = __shfl_sync(kFull, b, 1 + ll) | (__shfl_sync(kFull, b, 2 + ll) << 8);
        uint32_t ml = (tok & 15u) + 4u;
        bool fits = true;
        if ((tok & 15u) == 15u) {
          const unsigned e = __ballot_sync(kFull, b != 255u) & ~((1u << used) - 1u);
          if (e == 0u) fits = false;                               // extension runs past the window
          else {
            const uint32_t p = (uint32_t)__ffs(e) - 1u;
            ml += 255u * (p - used) + __shfl_sync(kFull, b, p);
            used = p + 1u;
          }
        }
        if (fits) {
          if (ll > cap - op || ml > cap - op - ll || off == 0u || off > op + ll) return false;
          if (ul - 1u < ll) out[op + ul - 1u] = (uint8_t)b;       // literals: window lanes 1..ll
          uint8_t* dst = out + op + ll;
          if (!(off <= ll && off <= 8u && (off & (off - 1u)) == 0u)) {
            // general match: copy through memory (fields came from the window, no further input loads)
            __syncwarp();
            warp_match_copy(dst, off, ml, lane);
            __syncwarp();
            op += ll + ml;
            ip += used;
            continue;
          }
          // period (1, 2, 4 or 8 bytes) inside this sequence's literals: expand from the window
          lz_expand_period_from_window(dst, ml, off, b, 1u + ll - off, ul);
          op += ll + ml;
          ip += used;
          continue;
        }
      }
    }
    // ---- generic path: one sequence, field by field
    const uint32_t tok = in[ip++];
    uint32_t ll = tok >> 4;
    if (ll == 15) { if (!lz4_read_ext(in, in_n, ip, ll, lane)) return false; }
    if (ll > in_n - ip || ll > cap - op) return false;
    if (ll) warp_copy<true>(out + op, in + ip, ll, lane);
    ip += ll; op += ll;
    if (ip >= in_n) break;                 // last sequence carries literals only
    if (in_n - ip < 2) return false;
    const uint32_t off = load_u16(in + ip);
    ip += 2;
    uint32_t ml = tok & 15u;
    if (ml == 15) { if (!lz4_read_ext(in, in_n, ip, ml, lane)) return false; }
    if (ml > 0xfffffff0u) return false;
    ml += 4;
    if (off == 0 || off > op || ml > cap - op) return false;
    __syncwarp();                          // prior stores visible to all lanes
    warp_match_copy(out + op, off, ml, lane);
    __syncwarp();
    op += ml;
  }
  *produced = op;
  return true;
}

// ---------------------------------------------------------------------------
// v2 decode (lz_decode.cuh): lane-parallel short-token path + this slow path
// ---------------------------------------------------------------------------
struct Lz4Decode : Lz4Policy {
  __device__ static __forceinline__ bool at_end(const LzState&) { return false; }   // ends inside serial_token
  // one full sequence (token, literals, match), parsed once; 2 = final literals consumed
  __device__ static __forceinline__ int serial_token(LzState& s, int lane) {
    const uint8_t* __restrict__ in = s.in;
    const uint32_t in_n = s.in_n;
    uint32_t ip = s.ip;
    if (ip >= in_n) return -1;
    const uint32_t tok = in[ip++];
    uint32_t ll = tok >> 4;
    if (ll == 15) { if (!lz4_read_ext(in, in_n, ip, ll, lane)) return -1; }
    if (ll > in_n - ip) return -1;
    if ((uint64_t)ll > s.out_cap - s.op) return -1;
    const uint32_t lit_at = ip;
    ip += ll;
    if (ip >= in_n) {                              // last sequence: literals only
      lz_emit_literals(s, in + lit_at, ll, lane);
      s.ip = ip;
      return 2;
    }
    if (in_n - ip < 2) return -1;
    const uint32_t off = load_u16(in + ip);
    ip += 2;
    uint32_t ml = tok & 15u;
    if (ml == 15) { if (!lz4_read_ext(in, in_n, ip, ml, lane)) return -1; }
    ml += 4;
    if (off == 0 || (uint64_t)off > (uint64_t)s.op + ll) return -1;
    if ((uint64_t)ml > s.out_cap - s.op - ll) return -1;
    lz_serial_lookahead<Lz4Policy>(s, ip, lane);
    lz_emit_literals(s, in + lit_at, ll, lane);
    lz_emit_match(s, off, ml, lane);
    s.ip = ip;
    return 1;
  }
};

__device__ __forceinline__ bool lz4_decode_chunk_v2(const uint8_t* in, uint32_t in_n, uint8_t* out,
                                                    uint64_t out_cap, uint32_t* produced,
                                                    uint8_t* ring, uint32_t& tma_parity, int lane, bool allow_direct = true) {
  if (in_n == 0) { *produced = 0; return true; }
  // Adaptive strategy: a chunk that compressed >= 4x is dominated by long matches; the ring /
  // lane-parallel machinery only costs instructions there, so it is decoded by the direct
  // global-memory token loop (16-byte vector copies).  Dense short-token chunks take the
  // lane-parallel path.
  if (allow_direct && out_cap >= 4ull * in_n) return lz4_decode_chunk_direct(in, in_n, out, out_cap, produced, lane);
  LzState s;
  s.in = in; s.in_n = in_n; s.out = out; s.out_cap = out_cap > 0xffffffffull ? 0xffffffffull : out_cap;
  s.ip = 0; s.op = 0; s.flushed = 0; s.ring_lo = 0;
  s.align = (uint32_t)((uintptr_t)out & 15u);
  s.ring = smem_addr(ring);
  s.cur = 0; s.pf_ip = kNoPrefetch; s.parity = tma_parity; s.next = kNextUnknown;
  const bool ok = lz_decode_stream<Lz4Decode>(s, lane);
  tma_parity = s.parity;                 // the barrier outlives the chunk: carry its phase to the next one
  if (!ok) return false;
  *produced = s.op;
  return true;
}

// One block of a linked LZ4 frame (lz4frame_decode.cuh) with the block-parallel decoder: `out` is the frame's first
// output byte, the block starts at position op0 with the op0 bytes before it final in global memory, and out_cap is
// the end of the block's room as a position in the frame.  The decoder's state already keeps positions relative to
// `out` and reads sources below ring_lo from global memory, so the history is only a starting state: op, flushed and
// ring_lo at op0.  Matches may reach back to the frame's first byte.  *produced is the end position.
__device__ __forceinline__ bool lz4_decode_block_v2_linked(const uint8_t* in, uint32_t in_n, uint8_t* out,
                                                           uint64_t out_cap, uint32_t op0, uint32_t* produced,
                                                           uint8_t* ring, uint32_t& tma_parity, int lane) {
  if (in_n == 0) { *produced = op0; return true; }
  LzState s;
  s.in = in; s.in_n = in_n; s.out = out; s.out_cap = out_cap > 0xffffffffull ? 0xffffffffull : out_cap;
  s.ip = 0; s.op = op0; s.flushed = op0; s.ring_lo = op0;
  s.align = (uint32_t)((uintptr_t)out & 15u);
  s.ring = smem_addr(ring);
  s.cur = 0; s.pf_ip = kNoPrefetch; s.parity = tma_parity; s.next = kNextUnknown;
  const bool ok = lz_decode_stream<Lz4Decode>(s, lane);
  tma_parity = s.parity;
  if (!ok) return false;
  *produced = s.op;
  return true;
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
