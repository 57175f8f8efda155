// nvcomp/device/detail/lz4frame_decode.cuh -- one warp walks one chunk of LZ4 frames (the LZ4 frame format, magic
// 0x184D2204, as liblz4's LZ4F_* API writes it): headers, block framing, skippable frames and the XXH32 checksums.
// Compressed blocks go to the LZ4 block bodies of lz4_decode.cuh.  The batched kernel is in
// nvcomp_b200/csrc/lz4frame.cu, the device API in nvcomp/device/lz4frame.cuh; include/nvcomp/lz4frame.h states the
// contract.
//
// A chunk is zero or more LZ4 frames and skippable frames (magic 0x184D2A50-5F) back to back, filling the chunk
// exactly.  Inside a frame the checks run in liblz4 1.9.4's order, so the first failing one decides the status:
//   header     magic; FLG reserved bit 1 and version 01; then, with the whole descriptor present, BD reserved bit 7,
//              block-size ID 4-7, BD reserved bits 0-3, and the header checksum (XXH32(descriptor) >> 8) & 0xFF.
//              The optional content size (8 bytes) and dictID (4 bytes) are read.
//   blocks     a 4-byte size; 0 (high bit ignored) is the EndMark; more than the maximum block size is rejected.  The
//              high bit marks an uncompressed block: its bytes are copied, then its optional XXH32 is checked (liblz4
//              writes the bytes before it sees the checksum).  A compressed block's optional XXH32 over its stored
//              bytes is checked before the block is decoded.  No block decodes to more than the maximum block size.
//   end        a non-zero content size must equal the frame's decoded size (liblz4 treats 0 as "not given"); then
//              the optional content XXH32 over the frame's decoded bytes.
// Match reach: a linked frame's blocks may reach back into the earlier blocks of their frame, never before the
// frame's first output byte; an independent frame's blocks only into themselves.
//
// kCount is the size query: the same walk with stores off.  It checks everything except the content checksum, which
// needs the decoded bytes.
#pragma once

#include "nvcomp/device/detail/lz4_decode.cuh"
#include "nvcomp/device/detail/lz_decode.cuh"
#include "nvcomp/device/detail/xxhash32.cuh"

namespace nvcomp {
namespace device {
namespace lz4frame {
namespace detail {

constexpr uint32_t kLz4fMagic = 0x184D2204u;
constexpr uint32_t kLz4fSkippableMagic = 0x184D2A50u;   // low 4 bits free
constexpr uint32_t kLz4fSkippableMask = 0xFFFFFFF0u;
constexpr uint32_t kLz4fMinHeader = 7;                  // magic, FLG, BD, HC

// results of lz4f_chunk
constexpr int kLz4fOk = 0, kLz4fBad = 1, kLz4fBadChecksum = 2;

__device__ __forceinline__ uint32_t lz4f_le32(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// One compressed block of a frame: `fout` is the frame's first output byte, the block starts at frame position pos,
// and may produce at most `room` bytes.  Linked frames reach back to fout, independent ones only to fout + pos.
// Returns false on a malformed block; *end receives the block's end position in the frame.  The body is the one the
// LZ4 device API picks for the block (lz_chunk_is_light on the block's room and stored size).
template <bool kCount>
__device__ __forceinline__ bool lz4f_block(const uint8_t* in, uint32_t n, uint8_t* fout, uint32_t pos, uint32_t room,
                                           bool linked, uint32_t* end, uint8_t* ring, uint32_t& parity, int lane) {
  using namespace lz::detail;
  uint32_t e = 0;
  bool ok;
  if (kCount) {
    ok = linked ? lz4_walk_chunk<true>(in, n, &e, lane, pos) : lz4_walk_chunk(in, n, &e, lane);
    if (!linked) e += pos;
    ok = ok && e - pos <= room;
  } else if (linked) {
    const uint64_t cap = (uint64_t)pos + room;
    ok = lz_chunk_is_light((uint64_t)room, (uint64_t)n)
             ? lz4_decode_chunk_direct<true>(in, n, fout, cap, &e, lane, pos)
             : lz4_decode_block_v2_linked(in, n, fout, cap, pos, &e, ring, parity, lane);
  } else {
    ok = lz_chunk_is_light((uint64_t)room, (uint64_t)n)
             ? lz4_decode_chunk_direct(in, n, fout + pos, (uint64_t)room, &e, lane)
             : lz4_decode_chunk_v2(in, n, fout + pos, (uint64_t)room, &e, ring, parity, lane, false);
    e += pos;
  }
  *end = e;
  return ok;
}

// Decode (kCount: walk) the chunk in[0, n) into out[0, cap).  *produced receives the decoded total on kLz4fOk.
// `ring` is the warp's kLzWarpSmem region with an initialised mbarrier whose phase `parity` carries across calls.
// The caller guarantees n < 2^32 and cap < 2^32; kCount passes out = nullptr and cap = 0xffffffff.
template <bool kCount>
__device__ __forceinline__ int lz4f_chunk(const uint8_t* __restrict__ in, uint32_t n, uint8_t* out, uint32_t cap,
                                          uint32_t* produced, uint8_t* ring, uint32_t& parity, int lane) {
  using namespace lz::detail;
  uint32_t ip = 0, op = 0;
  while (ip < n) {
    const uint32_t left = n - ip;
    if (left < kLz4fMinHeader) return kLz4fBad;                 // liblz4 reads no frame type from fewer bytes
    const uint32_t magic = lz4f_le32(in + ip);
    if ((magic & kLz4fSkippableMask) == kLz4fSkippableMagic) {
      if (left < 8) return kLz4fBad;
      const uint32_t sz = lz4f_le32(in + ip + 4);
      if (sz > left - 8) return kLz4fBad;
      ip += 8 + sz;
      continue;
    }
    if (magic != kLz4fMagic) return kLz4fBad;                   // legacy frames (0x184C2102) included
    const uint32_t flg = in[ip + 4];
    if ((flg >> 1) & 1u) return kLz4fBad;                        // reserved
    if ((flg >> 6) != 1u) return kLz4fBad;                       // version 01
    const uint32_t hsize = kLz4fMinHeader + ((flg & 8u) ? 8u : 0u) + ((flg & 1u) ? 4u : 0u);
    if (left < hsize) return kLz4fBad;
    const uint32_t bd = in[ip + 5];
    if (bd & 0x80u) return kLz4fBad;                             // reserved
    const uint32_t bsid = (bd >> 4) & 7u;
    if (bsid < 4u) return kLz4fBad;
    if (bd & 0x0Fu) return kLz4fBad;                             // reserved
    const uint32_t hc = (xxh32_warp(in + ip + 4, hsize - 5, lane) >> 8) & 0xFFu;
    if (hc != in[ip + hsize - 1]) return kLz4fBadChecksum;
    uint64_t content_size = 0;
    if (flg & 8u) content_size = (uint64_t)lz4f_le32(in + ip + 6) | ((uint64_t)lz4f_le32(in + ip + 10) << 32);
    // (the dictID, when present, is read by skipping it: dictionaries are not supported, and liblz4's LZ4F_decompress
    // decodes such a frame without one)
    const bool linked = !(flg & 0x20u), block_sum = flg & 0x10u, content_sum = flg & 4u;
    const uint32_t max_block = 1u << (8 + 2 * bsid);              // 64 KB, 256 KB, 1 MB, 4 MB
    const uint32_t sum_bytes = block_sum ? 4u : 0u;
    ip += hsize;
    const uint32_t fstart = op;
    uint8_t* const fout = kCount ? nullptr : out + fstart;
    while (true) {
      if (n - ip < 4) return kLz4fBad;
      const uint32_t bh = lz4f_le32(in + ip);
      const uint32_t bsize = bh & 0x7FFFFFFFu;
      ip += 4;
      if (bsize == 0) break;                                     // EndMark
      if (bsize > max_block) return kLz4fBad;
      if (bsize > n - ip || sum_bytes > n - ip - bsize) return kLz4fBad;
      const uint8_t* const blk = in + ip;
      if (bh & 0x80000000u) {
        // uncompressed: liblz4 writes the bytes, then checks the block checksum
        if (bsize > cap - op) return kLz4fBad;
        if (!kCount) {
          warp_copy<true>(out + op, blk, bsize, lane);
          __syncwarp();
        }
        if (block_sum && xxh32_warp(blk, bsize, lane) != lz4f_le32(blk + bsize)) return kLz4fBadChecksum;
        op += bsize;
      } else {
        // compressed: the checksum of the stored bytes first, then the block
        if (block_sum && xxh32_warp(blk, bsize, lane) != lz4f_le32(blk + bsize)) return kLz4fBadChecksum;
        const uint32_t room = min(cap - op, max_block);
        uint32_t end = 0;
        if (!lz4f_block<kCount>(blk, bsize, fout, op - fstart, room, linked, &end, ring, parity, lane)) return kLz4fBad;
        op = fstart + end;
        __syncwarp();
      }
      ip += bsize + sum_bytes;
    }
    if (content_size != 0 && content_size != (uint64_t)(op - fstart)) return kLz4fBad;
    if (content_sum) {
      if (n - ip < 4) return kLz4fBad;
      if (!kCount && xxh32_warp(fout, op - fstart, lane) != lz4f_le32(in + ip)) return kLz4fBadChecksum;
      ip += 4;
    }
  }
  *produced = op;
  return kLz4fOk;
}

}  // namespace detail
}  // namespace lz4frame
}  // namespace device
}  // namespace nvcomp
