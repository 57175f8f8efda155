// nvcomp/device/bitcomp.cuh -- warp-level Bitcomp compression, decompression and in-register visiting inside a
// user's own kernels.
//
// This is this library's own interface; the reference ships no device API for Bitcomp.  The streams are the ones the
// batched C API (nvcomp/bitcomp.h) reads and writes: compress_warp writes byte for byte what
// nvcompBatchedBitcompCompressAsync writes, and decompress_warp returns, for every chunk and capacity, the status,
// size and bytes that nvcompBatchedBitcompDecompressAsync returns.  Both run the batched kernels' per-block coder
// (detail/bitcomp_impl.cuh).  for_each_block hands the decoded elements to the caller in registers, one 128-element
// block at a time, so a kernel can consume a compressed column without storing it.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp, decompress_warp and for_each_block:
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - compress_warp's `smem` is this warp's own shared-memory region of kCompressSmemBytes bytes, aligned to
//     kSmemAlignment.  The size is a multiple of kSmemAlignment, so warp w of a CTA can use
//     smem_base + w * kCompressSmemBytes.  decompress_warp and for_each_block need no shared memory.
//   - Alignment follows nvcomp/bitcomp.h: compressed pointers are 8-byte aligned (nvcompBitcompRequiredAlignment)
//     and uncompressed pointers are aligned to the element size.  A misaligned stream, or a decode output not
//     aligned to the stream's element size, is rejected with nvcompErrorCannotDecompress, as the batched decoder
//     rejects it.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n, opts)).  A successful decode writes exactly *actual bytes.
//   - A chunk that cannot be decoded (malformed, truncated, or larger than capacity) returns
//     nvcompErrorCannotDecompress with *actual = 0; no input causes an out-of-bounds access.
//   - Several warps of one CTA may use the API at once on different chunks, each compressing, decompressing or
//     visiting, each compressing warp with its own smem.
#pragma once

#include "nvcomp/bitcomp.h"
#include "nvcomp/device/detail/bitcomp_impl.cuh"

namespace nvcomp {
namespace device {
namespace bitcomp {

// Largest chunk compress_warp accepts (2^24 bytes).
constexpr size_t kMaxChunkBytes = nvcompBitcompCompressionMaxAllowedChunkSize;

// Alignment of each compressing warp's shared-memory region (it holds 64-bit packing words).
constexpr size_t kSmemAlignment = 8;

// Shared memory of one compressing warp: one block's packing words.
constexpr size_t kCompressSmemBytes = detail::kBtcPackWords * sizeof(unsigned long long);
static_assert(kCompressSmemBytes % kSmemAlignment == 0, "warp regions stay aligned");

// Upper bound of one compressed chunk of n bytes; nvcompBatchedBitcompCompressGetMaxOutputChunkSize returns the same.
// 0 for options that chunk does not accept (an unknown type, an algorithm other than 0 and 1) or n > kMaxChunkBytes.
__host__ __device__ inline size_t max_compressed_bytes(size_t n, nvcompBatchedBitcompFormatOpts opts) {
  const size_t ts = detail::btc_type_size(opts.data_type);
  if (ts == 0 || opts.algorithm_type < 0 || opts.algorithm_type > 1 || n > kMaxChunkBytes) return 0;
  const size_t nblocks = (n / ts + detail::kBtcBlock - 1) / detail::kBtcBlock;
  // header + descriptors + per block: 16 bytes of header/mask + 128 elements at full width (+ the trailing-bytes word)
  return 16 + ((2 * nblocks + 7) & ~(size_t)7) + nblocks * (16 + detail::kBtcBlock * ts) + 16;
}

// Uncompressed size recorded in the header of `comp`, or 0 if the header is not valid -- what
// nvcompBatchedBitcompGetDecompressSizeAsync reports for the chunk.  Any thread may call it on its own.
__device__ inline size_t decompressed_size(const void* comp, size_t comp_bytes) {
  detail::BtcHeader h;
  return detail::btc_read_header((const uint8_t*)comp, comp_bytes, h) ? (size_t)h.uncompressed : 0;
}

namespace detail {

// Descriptors g .. g + 31 of the stream: lane i gets block g + i's descriptor `d` and payload offset `off` (the
// first block's payload at base_off); returns the 32 payloads' total size.  `bad` is set on every lane if one of
// the descriptors is rejected.  Blocks past nblocks count as empty.
__device__ __forceinline__ uint32_t group_offsets(const uint8_t* in, const BtcHeader& h, uint32_t g,
                                                  uint32_t base_off, int lane, uint32_t& d, uint32_t& off,
                                                  bool& bad) {
  const uint32_t b = g + (uint32_t)lane;
  d = b < h.nblocks ? ((const uint16_t*)(in + 16))[b] : 0u;
  const uint32_t sz = b < h.nblocks ? btc_block_bytes(h.algo, d) : 0u;
  bad = __any_sync(kFullMask, btc_desc_bad(h.algo, d));
  uint32_t incl = sz;
#pragma unroll
  for (int k = 1; k < 32; k <<= 1) {
    const uint32_t o = __shfl_up_sync(kFullMask, incl, k);
    if (lane >= k) incl += o;
  }
  off = base_off + incl - sz;
  return __shfl_sync(kFullMask, incl, 31);
}

__device__ __forceinline__ uint32_t first_payload(const BtcHeader& h) { return (16u + 2u * h.nblocks + 7u) & ~7u; }

// Every check decompress_warp makes except the capacity and the output alignment: the descriptors, the payload span,
// every sparse mask and the tail word.  Warp-uniform.
__device__ inline bool validate_stream(const uint8_t* in, size_t in_bytes, const BtcHeader& h, int lane) {
  uint32_t base_off = first_payload(h);
  for (uint32_t g = 0; g < h.nblocks; g += 32) {
    uint32_t d, off;
    bool bad;
    const uint32_t total = group_offsets(in, h, g, base_off, lane, d, off, bad);
    if (bad || (uint64_t)base_off + total > in_bytes) return false;
    if (h.algo == 1) {
      // the same check btc_decode_values makes: the mask's popcount is the descriptor's non-zero count
      bool mask_bad = false;
      if (g + (uint32_t)lane < h.nblocks) {
        const uint64_t* p64 = (const uint64_t*)(in + off);
        mask_bad = (uint32_t)(__popcll(p64[0]) + __popcll(p64[1])) != (d & 0xffu);
      }
      if (__any_sync(kFullMask, mask_bad)) return false;
    }
    base_off += total;
  }
  const uint32_t ts = btc_type_size(h.type);
  const uint32_t tail = h.uncompressed - h.uncompressed / ts * ts;
  return !(tail && (uint64_t)base_off + 8u > in_bytes);
}

template <int TS>
__device__ inline bool decompress_blocks(const uint8_t* in, size_t in_bytes, const BtcHeader& h, uint8_t* out,
                                         int lane) {
  using T = typename BtcElem<TS>::T;
  const uint32_t n_elems = h.uncompressed / TS;
  uint32_t base_off = first_payload(h);
  for (uint32_t g = 0; g < h.nblocks; g += 32) {
    uint32_t d, off;
    bool bad;
    const uint32_t total = group_offsets(in, h, g, base_off, lane, d, off, bad);
    if (bad || (uint64_t)base_off + total > in_bytes) return false;
    const uint32_t nb = min(32u, h.nblocks - g);
    bool good = true;
    for (uint32_t j = 0; j < nb; ++j) {
      const uint32_t e0 = (g + j) * kBtcBlock;
      const uint32_t o = __shfl_sync(kFullMask, off, j), dj = __shfl_sync(kFullMask, d, j);
      good &= btc_decode_block<TS>(h.algo, dj, in + o, (T*)out + e0, min(kBtcBlock, n_elems - e0), lane);
    }
    if (!good) return false;
    base_off += total;
  }
  // trailing bytes of a chunk whose length is not a multiple of the element size: stored verbatim
  const uint32_t tail = h.uncompressed - n_elems * TS;
  if (tail) {
    if ((uint64_t)base_off + 8u > in_bytes) return false;
    if ((uint32_t)lane < tail) out[n_elems * TS + lane] = in[base_off + lane];
  }
  return true;
}

template <int TS>
__device__ inline void compress_blocks(const uint8_t* in, uint32_t n_bytes, uint8_t* out, size_t* comp_bytes,
                                       int algo, int type, unsigned long long* words, int lane) {
  using T = typename BtcElem<TS>::T;
  const uint32_t n_elems = n_bytes / TS;
  const uint32_t nblocks = (n_elems + kBtcBlock - 1) / kBtcBlock;
  if (lane == 0) {
    uint32_t* hw = (uint32_t*)out;
    hw[0] = kBtcMagic; hw[1] = (uint32_t)algo | ((uint32_t)type << 8); hw[2] = n_bytes; hw[3] = nblocks;
  }
  uint16_t* desc = (uint16_t*)(out + 16);
  uint32_t off = (16u + 2u * nblocks + 7u) & ~7u;
  // clear the descriptor pad so the stream is deterministic
  if (lane < 4) { const uint32_t i = nblocks + lane; if (16u + 2u * i < off) desc[i] = 0; }
  // one pass: a block's payload size is known as soon as it is analysed, so it is packed at the running offset
  for (uint32_t b = 0; b < nblocks; ++b) {
    const uint32_t e0 = b * kBtcBlock;
    const uint32_t nv = min(kBtcBlock, n_elems - e0);
    const uint32_t d = btc_analyse_block<TS>(algo, (const T*)in + e0, nv, lane);
    if (lane == 0) desc[b] = (uint16_t)d;
    btc_pack_block<TS>(algo, d, (const T*)in + e0, nv, out + off, words, lane);
    off += btc_block_bytes(algo, d);
  }
  const uint32_t tail = n_bytes - n_elems * TS;
  if (tail && lane < 8) out[off + lane] = (uint32_t)lane < tail ? in[n_elems * TS + lane] : (uint8_t)0;
  if (lane == 0 && comp_bytes) *comp_bytes = off + (tail ? 8u : 0u);
}

template <class T>
__device__ __forceinline__ T bit_cast_elem(uint64_t v) {
  const typename BtcElem<sizeof(T)>::T u = (typename BtcElem<sizeof(T)>::T)v;
  T t;
  __builtin_memcpy(&t, &u, sizeof(T));
  return t;
}

}  // namespace detail

// Decode the comp_bytes-byte stream at `comp` into [out, out + capacity).  Warp-collective (see above).  Block
// payload offsets come from a warp scan over 32 descriptors at a time.
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual) {
  using namespace detail;
  const int lane = lane_id();
  const uint8_t* in = (const uint8_t*)comp;
  uint8_t* o = (uint8_t*)out;
  BtcHeader h;
  bool ok = btc_read_header(in, comp_bytes, h);
  const uint32_t ts = ok ? btc_type_size(h.type) : 1;
  if (ok && (h.uncompressed > capacity || ((uintptr_t)o & (ts - 1)))) ok = false;
  if (ok) {
    switch (ts) {
      case 1: ok = decompress_blocks<1>(in, comp_bytes, h, o, lane); break;
      case 2: ok = decompress_blocks<2>(in, comp_bytes, h, o, lane); break;
      case 4: ok = decompress_blocks<4>(in, comp_bytes, h, o, lane); break;
      default: ok = decompress_blocks<8>(in, comp_bytes, h, o, lane); break;
    }
  }
  if (lane == 0 && actual) *actual = ok ? (size_t)h.uncompressed : 0;
  __syncwarp();
  return ok ? nvcompSuccess : nvcompErrorCannotDecompress;
}

// Compress the n_bytes bytes at `in` (aligned to the element size) into the stream at `out` (8-byte aligned,
// max_compressed_bytes(n_bytes, opts) bytes) and its size into *comp_bytes.  Warp-collective (see above).  Options
// the batched call rejects return nvcompErrorInvalidValue, n_bytes > kMaxChunkBytes returns
// nvcompErrorChunkSizeTooLarge; both with *comp_bytes = 0 and nothing else written.
__device__ inline nvcompStatus_t compress_warp(const void* in, size_t n_bytes, void* out, size_t* comp_bytes,
                                               nvcompBatchedBitcompFormatOpts opts, void* smem) {
  using namespace detail;
  const int lane = lane_id();
  const uint32_t ts = btc_type_size(opts.data_type);
  nvcompStatus_t st = nvcompSuccess;
  if (ts == 0 || opts.algorithm_type < 0 || opts.algorithm_type > 1) st = nvcompErrorInvalidValue;
  else if (n_bytes > kMaxChunkBytes) st = nvcompErrorChunkSizeTooLarge;
  if (st != nvcompSuccess) {
    if (lane == 0 && comp_bytes) *comp_bytes = 0;
    return st;
  }
  const uint8_t* i8 = (const uint8_t*)in;
  uint8_t* o8 = (uint8_t*)out;
  unsigned long long* words = (unsigned long long*)smem;
  const int algo = opts.algorithm_type, type = (int)opts.data_type;
  switch (ts) {
    case 1: compress_blocks<1>(i8, (uint32_t)n_bytes, o8, comp_bytes, algo, type, words, lane); break;
    case 2: compress_blocks<2>(i8, (uint32_t)n_bytes, o8, comp_bytes, algo, type, words, lane); break;
    case 4: compress_blocks<4>(i8, (uint32_t)n_bytes, o8, comp_bytes, algo, type, words, lane); break;
    default: compress_blocks<8>(i8, (uint32_t)n_bytes, o8, comp_bytes, algo, type, words, lane); break;
  }
  __syncwarp();
  return nvcompSuccess;
}

// Visit the decoded elements of the stream at `comp` in registers, one 128-element block at a time, in stream order.
// Warp-collective (see above).
//
// The whole stream is validated first -- the header, every descriptor, the payload span, every sparse mask and the
// tail word, i.e. everything decompress_warp checks except the capacity and the output alignment -- so `f` is either
// called for every block or never.  Then, for each block, every lane calls
//     f(const T (&v)[4], uint32_t first_element, uint32_t valid)
// with its four consecutive elements v[0..3] = elements first_element .. first_element + 3 of the chunk, of which
// the first `valid` (0..4) exist; the others are unspecified.  first_element is block * 128 + 4 * lane.  The values
// stay in registers and nothing is stored; all 32 lanes call f together, so f may use warp intrinsics.
//
// Returns nvcompSuccess exactly when decompress_warp would succeed with unlimited capacity, and otherwise
// nvcompErrorCannotDecompress without calling f.  A stream whose element size is not sizeof(T) returns
// nvcompErrorInvalidValue without calling f (a header that is not valid at all returns nvcompErrorCannotDecompress).
// T is any 1-, 2-, 4- or 8-byte trivially copyable type; the element's bits are copied into it.  A chunk whose length
// is not a multiple of the element size keeps its last bytes in the stream's tail word, and f is not given them.
template <class T, class F>
__device__ inline nvcompStatus_t for_each_block(const void* comp, size_t comp_bytes, F&& f) {
  using namespace detail;
  static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8, "element of 1, 2, 4 or 8 bytes");
  constexpr int TS = (int)sizeof(T);
  const int lane = lane_id();
  const uint8_t* in = (const uint8_t*)comp;
  BtcHeader h;
  if (!btc_read_header(in, comp_bytes, h)) return nvcompErrorCannotDecompress;
  if (btc_type_size(h.type) != sizeof(T)) return nvcompErrorInvalidValue;
  if (!validate_stream(in, comp_bytes, h, lane)) return nvcompErrorCannotDecompress;
  const uint32_t n_elems = h.uncompressed / TS;
  uint32_t base_off = first_payload(h);
  for (uint32_t g = 0; g < h.nblocks; g += 32) {
    uint32_t d, off;
    bool bad;
    const uint32_t total = group_offsets(in, h, g, base_off, lane, d, off, bad);
    const uint32_t nb = min(32u, h.nblocks - g);
    for (uint32_t j = 0; j < nb; ++j) {
      const uint32_t o = __shfl_sync(kFullMask, off, j), dj = __shfl_sync(kFullMask, d, j);
      uint64_t v[4];
      btc_decode_values<TS>(h.algo, dj, in + o, lane, v);
      const T t[4] = {bit_cast_elem<T>(v[0]), bit_cast_elem<T>(v[1]), bit_cast_elem<T>(v[2]), bit_cast_elem<T>(v[3])};
      const uint32_t first = (g + j) * kBtcBlock + 4u * (uint32_t)lane;
      const uint32_t valid = first < n_elems ? min(4u, n_elems - first) : 0u;
      f(t, first, valid);
    }
    base_off += total;
  }
  return nvcompSuccess;
}

}  // namespace bitcomp
}  // namespace device
}  // namespace nvcomp
