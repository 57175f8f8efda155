// nvcomp/device/ans.cuh -- warp-level ANS compression and decompression inside a user's own kernels.
//
// This is this library's own interface: nvCOMP 3.0 ships a device-side ANS API, but no header or caller of it
// is available to pin its names, so nothing here claims them.  The streams are the ones the batched C API
// (nvcomp/ans.h) reads and writes: compress_warp writes byte for byte what nvcompBatchedANSCompressAsync writes,
// and decompress_warp returns, for every chunk and capacity, the status, size and bytes that
// nvcompBatchedANSDecompressAsync returns.  Both run the same device code as those kernels
// (detail/ans_impl.cuh).
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp and decompress_warp:
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - `smem` is this warp's own shared-memory region of kDecompressSmemBytes / kCompressSmemBytes bytes, aligned
//     to kSmemAlignment.  Both sizes are multiples of kSmemAlignment, so warp w of a CTA can use
//     smem_base + w * size.  `tmp` is this warp's own global scratch of compress_tmp_bytes() bytes, 4-byte
//     aligned.  Compressed streams, `out`, `in` and `tmp` are global memory.
//   - Alignment follows nvcomp/ans.h: compressed pointers are 8-byte aligned (nvcompANSRequiredAlignment).  A
//     misaligned stream is rejected with nvcompErrorCannotDecompress, as the batched decoder rejects it.
//     Uncompressed pointers may have any alignment.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n)).  A successful decode writes exactly *actual bytes.
//   - A chunk that cannot be decoded (malformed, truncated, or larger than capacity) returns
//     nvcompErrorCannotDecompress with *actual = 0; no input causes an out-of-bounds access.
//   - n > kMaxChunkBytes returns nvcompErrorChunkSizeTooLarge with *comp_bytes = 0 and writes nothing else.
//   - Several warps of one CTA may use the API at once on different chunks, some compressing and some
//     decompressing, each with its own smem and tmp.
#pragma once

#include "nvcomp/ans.h"
#include "nvcomp/device/detail/ans_impl.cuh"

namespace nvcomp {
namespace device {
namespace ans {

// Largest chunk either function accepts (2^24 bytes).
constexpr size_t kMaxChunkBytes = nvcompANSCompressionMaxAllowedChunkSize;

// Alignment of each warp's shared-memory region: the decoder's cp.async word ring is addressed as
// (offset & 1023) | base, so it needs 1 KB alignment.
constexpr size_t kSmemAlignment = detail::kRingBytes;

// Shared memory of one decompressing warp: the word ring (1 KB), the 4096-entry decode LUT (16 KB) and the 257
// cumulative frequencies, rounded up to kSmemAlignment (19 KB).
constexpr size_t kDecompressSmemBytes =
    (detail::kRingBytes + 4 * detail::kM + 4 * 257 + kSmemAlignment - 1) / kSmemAlignment * kSmemAlignment;

// Shared memory of one compressing warp: the histogram and the frequency and cumulative tables (2 KB).
constexpr size_t kCompressSmemBytes = (4 * 256 + 2 * 256 + 2 * 256 + kSmemAlignment - 1) / kSmemAlignment * kSmemAlignment;

// Upper bound of one compressed chunk of n bytes, a multiple of 8; nvcompBatchedANSCompressGetMaxOutputChunkSize
// returns the same.  The encoder stores a chunk raw (16 + n bytes) whenever rANS would be larger, but the rANS
// attempt is laid out in the header area first.
__host__ __device__ constexpr size_t max_compressed_bytes(size_t n) {
  return (16 + 512 + 4 * ((n + detail::kSeg - 1) / detail::kSeg + 1) + n + 16 + 7) & ~(size_t)7;
}

// Global scratch one compressing warp needs: one segment's worth, since segments are encoded one at a time.
// Independent of the chunk size.
__host__ __device__ constexpr size_t compress_tmp_bytes() { return detail::scratch_per_seg(); }

// Uncompressed size recorded in the header of `comp`, or 0 if the header is not valid -- what
// nvcompBatchedANSGetDecompressSizeAsync reports for the chunk.  Any thread may call it on its own.
__device__ inline size_t decompressed_size(const void* comp, size_t comp_bytes) {
  detail::Header h;
  return detail::read_header((const uint8_t*)comp, comp_bytes, h) ? (size_t)h.n : 0;
}

// Decode the comp_bytes-byte stream at `comp` into [out, out + capacity).  Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem) {
  using namespace detail;
  const int lane = threadIdx.x & 31;
  const uint8_t* in = (const uint8_t*)comp;
  uint8_t* o = (uint8_t*)out;
  uint8_t* s = (uint8_t*)smem;
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(s);
  uint32_t* s_lut = (uint32_t*)(s + kRingBytes);
  uint32_t* s_cum = s_lut + kM;
  Header h;
  bool ok = read_header(in, comp_bytes, h) && h.n <= capacity;
  if (ok && h.mode == 1) {
    for (uint32_t i = lane; i < h.n; i += 32) o[i] = in[16 + i];
  } else if (ok && h.mode == 2) {
    const uint8_t sym = in[16];
    for (uint32_t i = lane; i < h.n; i += 32) o[i] = sym;
  } else if (ok) {
    ok = cum_scan((const uint16_t*)(in + 16), s_cum, lane);
    __syncwarp();
    if (ok) {
      bool lut_ok = true;
      for (uint32_t sym0 = 0; sym0 < 256; sym0 += 32) lut_ok &= lut_fill32(s_cum, s_lut, sym0, lane);
      ok = __all_sync(kFullMask, lut_ok);
      __syncwarp();
    }
    if (ok) {
      // every segment is decoded even after one fails, as the batched decoder does
      const uint32_t lut = (uint32_t)__cvta_generic_to_shared(s_lut);
      for (uint32_t sg = 0; sg < h.nseg; ++sg) ok &= decode_segment(in, comp_bytes, h.n, sg, o, lut, ring, lane);
    }
  }
  if (lane == 0 && actual) *actual = ok ? (size_t)h.n : 0;
  return ok ? nvcompSuccess : nvcompErrorCannotDecompress;
}

// Compress the n bytes at `in` into the stream at `out` (8-byte aligned, max_compressed_bytes(n) bytes) and its
// size into *comp_bytes.  Warp-collective (see above).
__device__ inline nvcompStatus_t compress_warp(const void* in_ptr, size_t n_bytes, void* out_ptr, size_t* comp_bytes,
                                               void* smem, void* tmp) {
  using namespace detail;
  const int lane = threadIdx.x & 31;
  if (n_bytes > kMaxChunkBytes) {
    if (lane == 0 && comp_bytes) *comp_bytes = 0;
    return nvcompErrorChunkSizeTooLarge;
  }
  const uint8_t* in = (const uint8_t*)in_ptr;
  uint8_t* out = (uint8_t*)out_ptr;
  uint8_t* scratch = (uint8_t*)tmp;
  const uint32_t n = (uint32_t)n_bytes;
  uint32_t* s_hist = (uint32_t*)smem;
  uint16_t* s_freq = (uint16_t*)(s_hist + 256);
  uint16_t* s_cum = s_freq + 256;
  hist_clear(s_hist, lane, 32);
  __syncwarp();
  hist_add(in, n, s_hist, lane, 32);
  __syncwarp();
  uint32_t mode = 0;
  if (lane == 0) mode = normalize(s_hist, s_freq, s_cum, n);
  mode = __shfl_sync(kFullMask, mode, 0);
  __syncwarp();
  const uint32_t nseg = (n + kSeg - 1) / kSeg;
  uint32_t total = 0;
  if (mode == 0) {
    // Segments are encoded in order, so each one's offset is known when it is encoded.  The stream is stored raw
    // as soon as the offsets reach 16 + n; every segment copied before that lies below 16 + n, where the raw
    // bytes go.
    uint32_t off = header_bytes(nseg);
    uint32_t* seg_off = (uint32_t*)(out + 16 + 512);
    for (uint32_t sg = 0; sg < nseg && mode == 0; ++sg) {
      const uint32_t begin = sg * kSeg;
      const uint32_t nw = encode_segment(in + begin, min(kSeg, n - begin), s_freq, s_cum, scratch, lane);
      const uint32_t next = off + seg_bytes(nw);
      if (next >= 16u + n) {
        mode = 1;
      } else {
        if (lane == 0) seg_off[sg] = off;
        copy_segment(out + off, scratch, nw, lane, 32);
        __syncwarp();                 // the scratch is reused by the next segment
        off = next;
      }
    }
    if (mode == 0) {
      if (lane == 0) seg_off[nseg] = off;
      write_freq(out, s_freq, lane, 32);
      total = off;
    }
  }
  if (lane == 0) write_header(out, n, mode, nseg);
  if (mode == 1) {
    copy_stored(out, in, n, lane, 32);
    total = 16u + n;
  } else if (mode == 2) {
    if (lane == 0) out[16] = in[0];
    total = 17;
  }
  if (lane == 0 && comp_bytes) *comp_bytes = total;
  __syncwarp();
  return nvcompSuccess;
}

}  // namespace ans
}  // namespace device
}  // namespace nvcomp
