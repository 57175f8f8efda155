// nvcomp/device/cascaded.cuh -- warp-level Cascaded compression, decompression and in-register visiting inside a
// user's own kernels.
//
// This is this library's own interface; the reference ships no device API for Cascaded.  The streams are the ones
// the batched C API (nvcomp/cascaded.h) reads and writes: compress_warp writes byte for byte what
// nvcompBatchedCascadedCompressAsync writes, and decompress_warp returns, for every chunk and capacity, the status,
// size and bytes that nvcompBatchedCascadedDecompressAsync returns.  Both run the batched kernels' per-partition coder
// (detail/cascaded_impl.cuh).  for_each_block hands the decoded elements to the caller in registers, one block of up
// to 128 elements at a time, so a kernel can consume a compressed column without storing it.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of compress_warp, decompress_warp and for_each_block:
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual / *comp_bytes is written once (by lane 0; either pointer may be null).
//   - `smem` is this warp's own shared-memory region, aligned to kSmemAlignment: compress_smem_bytes(opts) bytes for
//     compress_warp, smem_bytes for decompress_warp and for_each_block.  A stream decodes in a region of
//     decompress_smem_bytes(opts) bytes for the options it was written with, and in any stream's
//     kMaxDecompressSmemBytes.  All sizes are multiples of kSmemAlignment, so warp w of a CTA can use
//     smem_base + w * size.
//   - Alignment follows nvcomp/cascaded.h: compressed pointers are 8-byte aligned and uncompressed pointers are
//     aligned to the element size.  A misaligned stream, or a decode output not aligned to the stream's element
//     size, is rejected with nvcompErrorCannotDecompress, as the batched decoder rejects it.
//   - decompress_warp writes only inside [out, out + capacity), compress_warp only inside
//     [out, out + max_compressed_bytes(n, opts)).  A successful decode writes exactly *actual bytes.
//   - A chunk that cannot be decoded (malformed, truncated, or larger than capacity) returns
//     nvcompErrorCannotDecompress with *actual = 0; no input causes an out-of-bounds access.  A valid header whose
//     partitions need more than smem_bytes returns nvcompErrorInvalidValue with *actual = 0 and nothing written.
//   - Several warps of one CTA may use the API at once on different chunks, each compressing, decompressing or
//     visiting, each with its own smem.
#pragma once

#include "nvcomp/cascaded.h"
#include "nvcomp/device/detail/cascaded_impl.cuh"

namespace nvcomp {
namespace device {
namespace cascaded {

// Largest chunk compress_warp accepts (2^24 bytes).
constexpr size_t kMaxChunkBytes = nvcompCascadedCompressionMaxAllowedChunkSize;

// Alignment of each warp's shared-memory region (the decoder uses 16-byte vector accesses on it).
constexpr size_t kSmemAlignment = 16;

// Shared memory decompress_warp and for_each_block need for any legal stream: a 16 KB partition of 1-byte elements
// with more than one layer pair.
constexpr size_t kMaxDecompressSmemBytes = detail::casc_decode_smem_bytes(detail::kCascMaxPart, 0, true);
static_assert(kMaxDecompressSmemBytes % kSmemAlignment == 0, "warp regions stay aligned");

// Upper bound of one compressed chunk of n bytes; nvcompBatchedCascadedCompressGetMaxOutputChunkSize returns the
// same.  0 for options that call rejects or n > kMaxChunkBytes.
__host__ __device__ inline size_t max_compressed_bytes(size_t n, nvcompBatchedCascadedOpts_t opts) {
  if (detail::casc_check_opts(opts) != nvcompSuccess || n > kMaxChunkBytes) return 0;
  return detail::casc_max_output_bytes(n, opts);
}

// Shared memory of one compressing warp: the batched encoder's per-warp region.  0 for invalid options.
__host__ __device__ inline size_t compress_smem_bytes(nvcompBatchedCascadedOpts_t opts) {
  if (detail::casc_check_opts(opts) != nvcompSuccess) return 0;
  return (detail::kCascCompSmemPerWarp((uint32_t)opts.chunk_size) + 15u) & ~15u;
}

// Shared memory of one decompressing or visiting warp for streams written with `opts`: the batched decoder's
// per-warp region for that partition size, element type and layer count.  0 for invalid options.
__host__ __device__ inline size_t decompress_smem_bytes(nvcompBatchedCascadedOpts_t opts) {
  if (detail::casc_check_opts(opts) != nvcompSuccess) return 0;
  const uint32_t ts = detail::casc_type_size(opts.type);
  const uint32_t shift = ts == 1 ? 0u : ts == 2 ? 1u : ts == 4 ? 2u : 3u;
  return detail::casc_decode_smem_bytes((uint32_t)opts.chunk_size, shift,
                                        (opts.num_RLEs > opts.num_deltas ? opts.num_RLEs : opts.num_deltas) > 1);
}

// Uncompressed size recorded in the header of `comp`, or 0 if the header is not valid -- what
// nvcompBatchedCascadedGetDecompressSizeAsync reports for the chunk.  Any thread may call it on its own.
__device__ inline size_t decompressed_size(const void* comp, size_t comp_bytes) {
  detail::CascHeader h;
  return detail::casc_read_header((const uint8_t*)comp, comp_bytes, h) ? (size_t)h.uncompressed : 0;
}

namespace detail {

__device__ __forceinline__ uint32_t header_smem_bytes(const CascHeader& h) {
  const uint32_t ts = casc_type_size(h.type);
  return casc_decode_smem_bytes(h.part_bytes, (uint32_t)(__ffs((int)ts) - 1), (h.R > h.D ? h.R : h.D) > 1);
}

// Walk the partitions of a stream whose header h is valid, in order, through casc_decode_part in MODE, and check the
// trailing word (kCascDecode also copies its bytes).  kCascVisit calls f(v, first_element, valid) with chunk element
// indices.  Stops at the first partition that fails.  Warp-uniform; every partition ends with a __syncwarp, so the
// warp's region is free again when the walk returns.
template <int TS, int MODE, class F>
__device__ inline bool walk_chunk(const uint8_t* in, size_t in_bytes, const CascHeader& h, uint8_t* out, uint8_t* sm,
                                  const F& f, int lane) {
  using T = typename Elem<TS>::T;
  const uint32_t* part_off = (const uint32_t*)(in + 20);
  const uint32_t P = h.part_bytes;
  const bool two_bufs = (h.R > h.D ? h.R : h.D) > 1;
  const uint32_t whole = h.uncompressed - h.uncompressed % TS;
  for (uint32_t p = 0; p < h.num_parts; ++p) {
    const uint32_t o0 = part_off[p], o1 = part_off[p + 1];
    if (!casc_part_span_ok(o0, o1, in_bytes)) return false;
    const uint32_t begin = p * P;
    const uint32_t n = min(P, whole - begin) / TS;
    const uint32_t e0 = begin / TS;
    const auto g = [&](const T (&v)[4], uint32_t k, uint32_t valid) { f(v, e0 + k, valid); };
    const bool ok = casc_decode_part<TS, MODE>(in + o0, o1 - o0, out + begin, n, h.R, h.D, sm, P, two_bufs, lane, g);
    // the partition's last reads of the region (write-out, gather, visit) have lane-dependent trip counts, and the
    // next partition -- or the caller's next call -- starts by storing its header window there
    __syncwarp();
    if (!ok) return false;
  }
  // trailing bytes of a chunk whose length is not a multiple of the element size
  const uint32_t tail = h.uncompressed % TS;
  if (tail) {
    const uint32_t to = part_off[h.num_parts];
    if ((uint64_t)to + 8u > in_bytes) return false;
    if (MODE == kCascDecode && (uint32_t)lane < tail) out[whole + lane] = in[to + lane];
  }
  return true;
}

template <int MODE, class F>
__device__ __forceinline__ bool walk_chunk_ts(uint32_t ts, const uint8_t* in, size_t in_bytes, const CascHeader& h,
                                              uint8_t* out, uint8_t* sm, const F& f, int lane) {
  switch (ts) {
    case 1: return walk_chunk<1, MODE>(in, in_bytes, h, out, sm, f, lane);
    case 2: return walk_chunk<2, MODE>(in, in_bytes, h, out, sm, f, lane);
    case 4: return walk_chunk<4, MODE>(in, in_bytes, h, out, sm, f, lane);
    default: return walk_chunk<8, MODE>(in, in_bytes, h, out, sm, f, lane);
  }
}

// One chunk with one warp, partitions in order: the batched encoder's stream.  opts are valid, n <= kMaxChunkBytes.
// The chunk framing (header words, offset table, pad word, trailing word) is the same as cascaded_compress_kernel's
// per-chunk loop in nvcomp_b200/csrc/cascaded.cu; a change to the stream format changes both.  (Calling one shared
// function from the batched kernel changed its machine code, so the loop is kept twice.)
__device__ inline void compress_chunk(const uint8_t* in, uint32_t n, uint8_t* out, size_t* comp_bytes,
                                      const nvcompBatchedCascadedOpts_t& opts, uint8_t* sm, int lane) {
  const uint32_t ts = casc_type_size(opts.type);
  const uint32_t P = (uint32_t)opts.chunk_size;
  const uint32_t tail = n % ts, whole = n - tail;
  const uint32_t num_parts = (whole + P - 1) / P;
  if (lane == 0) {
    uint32_t* hw = (uint32_t*)out;
    hw[0] = kCascMagic;
    hw[1] = (uint32_t)(opts.type & 0xff) | ((uint32_t)opts.num_RLEs << 8) | ((uint32_t)opts.num_deltas << 16)
            | ((uint32_t)(opts.use_bp ? 1 : 0) << 24);
    hw[2] = n; hw[3] = P; hw[4] = num_parts;
  }
  uint32_t* part_off = (uint32_t*)(out + 20);
  uint32_t off = (20u + 4u * (num_parts + 1) + 7u) & ~7u;
  // pad bytes are zero: an odd partition count leaves one word between the offset table and the first partition
  if (lane == 0 && (num_parts & 1u)) part_off[num_parts + 1] = 0u;
  const bool bp = opts.use_bp != 0, sgn = casc_type_signed(opts.type);
  for (uint32_t p = 0; p < num_parts; ++p) {
    if (lane == 0) part_off[p] = off;
    const uint32_t begin = p * P;
    const uint32_t nb = min(P, whole - begin);
    uint32_t sz;
    switch (ts) {
      case 1: sz = casc_encode_part<1>(in + begin, nb, opts.num_RLEs, opts.num_deltas, bp, sgn, out + off, sm, P, lane); break;
      case 2: sz = casc_encode_part<2>(in + begin, nb / 2, opts.num_RLEs, opts.num_deltas, bp, sgn, out + off, sm, P, lane); break;
      case 4: sz = casc_encode_part<4>(in + begin, nb / 4, opts.num_RLEs, opts.num_deltas, bp, sgn, out + off, sm, P, lane); break;
      default: sz = casc_encode_part<8>(in + begin, nb / 8, opts.num_RLEs, opts.num_deltas, bp, sgn, out + off, sm, P, lane); break;
    }
    off += (sz + 7u) & ~7u;
  }
  if (lane == 0) { part_off[num_parts] = off; if (comp_bytes) *comp_bytes = off + (tail ? 8u : 0u); }
  if (tail && lane < 8) out[off + lane] = (uint32_t)lane < tail ? in[whole + lane] : (uint8_t)0;
}

template <class T, class U>
__device__ __forceinline__ T bit_cast_elem(U u) {
  static_assert(sizeof(T) == sizeof(U), "same width");
  T t;
  __builtin_memcpy(&t, &u, sizeof(T));
  return t;
}

}  // namespace detail

// Decode the comp_bytes-byte stream at `comp` into [out, out + capacity), partition after partition, with `smem`
// (smem_bytes bytes) as the partition workspace.  Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem, size_t smem_bytes) {
  using namespace detail;
  const int lane = lane_id();
  const uint8_t* in = (const uint8_t*)comp;
  uint8_t* o = (uint8_t*)out;
  CascHeader h;
  nvcompStatus_t st = nvcompSuccess;
  if (!casc_read_header(in, comp_bytes, h)) st = nvcompErrorCannotDecompress;
  else if (header_smem_bytes(h) > smem_bytes) st = nvcompErrorInvalidValue;
  else {
    const uint32_t ts = casc_type_size(h.type);
    if (h.uncompressed > capacity || ((uintptr_t)o & (ts - 1)) ||
        !walk_chunk_ts<kCascDecode>(ts, in, comp_bytes, h, o, (uint8_t*)smem, CascNoVisit(), lane))
      st = nvcompErrorCannotDecompress;
  }
  if (lane == 0 && actual) *actual = st == nvcompSuccess ? (size_t)h.uncompressed : 0;
  __syncwarp();
  return st;
}

// Compress the n_bytes bytes at `in` (aligned to the element size) into the stream at `out` (8-byte aligned,
// max_compressed_bytes(n_bytes, opts) bytes) and its size into *comp_bytes, with `smem` (compress_smem_bytes(opts)
// bytes) as the partition workspace.  Warp-collective (see above).  Options the batched call rejects return
// nvcompErrorInvalidValue, n_bytes > kMaxChunkBytes returns nvcompErrorChunkSizeTooLarge; both with *comp_bytes = 0
// and nothing else written.
__device__ inline nvcompStatus_t compress_warp(const void* in, size_t n_bytes, void* out, size_t* comp_bytes,
                                               nvcompBatchedCascadedOpts_t opts, void* smem) {
  using namespace detail;
  const int lane = lane_id();
  nvcompStatus_t st = casc_check_opts(opts);
  if (st == nvcompSuccess && n_bytes > kMaxChunkBytes) st = nvcompErrorChunkSizeTooLarge;
  if (st != nvcompSuccess) {
    if (lane == 0 && comp_bytes) *comp_bytes = 0;
    return st;
  }
  compress_chunk((const uint8_t*)in, (uint32_t)n_bytes, (uint8_t*)out, comp_bytes, opts, (uint8_t*)smem, lane);
  __syncwarp();
  return nvcompSuccess;
}

// Visit the decoded elements of the stream at `comp` in registers, in stream order, with `smem` (smem_bytes bytes)
// as the partition workspace.  Warp-collective (see above).
//
// The whole stream is checked first -- the header, every partition offset, every stream header, count and run
// length, and the tail word, i.e. everything decompress_warp checks except the capacity and the output alignment --
// by walking the partitions in a mode that unpacks only the run-length streams.  So `f` is either called for every
// block or never.  Then each partition is decoded into `smem` and, for each block of up to 128 consecutive elements
// (a block never crosses a partition), every lane calls
//     f(const T (&v)[4], uint32_t first_element, uint32_t valid)
// with its four consecutive elements v[0..3] = elements first_element .. first_element + 3 of the chunk, of which
// the first `valid` (0..4) exist; the others are unspecified.  first_element is the partition's first element +
// 128 * block + 4 * lane.  Nothing is stored outside `smem`; all 32 lanes call f together, so f may use warp
// intrinsics.
//
// Returns nvcompSuccess exactly when decompress_warp would succeed with unlimited capacity, and otherwise
// nvcompErrorCannotDecompress without calling f.  A stream whose element size is not sizeof(T), or whose partitions
// need more than smem_bytes, returns nvcompErrorInvalidValue without calling f (a header that is not valid at all
// returns nvcompErrorCannotDecompress).  T is any 1-, 2-, 4- or 8-byte trivially copyable type; the element's bits
// are copied into it.  A chunk whose length is not a multiple of the element size keeps its last bytes in the
// stream's tail word, and f is not given them.
template <class T, class F>
__device__ inline nvcompStatus_t for_each_block(const void* comp, size_t comp_bytes, void* smem, size_t smem_bytes,
                                                F&& f) {
  using namespace detail;
  static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8, "element of 1, 2, 4 or 8 bytes");
  constexpr int TS = (int)sizeof(T);
  using U = typename Elem<TS>::T;
  const int lane = lane_id();
  const uint8_t* in = (const uint8_t*)comp;
  CascHeader h;
  uint8_t* sm = (uint8_t*)smem;
  nvcompStatus_t st = nvcompSuccess;
  if (!casc_read_header(in, comp_bytes, h)) st = nvcompErrorCannotDecompress;
  else if (casc_type_size(h.type) != sizeof(T) || header_smem_bytes(h) > smem_bytes) st = nvcompErrorInvalidValue;
  else if (!walk_chunk<TS, kCascCheck>(in, comp_bytes, h, nullptr, sm, CascNoVisit(), lane))
    st = nvcompErrorCannotDecompress;
  else {
    const auto visit = [&](const U (&v)[4], uint32_t first, uint32_t valid) {
      const T t[4] = {bit_cast_elem<T>(v[0]), bit_cast_elem<T>(v[1]), bit_cast_elem<T>(v[2]), bit_cast_elem<T>(v[3])};
      f(t, first, valid);
    };
    walk_chunk<TS, kCascVisit>(in, comp_bytes, h, nullptr, sm, visit, lane);
  }
  __syncwarp();                                      // every return leaves the warp converged and its region free
  return st;
}

}  // namespace cascaded
}  // namespace device
}  // namespace nvcomp
