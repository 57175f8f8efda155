// nvcomp/device/gzip.cuh -- warp-level Gzip (RFC 1952) decompression inside a user's own kernels.
//
// This is this library's own interface.  decompress_warp returns, for every chunk and capacity, the status, size and
// bytes that nvcompBatchedGzipDecompressAsync (nvcomp/gzip.h) returns: the first member of the chunk is decoded, its
// header checked (and its header CRC, when FHCRC is set), its CRC-32 and ISIZE compared with the decoded bytes.  It
// runs the batched kernel's own code (detail/inflate_decode.cuh, detail/crc32.cuh).  There is no Gzip compression.
//
// Header-only device code for sm_90a: compile with -Iinclude -gencode arch=compute_90a,code=sm_90a; no link
// against libnvcomp.so is needed.
//
// Contract of decompress_warp and decompressed_size_warp: as in nvcomp/device/lz4.cuh --
//   - All 32 lanes of a converged warp call with identical arguments.  The returned status is warp-uniform, and
//     *actual is written once (by lane 0; the pointer may be null).
//   - Compressed streams and outputs are global memory and must not overlap.  Any alignment is accepted.
//   - `smem` is this warp's own shared-memory region of kDecompressSmemBytes bytes, aligned to kSmemAlignment.  It
//     holds nothing between calls: every call builds the CRC-32 tables in the region's tail (the batched kernel
//     builds them once per CTA) and the fixed-code tables when it needs them.  Every return passes a __syncwarp.
//   - decompress_warp writes only inside [out, out + capacity).  A successful decode writes exactly *actual bytes.
//   - A CRC-32 or ISIZE mismatch returns nvcompErrorBadChecksum, any other chunk that cannot be decoded (malformed,
//     larger than capacity, or comp_bytes or capacity of 2^32 or more) nvcompErrorCannotDecompress; both with
//     *actual = 0.  No input causes an out-of-bounds access.
//   - Several warps of one CTA may run any mix of Deflate, Gzip and Zstd calls at once, each with its own region.
//     No call uses global scratch memory.
#pragma once

#include "nvcomp/gzip.h"
#include "nvcomp/device/detail/inflate_region.cuh"

namespace nvcomp {
namespace device {
namespace gzip {

// Alignment of each warp's shared-memory region.
constexpr size_t kSmemAlignment = 16;

// Shared memory of one decoding warp: the Deflate decoder's 10 368 bytes, then the CRC-32 byte table and the
// x^(2^k) table (1 152 bytes).
constexpr size_t kDecompressSmemBytes = deflate::detail::kGzipWarpSmem;

static_assert(kDecompressSmemBytes % kSmemAlignment == 0, "warp regions stay aligned");

// Decompressed size of the Gzip member at `comp` -- what nvcompBatchedGzipGetDecompressSizeAsync reports for the
// chunk: the warp walks the member without writing and checks its ISIZE, not its CRC-32.  0 for a chunk it rejects.
// `smem`: kDecompressSmemBytes bytes.  Warp-collective (see above).
__device__ inline size_t decompressed_size_warp(const void* comp, size_t comp_bytes, void* smem) {
  return deflate::detail::inflate_size_warp<true>(comp, comp_bytes, smem);
}

// Decode the first Gzip member of the comp_bytes-byte chunk at `comp` into [out, out + capacity) with `smem`
// (kDecompressSmemBytes bytes).  Warp-collective (see above).
__device__ inline nvcompStatus_t decompress_warp(const void* comp, size_t comp_bytes, void* out, size_t capacity,
                                                 size_t* actual, void* smem) {
  return deflate::detail::inflate_decompress_warp<true>(comp, comp_bytes, out, capacity, actual, smem);
}

}  // namespace gzip
}  // namespace device
}  // namespace nvcomp
