/*
 * nvcomp/gzip.h -- batched Gzip DECOMPRESSION (csrc/deflate.cu; decode only, as in the reference; call sites
 * examples/gzip_gpu_decompression.cu:110-164).
 *
 * A chunk is one RFC 1952 member: ID1/ID2 and CM = 8 are checked, reserved FLG bits are rejected, FEXTRA / FNAME /
 * FCOMMENT are skipped, FHCRC (the low 16 bits of the header's CRC-32) is checked, then the Deflate body, then the
 * CRC-32 and ISIZE of the output.  Only the first member is decoded; bytes after its trailer are ignored (zlib leaves
 * them in unused_data).  A chunk decodes iff zlib 1.3 accepts it and its output fits in its capacity.
 *   DecompressGetTempSize   256 bytes (one chunk ticket counter); DecompressAsync also runs with temp == nullptr.
 *   DecompressAsync         chunk i -> out[i] (capacity caps[i]); actual and statuses may be null, actual may alias
 *                           caps.  Per chunk: nvcompSuccess with exactly actual[i] bytes written;
 *                           nvcompErrorBadChecksum when the body decodes but its CRC-32 or ISIZE disagree;
 *                           nvcompErrorCannotDecompress for anything else (structural error, output over the
 *                           capacity, compressed size / capacity >= 2^32).  actual[i] = 0 on failure.  Any alignment.
 *   GetDecompressSizeAsync  walks each member without writing: its decoded length, or 0 if it is rejected.  It checks
 *                           ISIZE but cannot check the CRC-32 (it produces no bytes).
 */
#ifndef NVCOMP_GZIP_H
#define NVCOMP_GZIP_H

#include "shared_types.h"

#ifdef __cplusplus
extern "C" {
#endif

nvcompStatus_t nvcompBatchedGzipDecompressGetTempSize(
    size_t num_chunks, size_t max_uncompressed_chunk_bytes, size_t* temp_bytes);
nvcompStatus_t nvcompBatchedGzipGetDecompressSizeAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    size_t* device_uncompressed_bytes, size_t batch_size, cudaStream_t stream);
nvcompStatus_t nvcompBatchedGzipDecompressAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    const size_t* device_uncompressed_bytes, size_t* device_actual_uncompressed_bytes, size_t batch_size,
    void* const device_temp_ptr, size_t temp_bytes, void* const* device_uncompressed_ptrs,
    nvcompStatus_t* device_statuses, cudaStream_t stream);

#ifdef __cplusplus
}
#endif

#endif
