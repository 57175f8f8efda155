/*
 * nvcomp/deflate.h -- batched Deflate compression and decompression (csrc/deflate.cu, csrc/deflate_compress.cuh).
 *
 * A chunk is one raw RFC 1951 stream (zlib wbits = -15, as the reference's deflate_cpu_* examples write it), with a
 * 32 KB window and no state across chunks.  Bytes after the end of the final block are ignored (zlib leaves them in
 * unused_data).  A chunk decodes iff zlib 1.3 accepts it and its output fits in its capacity.
 *   DecompressGetTempSize   256 bytes (one chunk ticket counter); DecompressAsync also runs with temp == nullptr.
 *   DecompressAsync         chunk i -> out[i] (capacity caps[i]); actual and statuses may be null, actual may alias
 *                           caps.  Per chunk: nvcompSuccess with exactly actual[i] bytes written, or
 *                           nvcompErrorCannotDecompress (any structural error, output over the capacity, or a
 *                           compressed size / capacity >= 2^32) with actual[i] = 0.  Any byte alignment.
 *   GetDecompressSizeAsync  walks each stream without writing: its decoded length, or 0 if it is rejected.
 *
 * Compression writes each chunk (0 to 65 536 bytes) as one raw RFC 1951 stream with a single final block: stored,
 * fixed-code or dynamic-code, whichever is smallest.  The output is a deterministic function of the chunk and algo.
 *   opts.algo  0: high throughput (default): greedy LZ77 parse, 4096-entry hash table.
 *              1: high compression: 32 768-entry hash table and a one-position lazy step (a match is dropped for a
 *                 longer one at the next position and a distance no larger).
 *              2: entropy only: no matches, Huffman-coded literals.
 *              Anything else: nvcompErrorInvalidValue from all three Compress* entry points.  This mapping is this
 *              library's own, modelled on the names of GDeflate's variants; it is not verified against NVIDIA's
 *              binary.
 *   max_uncompressed_chunk_bytes > nvcompDeflateCompressionMaxAllowedChunkSize: nvcompErrorChunkSizeTooLarge.
 *   CompressGetMaxOutputChunkSize  m + 5 * (m / 65535 + 1) (the stored encoding; no stream is larger).
 *   CompressGetTempSize            256 bytes (one chunk ticket counter); CompressAsync also runs with temp == nullptr.
 *   CompressAsync                  writes only inside [out[i], out[i] + max output size) and exactly out_bytes[i]
 *                                  bytes.  Any byte alignment.
 */
#ifndef NVCOMP_DEFLATE_H
#define NVCOMP_DEFLATE_H

#include "shared_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct
{
  int algo;
} nvcompBatchedDeflateOpts_t;

static const nvcompBatchedDeflateOpts_t nvcompBatchedDeflateDefaultOpts = {0};
static const size_t nvcompDeflateCompressionMaxAllowedChunkSize = 1 << 16;
static const size_t nvcompDeflateRequiredAlignment = 8;

nvcompStatus_t nvcompBatchedDeflateCompressGetTempSize(
    size_t batch_size, size_t max_uncompressed_chunk_bytes, nvcompBatchedDeflateOpts_t format_opts, size_t* temp_bytes);
nvcompStatus_t nvcompBatchedDeflateCompressGetTempSizeEx(
    size_t batch_size, size_t max_uncompressed_chunk_bytes, nvcompBatchedDeflateOpts_t format_opts, size_t* temp_bytes,
    const size_t max_total_uncompressed_bytes);
nvcompStatus_t nvcompBatchedDeflateCompressGetMaxOutputChunkSize(
    size_t max_uncompressed_chunk_bytes, nvcompBatchedDeflateOpts_t format_opts, size_t* max_compressed_bytes);
nvcompStatus_t nvcompBatchedDeflateCompressAsync(
    const void* const* device_uncompressed_ptrs, const size_t* device_uncompressed_bytes,
    size_t max_uncompressed_chunk_bytes, size_t batch_size, void* device_temp_ptr, size_t temp_bytes,
    void* const* device_compressed_ptrs, size_t* device_compressed_bytes,
    nvcompBatchedDeflateOpts_t format_opts, cudaStream_t stream);
nvcompStatus_t nvcompBatchedDeflateDecompressGetTempSize(
    size_t num_chunks, size_t max_uncompressed_chunk_bytes, size_t* temp_bytes);
nvcompStatus_t nvcompBatchedDeflateDecompressGetTempSizeEx(
    size_t num_chunks, size_t max_uncompressed_chunk_bytes, size_t* temp_bytes, size_t max_total_uncompressed_bytes);
nvcompStatus_t nvcompBatchedDeflateGetDecompressSizeAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    size_t* device_uncompressed_bytes, size_t batch_size, cudaStream_t stream);
nvcompStatus_t nvcompBatchedDeflateDecompressAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    const size_t* device_uncompressed_bytes, size_t* device_actual_uncompressed_bytes, size_t batch_size,
    void* const device_temp_ptr, size_t temp_bytes, void* const* device_uncompressed_ptrs,
    nvcompStatus_t* device_statuses, cudaStream_t stream);

#ifdef __cplusplus
}
#endif

#endif
