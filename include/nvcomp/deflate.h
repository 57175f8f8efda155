/*
 * nvcomp/deflate.h -- batched Deflate DECOMPRESSION (csrc/deflate.cu).
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
 * Compression (the three Compress* entry points) and DeflateManager are not supported: they return / throw
 * nvcompErrorNotSupported.  They exist so the reference's globbed benchmarks and benchmark_hlif.cpp (which names
 * DeflateManager, benchmarks/benchmark_hlif.cpp:207-212) compile and link.
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
nvcompStatus_t nvcompBatchedDeflateCompressGetMaxOutputChunkSize(
    size_t max_uncompressed_chunk_bytes, nvcompBatchedDeflateOpts_t format_opts, size_t* max_compressed_bytes);
nvcompStatus_t nvcompBatchedDeflateCompressAsync(
    const void* const* device_uncompressed_ptrs, const size_t* device_uncompressed_bytes,
    size_t max_uncompressed_chunk_bytes, size_t batch_size, void* device_temp_ptr, size_t temp_bytes,
    void* const* device_compressed_ptrs, size_t* device_compressed_bytes,
    nvcompBatchedDeflateOpts_t format_opts, cudaStream_t stream);
nvcompStatus_t nvcompBatchedDeflateDecompressGetTempSize(
    size_t num_chunks, size_t max_uncompressed_chunk_bytes, size_t* temp_bytes);
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
