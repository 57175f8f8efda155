/*
 * nvcomp/zstd.h -- batched Zstandard (RFC 8878) DECOMPRESSION (csrc/zstd.cu).  Compression is not provided: the three
 * Compress entry points return nvcompErrorNotSupported (and ZstdManager, which compresses, throws NotSupported).
 *
 * A chunk is what libzstd 1.5.5's one-shot ZSTD_decompress(dst, cap, src, n) accepts: zero or more Zstandard frames
 * and skippable frames (magic 0x184D2A5?), back to back, filling exactly n bytes.  An empty chunk decodes to 0 bytes;
 * two frames decode to their concatenation; a trailing byte, a frame with a non-zero Dictionary_ID, a legacy (pre-v1)
 * frame or a match that reaches back before the start of its own frame is rejected.  Any Zstandard producer's frames
 * decode (libzstd, pyarrow / Arrow, Parquet and ORC writers, ...), any window size.
 *   DecompressGetTempSize   256 bytes (one chunk ticket counter); DecompressAsync also runs with temp == nullptr.
 *   DecompressAsync         chunk i -> out[i] (capacity caps[i]); actual and statuses may be null, actual may alias
 *                           caps.  Per chunk:
 *                           nvcompSuccess exactly when libzstd succeeds: actual[i] = its length, the bytes are
 *                             identical and nothing is written in [actual[i], caps[i]);
 *                           nvcompErrorBadChecksum when libzstd's first error is a content checksum mismatch (the
 *                             low 32 bits of XXH64, seed 0; in a multi-frame chunk each frame's checksum is checked
 *                             before the next frame starts);
 *                           nvcompErrorCannotDecompress for anything else (structure errors, output over the
 *                             capacity, a dictionary ID, reserved bits, compressed size / capacity >= 2^32).
 *                           actual[i] = 0 on failure.  Any input or output alignment.
 *                           One known difference: libzstd 1.5.5 decodes 4-stream Huffman literals with a fast loop
 *                           that checks that each stream fills its quarter of the literals but not that it ends
 *                           exactly on its first bit; this decoder checks both, so a block whose 4-stream literal
 *                           stream does not end exactly (libzstd decodes it to wrong bytes, usually caught by its
 *                           checksum or content size) is nvcompErrorCannotDecompress here.
 *   GetDecompressSizeAsync  runs the same decoder with stores disabled (Frame_Content_Size is not trusted).  It
 *                           produces no bytes, so it cannot see a content checksum: it checks everything else and
 *                           walks on past each frame's checksum.  For a chunk of one frame, its size is non-zero
 *                           exactly when DecompressAsync with unlimited capacity would succeed or fail only on the
 *                           content checksum.  In a multi-frame chunk whose frame k has a wrong checksum,
 *                           DecompressAsync stops there with nvcompErrorBadChecksum, while the size query goes on to
 *                           the later frames and reports 0 if one of them is malformed (the total length
 *                           otherwise).  A checksum field cut short ends the walk: the size so far is reported.
 * nvcompZstdRequiredAlignment is kept for source compatibility; the decoder needs no alignment.
 */
#ifndef NVCOMP_ZSTD_H
#define NVCOMP_ZSTD_H

#include "shared_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct
{
  int algo;
} nvcompBatchedZstdOpts_t;

static const nvcompBatchedZstdOpts_t nvcompBatchedZstdDefaultOpts = {0};
static const size_t nvcompZstdCompressionMaxAllowedChunkSize = 1 << 16;
static const size_t nvcompZstdRequiredAlignment = 8;

nvcompStatus_t nvcompBatchedZstdCompressGetTempSize(
    size_t batch_size, size_t max_uncompressed_chunk_bytes, nvcompBatchedZstdOpts_t format_opts, size_t* temp_bytes);
nvcompStatus_t nvcompBatchedZstdCompressGetMaxOutputChunkSize(
    size_t max_uncompressed_chunk_bytes, nvcompBatchedZstdOpts_t format_opts, size_t* max_compressed_bytes);
nvcompStatus_t nvcompBatchedZstdCompressAsync(
    const void* const* device_uncompressed_ptrs, const size_t* device_uncompressed_bytes,
    size_t max_uncompressed_chunk_bytes, size_t batch_size, void* device_temp_ptr, size_t temp_bytes,
    void* const* device_compressed_ptrs, size_t* device_compressed_bytes,
    nvcompBatchedZstdOpts_t format_opts, cudaStream_t stream);
nvcompStatus_t nvcompBatchedZstdDecompressGetTempSize(
    size_t num_chunks, size_t max_uncompressed_chunk_bytes, size_t* temp_bytes);
nvcompStatus_t nvcompBatchedZstdGetDecompressSizeAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    size_t* device_uncompressed_bytes, size_t batch_size, cudaStream_t stream);
nvcompStatus_t nvcompBatchedZstdDecompressAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    const size_t* device_uncompressed_bytes, size_t* device_actual_uncompressed_bytes, size_t batch_size,
    void* const device_temp_ptr, size_t temp_bytes, void* const* device_uncompressed_ptrs,
    nvcompStatus_t* device_statuses, cudaStream_t stream);

#ifdef __cplusplus
}
#endif

#endif
