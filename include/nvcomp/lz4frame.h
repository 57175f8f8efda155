/*
 * nvcomp/lz4frame.h -- batched LZ4 frame-format DECOMPRESSION (csrc/lz4frame.cu; decode only).
 *
 * These are this library's own entry points: nvCOMP has no LZ4 frame decoder (its nvcompBatchedLZ4* calls read raw
 * LZ4 blocks, as nvcomp/lz4.h does here).  They read what liblz4's LZ4F_* API writes: Arrow IPC / Feather
 * LZ4_FRAME buffers, pyarrow.Codec("lz4"), .lz4 files.  The shapes are those of nvcompBatchedGzip*.
 *
 * A chunk is zero or more LZ4 frames (magic 0x184D2204) and skippable frames (0x184D2A50-5F) back to back, filling
 * exactly comp_bytes: what a loop of LZ4F_decompress calls reads, restarting after each frame end.  An empty chunk
 * decodes to 0 bytes; two frames decode to the concatenation of their outputs.  A legacy frame (0x184C2102) or any
 * other magic is rejected, as are trailing bytes and a truncated frame.  Inside a frame liblz4 1.9.4 decides every
 * rule: FLG version 01, reserved FLG / BD bits zero, block-size ID 4-7, the header checksum, the content size (when
 * given and non-zero) against the decoded size, the dictID field read, uncompressed blocks (size high bit), no block
 * stored or decoded larger than the maximum block size, the per-block XXH32 over the stored bytes, the EndMark and
 * the content XXH32.  Compressed blocks follow the LZ4 block grammar of nvcompBatchedLZ4DecompressAsync; a linked
 * frame's match may reach back into earlier blocks of its frame but never before the frame's first output byte, an
 * independent frame's only into its own block.  Dictionaries (LZ4F_decompress_usingDict) are not supported.
 *
 *   DecompressGetTempSize   256 bytes (one chunk ticket counter); DecompressAsync also runs with temp == nullptr.
 *   DecompressAsync         chunk i -> out[i] (capacity caps[i]); actual and statuses may be null, actual may alias
 *                           caps.  The first failing check in stream order decides the status:
 *                           nvcompSuccess with exactly actual[i] bytes written and nothing in [actual[i], caps[i]);
 *                           nvcompErrorBadChecksum for a header, block or content checksum mismatch whose preceding
 *                           output fits in the capacity (a compressed block's checksum is checked before the block
 *                           is decoded, an uncompressed block's after its bytes are copied, as liblz4 does);
 *                           nvcompErrorCannotDecompress for anything else (structural error, unknown frame type,
 *                           output over the capacity, compressed size / capacity >= 2^32).  actual[i] = 0 on failure.
 *                           Any input or output alignment.
 *   GetDecompressSizeAsync  walks every frame without writing and without trusting the content-size field: the
 *                           decoded total, or 0 if the chunk is rejected.  It checks everything DecompressAsync
 *                           checks except the content checksum (it produces no bytes).
 */
#ifndef NVCOMP_LZ4FRAME_H
#define NVCOMP_LZ4FRAME_H

#include "shared_types.h"

#ifdef __cplusplus
extern "C" {
#endif

nvcompStatus_t nvcompBatchedLZ4FrameDecompressGetTempSize(
    size_t num_chunks, size_t max_uncompressed_chunk_bytes, size_t* temp_bytes);
nvcompStatus_t nvcompBatchedLZ4FrameGetDecompressSizeAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    size_t* device_uncompressed_bytes, size_t batch_size, cudaStream_t stream);
nvcompStatus_t nvcompBatchedLZ4FrameDecompressAsync(
    const void* const* device_compressed_ptrs, const size_t* device_compressed_bytes,
    const size_t* device_uncompressed_bytes, size_t* device_actual_uncompressed_bytes, size_t batch_size,
    void* const device_temp_ptr, size_t temp_bytes, void* const* device_uncompressed_ptrs,
    nvcompStatus_t* device_statuses, cudaStream_t stream);

#ifdef __cplusplus
}
#endif

#endif
