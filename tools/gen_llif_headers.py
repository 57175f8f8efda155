#!/usr/bin/env python3
"""Generate include/nvcomp/<fmt>.h -- the low-level batched C API (LLIF) of each
codec.  The six entry points per format are exactly the ones the reference's
benchmarks/examples bind (SURVEY.md section 8b); every prototype cites the
reference call site it replaces."""
import os, textwrap

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "nvcomp")

FORMATS = {
    "lz4": dict(
        F="LZ4", guard="NVCOMP_LZ4_H", opts_t="nvcompBatchedLZ4Opts_t",
        opts_def="typedef struct\n{\n  /* element type hint: CHAR/UCHAR/BITS match bytes, SHORT/USHORT 2-byte\n   * aligned, INT/UINT 4-byte aligned candidates (CHANGELOG.md:169-170) */\n  nvcompType_t data_type;\n} nvcompBatchedLZ4Opts_t;",
        default="static const nvcompBatchedLZ4Opts_t nvcompBatchedLZ4DefaultOpts = {NVCOMP_TYPE_CHAR};",
        maxchunk="1 << 24", align="4",
        cites=dict(
            opts="benchmarks/benchmark_lz4_chunked.cu:32",
            ctemp="doc/lowlevel_c_quickstart.md:32-36; benchmarks/benchmark_template_chunked.cuh:420",
            cmax="benchmarks/benchmark_template_chunked.cuh:429-430",
            comp="doc/lowlevel_c_quickstart.md:53-63; examples/low_level_quickstart_example.cpp:86-96",
            dtemp="doc/lowlevel_c_quickstart.md:75-78; examples/lz4_cpu_compression.cu:103-104",
            size="doc/lowlevel_c_quickstart.md:104-109; examples/low_level_quickstart_example.cpp:112-117",
            decomp="doc/lowlevel_c_quickstart.md:127-137; examples/lz4_cpu_compression.cu:121-131"),
        note="Wire format: the public LZ4 *block* format, one block per chunk, interoperable\n * with liblz4 in both directions (examples/lz4_cpu_compression.cu:61-66,\n * examples/lz4_cpu_decompression.cu:143-147)."),
    "snappy": dict(
        F="Snappy", guard="NVCOMP_SNAPPY_H", opts_t="nvcompBatchedSnappyOpts_t",
        opts_def="typedef struct\n{\n  int reserved;\n} nvcompBatchedSnappyOpts_t;",
        default="static const nvcompBatchedSnappyOpts_t nvcompBatchedSnappyDefaultOpts = {0};",
        maxchunk="1 << 24", align="1",
        cites=dict(
            opts="benchmarks/benchmark_snappy_synth.cpp:131; benchmarks/benchmark_hlif.cpp:191",
            ctemp="benchmarks/benchmark_snappy_synth.cpp:128-133",
            cmax="benchmarks/benchmark_snappy_synth.cpp:139-143",
            comp="benchmarks/benchmark_snappy_synth.cpp:163-174",
            dtemp="benchmarks/benchmark_snappy_synth.cpp:220-224",
            size="doc/lowlevel_c_quickstart.md:104-109",
            decomp="benchmarks/benchmark_snappy_synth.cpp:241-252"),
        note="Wire format: the public Snappy raw format (varint32 length preamble, then\n * literal / copy-1 / copy-2 / copy-4 elements).  The decoder accepts every legal\n * stream, not only those its own encoder emits (CHANGELOG.md:182-184)."),
    "cascaded": dict(
        F="Cascaded", guard="NVCOMP_CASCADED_H", opts_t="nvcompBatchedCascadedOpts_t",
        opts_def="typedef struct\n{\n  /* bytes of each independently coded partition inside a chunk; multiple of\n   * the element size, 512..16384, default 4096 */\n  size_t chunk_size;\n  /* element type the RLE / delta / bit-pack layers operate on */\n  nvcompType_t type;\n  /* number of run-length layers (0..7) */\n  int num_RLEs;\n  /* number of delta layers (0..7) */\n  int num_deltas;\n  /* 1: frame-of-reference bit-pack every output stream, 0: store raw */\n  int use_bp;\n} nvcompBatchedCascadedOpts_t;",
        default="static const nvcompBatchedCascadedOpts_t nvcompBatchedCascadedDefaultOpts\n    = {4096, NVCOMP_TYPE_INT, 2, 1, 1};",
        maxchunk="1 << 24", align="8",
        cites=dict(
            opts="benchmarks/benchmark_cascaded_chunked.cu:35-36",
            ctemp="benchmarks/benchmark_cascaded_chunked.cu:138",
            cmax="benchmarks/benchmark_cascaded_chunked.cu:139",
            comp="benchmarks/benchmark_cascaded_chunked.cu:140",
            dtemp="benchmarks/benchmark_cascaded_chunked.cu:141",
            size="doc/lowlevel_c_quickstart.md:104-109",
            decomp="benchmarks/benchmark_cascaded_chunked.cu:142"),
        note="Algorithm: doc/cascaded_overview.md:7-42 (RLE and delta layers interleaved,\n * then frame-of-reference bit-packing of every stream).  The reference's bitstream\n * is undocumented; this library defines its own (DESIGN.md, 'Cascaded stream').\n * actual_bytes and statuses must be non-null for this codec (README.md:14)."),
    "bitcomp": dict(
        F="Bitcomp", guard="NVCOMP_BITCOMP_H", opts_t="nvcompBatchedBitcompFormatOpts",
        opts_def="typedef struct\n{\n  /* 0: default (delta + zig-zag + per-block bit-pack), 1: sparse (zero-mask +\n   * bit-packed non-zeros) */\n  int algorithm_type;\n  /* element type: CHAR..ULONGLONG */\n  nvcompType_t data_type;\n} nvcompBatchedBitcompFormatOpts;",
        default="static const nvcompBatchedBitcompFormatOpts nvcompBatchedBitcompDefaultOpts\n    = {0, NVCOMP_TYPE_UCHAR};",
        maxchunk="1 << 24", align="8",
        cites=dict(
            opts="benchmarks/benchmark_bitcomp_chunked.cu:32-33",
            ctemp="benchmarks/benchmark_bitcomp_chunked.cu:114",
            cmax="benchmarks/benchmark_bitcomp_chunked.cu:115",
            comp="benchmarks/benchmark_bitcomp_chunked.cu:116",
            dtemp="benchmarks/benchmark_bitcomp_chunked.cu:117",
            size="doc/lowlevel_c_quickstart.md:104-109",
            decomp="benchmarks/benchmark_bitcomp_chunked.cu:118"),
        note="Bitcomp is proprietary and undocumented in the reference; this library defines\n * its own lossless typed bit-packing stream (DESIGN.md, 'Bitcomp stream').  Unlike\n * the reference (README.md:15) decompression here is fully asynchronous."),
    "ans": dict(
        F="ANS", guard="NVCOMP_ANS_H", opts_t="nvcompBatchedANSOpts_t",
        opts_def="typedef enum nvcompANSType_t\n{\n  nvcomp_rANS = 0\n} nvcompANSType_t;\n\ntypedef struct\n{\n  nvcompANSType_t type;\n} nvcompBatchedANSOpts_t;",
        default="static const nvcompBatchedANSOpts_t nvcompBatchedANSDefaultOpts = {nvcomp_rANS};",
        maxchunk="1 << 24", align="8",
        cites=dict(
            opts="benchmarks/benchmark_ans_chunked.cu:32,39-41",
            ctemp="benchmarks/benchmark_ans_chunked.cu:68",
            cmax="benchmarks/benchmark_ans_chunked.cu:69",
            comp="benchmarks/benchmark_ans_chunked.cu:70",
            dtemp="benchmarks/benchmark_ans_chunked.cu:71",
            size="doc/lowlevel_c_quickstart.md:104-109",
            decomp="benchmarks/benchmark_ans_chunked.cu:72"),
        note="Byte-wise range-ANS entropy coder.  The reference's bitstream is undocumented;\n * this library defines its own interleaved rANS stream (DESIGN.md, 'ANS stream')."),
}

TEMPLATE = '''/*
 * nvcomp/{name}.h -- low-level batched {F} API (C ABI).
 *
 * Generated by tools/gen_llif_headers.py.  Every entry point replaces the
 * closed libnvcomp.so 3.0.3 symbol of the same name; citations are to the
 * reference tree's call sites that pin the signature.
 *
 * {note}
 *
 * All pointer / size arrays are device-accessible memory; every call only
 * enqueues work on `stream` and returns (no host synchronisation).
 */
#ifndef {guard}
#define {guard}

#include "shared_types.h"

#ifdef __cplusplus
extern "C" {{
#endif

/* Options, passed by value.  Reference: {c[opts]} */
{opts_def}

{default}

static const size_t nvcomp{F}CompressionMaxAllowedChunkSize = {maxchunk};
/* Minimum alignment of every chunk pointer handed to this codec. */
static const size_t nvcomp{F}RequiredAlignment = {align};

/* Workspace bytes CompressAsync needs for `batch_size` chunks of at most
 * `max_uncompressed_chunk_bytes`.  Host only.  Reference: {c[ctemp]} */
nvcompStatus_t nvcompBatched{F}CompressGetTempSize(
    size_t batch_size,
    size_t max_uncompressed_chunk_bytes,
    {opts_t} format_opts,
    size_t* temp_bytes);

/* Same, with the total uncompressed size of the batch as an extra hint
 * (CHANGELOG.md:36-38,114-117). */
nvcompStatus_t nvcompBatched{F}CompressGetTempSizeEx(
    size_t batch_size,
    size_t max_uncompressed_chunk_bytes,
    {opts_t} format_opts,
    size_t* temp_bytes,
    const size_t max_total_uncompressed_bytes);

/* Upper bound of one compressed chunk.  Host only.  Reference: {c[cmax]} */
nvcompStatus_t nvcompBatched{F}CompressGetMaxOutputChunkSize(
    size_t max_uncompressed_chunk_bytes,
    {opts_t} format_opts,
    size_t* max_compressed_bytes);

/* Compress `batch_size` independent chunks.  Reference: {c[comp]} */
nvcompStatus_t nvcompBatched{F}CompressAsync(
    const void* const* device_uncompressed_ptrs,
    const size_t* device_uncompressed_bytes,
    size_t max_uncompressed_chunk_bytes,
    size_t batch_size,
    void* device_temp_ptr,
    size_t temp_bytes,
    void* const* device_compressed_ptrs,
    size_t* device_compressed_bytes,
    {opts_t} format_opts,
    cudaStream_t stream);

/* Workspace bytes DecompressAsync needs.  Host only.  Reference: {c[dtemp]} */
nvcompStatus_t nvcompBatched{F}DecompressGetTempSize(
    size_t num_chunks,
    size_t max_uncompressed_chunk_bytes,
    size_t* temp_bytes);

nvcompStatus_t nvcompBatched{F}DecompressGetTempSizeEx(
    size_t num_chunks,
    size_t max_uncompressed_chunk_bytes,
    size_t* temp_bytes,
    size_t max_uncompressed_total_size);

/* Decompressed size of every chunk without materialising it.
 * Reference: {c[size]} */
nvcompStatus_t nvcompBatched{F}GetDecompressSizeAsync(
    const void* const* device_compressed_ptrs,
    const size_t* device_compressed_bytes,
    size_t* device_uncompressed_bytes,
    size_t batch_size,
    cudaStream_t stream);

/* Decompress `batch_size` chunks.  `device_uncompressed_bytes[i]` is the
 * capacity of output i; `device_actual_uncompressed_bytes` (may alias it,
 * benchmarks/benchmark_snappy_synth.cpp:244-245) receives the produced size,
 * 0 on failure; `device_statuses[i]` receives nvcompSuccess or
 * nvcompErrorCannotDecompress.  A malformed or truncated chunk never causes an
 * out-of-bounds access (CHANGELOG.md:160-164).  Reference: {c[decomp]} */
nvcompStatus_t nvcompBatched{F}DecompressAsync(
    const void* const* device_compressed_ptrs,
    const size_t* device_compressed_bytes,
    const size_t* device_uncompressed_bytes,
    size_t* device_actual_uncompressed_bytes,
    size_t batch_size,
    void* const device_temp_ptr,
    size_t temp_bytes,
    void* const* device_uncompressed_ptrs,
    nvcompStatus_t* device_statuses,
    cudaStream_t stream);

#ifdef __cplusplus
}}
#endif

#endif
'''

def main():
    os.makedirs(ROOT, exist_ok=True)
    for name, f in FORMATS.items():
        txt = TEMPLATE.format(name=name, c=f["cites"], **{k: v for k, v in f.items() if k != "cites"})
        with open(os.path.join(ROOT, name + ".h"), "w") as fh:
            fh.write(txt)
        print("wrote", name + ".h")

if __name__ == "__main__":
    main()
