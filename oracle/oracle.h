/*
 * oracle/ -- CPU restatement of the batched-codec hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference leg may load this library; nothing under nvcomp_b200/ links, imports
 * or calls it.  The product path is libnvcomp.so (CUDA, sm_90a) and has no CPU
 * fallback.
 *
 * What it restates: the reference's codec arithmetic lives in the closed,
 * un-vendored dependency nvcomp 3.0.3 (reference CMakeLists.txt:18, README.md:10),
 * so each function restates the *published* algorithm the reference names and is
 * pinned against the independent implementations the reference itself links or
 * names (SURVEY.md section 8c):
 *   - LZ4 block format   -> pinned against liblz4 1.9.4 (the reference links it:
 *                           examples/lz4_cpu_compression.cu:61-66,
 *                           examples/lz4_cpu_decompression.cu:143-147)
 *   - Snappy raw format  -> pinned against pyarrow 24's bundled snappy codec
 *                           (the reference has no CPU Snappy cross-check in-tree)
 *   - Cascaded / Bitcomp / ANS: the reference bitstreams are undocumented and no
 *     binary exists here => stream-level parity is UNPINNED; the oracle restates
 *     this repo's own stream definitions (DESIGN.md) as an independent second
 *     implementation, and lossless round-trip is the property checked.
 */
#ifndef ORACLE_H
#define ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* All decoders return the number of bytes produced, or -1 on a malformed /
 * truncated / overflowing stream (never read or write out of bounds). */
long oracle_lz4_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap);
long oracle_lz4_decompressed_size(const uint8_t* src, size_t n);
long oracle_lz4_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap);
size_t oracle_lz4_bound(size_t n);

long oracle_snappy_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap);
long oracle_snappy_decompressed_size(const uint8_t* src, size_t n);
long oracle_snappy_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap);
size_t oracle_snappy_bound(size_t n);

/* Test hook of the Cascaded / Bitcomp / ANS decoders (typed_oracle.c): skip the named rejection rules
 * (comma-separated; NULL: none) in the calling thread. */
void oracle_typed_skip_rules(const char* names);

/* codec ids for the threaded batch runner */
enum { ORACLE_LZ4 = 0, ORACLE_SNAPPY = 1, ORACLE_CASCADED = 2, ORACLE_BITCOMP = 3, ORACLE_ANS = 4,
       ORACLE_LIBLZ4 = 5 /* liblz4.so.1's LZ4_decompress_safe (dlopen), not the port */ };
int oracle_have_liblz4(void);

/* Decompress `count` chunks with `nthreads` pthreads (contiguous chunk range per
 * thread, SURVEY.md 8d "CPU baseline").  comp = base pointer of a slab,
 * comp_off/comp_len per chunk; outputs go to out + i*out_stride.  Returns wall
 * seconds (steady clock) or a negative value if any chunk failed. */
double oracle_batch_decompress(int codec, const uint8_t* comp, const size_t* comp_off,
                               const size_t* comp_len, size_t count, uint8_t* out,
                               size_t out_stride, size_t* out_len, int nthreads);

#ifdef __cplusplus
}
#endif
#endif
