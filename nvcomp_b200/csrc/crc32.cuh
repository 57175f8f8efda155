// crc32.cuh -- standard CRC-32 (IEEE 802.3, reflected polynomial 0xEDB88320, the zlib value): the internal interface
// of crc32.cu used by the high-level interface for its whole-buffer checksums, and the warp routine that hashes one
// span (crc0_warp + crc_finish), shared with the Gzip decoder (inflate_decode.cuh).
//
// A CRC is linear over GF(2): with a zero initial register, crc0(A || B) = crc0(A) * x^(8|B|) + crc0(B)
// (mod P).  So every lane hashes its own contiguous slice byte-table-wise, and slices / pieces are
// merged with one carry-less modular multiplication each; the 0xFFFFFFFF pre/post conditioning of
// the standard CRC is added once at the end:  crc32(M) = crc0(M) ^ x^(8|M|) * 0xFFFFFFFF ^ 0xFFFFFFFF.
//
// The device routines take their two tables (crc_table_entry, crc_x2n_entry) as pointers: constant memory in
// crc32.cu, shared memory in the Gzip decoder, host arrays in the host warp emulator (tests/emu).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "common.cuh"

namespace b200 {

constexpr uint32_t kCrcPoly = 0xedb88320u;     // IEEE 802.3, reflected
constexpr size_t kCrcPiece = 65536;            // bytes hashed by one warp

// u32 words of scratch crc32_buffer_async needs for a buffer of at most max_bytes
size_t crc_scratch_words(size_t max_bytes);

// *result = CRC-32 of data[0, n) where n = n_host, or (*len_dev - skip) when len_dev != nullptr (a length
// only the device knows, e.g. the compressed size); max_bytes bounds n and sizes the launch.  Asynchronous.
cudaError_t crc32_buffer_async(const uint8_t* data, size_t n_host, const unsigned long long* len_dev, size_t skip,
                               size_t max_bytes, uint32_t* piece_scratch, uint32_t* result, cudaStream_t stream);

// a * b mod P (reflected bit order)
__host__ __device__ __forceinline__ uint32_t crc_mulmod(uint32_t a, uint32_t b) {
  uint32_t r = 0;
#pragma unroll 4
  for (int k = 31; k >= 0; --k) {
    if ((a >> k) & 1u) r ^= b;
    b = (b & 1u) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return r;
}

// entry i of the byte table: crc0 of the single byte i
__host__ __device__ __forceinline__ uint32_t crc_table_entry(uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ kCrcPoly : c >> 1;
  return c;
}
// entry k of the power table: x^(2^k) mod P, reflected (x^1 is bit 30, x^0 bit 31)
__host__ __device__ __forceinline__ uint32_t crc_x2n_entry(int k) {
  uint32_t p = 1u << 30;
  for (int i = 0; i < k; ++i) p = crc_mulmod(p, p);
  return p;
}

// x^(8 n) mod P
__device__ __forceinline__ uint32_t crc_x8n(const uint32_t* x2n, uint64_t n) {
  uint32_t p = 1u << 31;        // x^0
  int k = 3;                    // x^(8n) = prod over set bits i of n of x^(2^(i+3))
  while (n) {
    if (n & 1ull) p = crc_mulmod(x2n[k & 31], p);
    n >>= 1;
    ++k;
  }
  return p;
}
// crc0 of bytes [p, p+n) continuing register c
__device__ __forceinline__ uint32_t crc_bytes(const uint32_t* __restrict__ table, uint32_t c,
                                              const uint8_t* __restrict__ p, size_t n) {
  size_t i = 0;
  // head up to 4-byte alignment, then word loads
  for (; i < n && (((uintptr_t)(p + i)) & 3u); ++i) c = table[(c ^ p[i]) & 255u] ^ (c >> 8);
  for (; i + 4 <= n; i += 4) {
    const uint32_t w = *(const uint32_t*)(p + i);
    c ^= w;
    c = table[c & 255u] ^ (c >> 8);
    c = table[c & 255u] ^ (c >> 8);
    c = table[c & 255u] ^ (c >> 8);
    c = table[c & 255u] ^ (c >> 8);
  }
  for (; i < n; ++i) c = table[(c ^ p[i]) & 255u] ^ (c >> 8);
  return c;
}

// crc0 of one span by one warp: contiguous slice per lane, merged with x^(8 * bytes after the slice)
__device__ __forceinline__ uint32_t crc0_warp(const uint32_t* table, const uint32_t* x2n, const uint8_t* p, size_t n,
                                              int lane) {
  const size_t slice = ((n + 31) / 32 + 3) & ~(size_t)3;
  const size_t lo = min((size_t)lane * slice, n), hi = min(lo + slice, n);
  uint32_t c = crc_bytes(table, 0u, p + lo, hi - lo);
  if (hi < n && c) c = crc_mulmod(crc_x8n(x2n, n - hi), c);
#pragma unroll
  for (int d = 16; d; d >>= 1) c ^= __shfl_xor_sync(kFull, c, d);
  return c;
}
__device__ __forceinline__ uint32_t crc_finish(const uint32_t* x2n, uint32_t crc0, uint64_t n) {
  return crc0 ^ crc_mulmod(crc_x8n(x2n, n), 0xffffffffu) ^ 0xffffffffu;
}

}  // namespace b200
