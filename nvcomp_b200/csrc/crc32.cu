// crc32.cu -- standard CRC-32 (IEEE 802.3, reflected polynomial 0xEDB88320, the zlib / boost::crc_32_type
// value) on the GPU: the low-level batched API (reference CHANGELOG.md:51 "Standard CRC32 support and its LLAPI";
// reference examples/standard_crc_checksum.cpp:94-104 checks it against boost::crc_32_type) and the
// whole-buffer checksums of the high-level interface (hlif.cu).  The warp routine and the method are in crc32.cuh.
#include "crc32.cuh"

#include "common.cuh"
#include "nvcomp/crc32.h"

namespace b200 {

__constant__ uint32_t c_crc_table[256];
__constant__ uint32_t c_crc_x2n[32];      // x^(2^k) mod P, reflected

static void crc_host_tables(uint32_t* table, uint32_t* x2n) {
  for (uint32_t i = 0; i < 256; ++i) table[i] = crc_table_entry(i);
  for (int k = 0; k < 32; ++k) x2n[k] = crc_x2n_entry(k);
}

// constant tables are per device: upload once per device (atomic memo, like ensure_dynamic_smem)
cudaError_t crc_init_tables() {
  static std::atomic<unsigned long long> memo{0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const bool tracked = dev >= 0 && dev < 64;
  if (tracked && ((memo.load(std::memory_order_acquire) >> dev) & 1ull)) return cudaSuccess;
  uint32_t table[256], x2n[32];
  crc_host_tables(table, x2n);
  e = cudaMemcpyToSymbol(c_crc_table, table, sizeof(table));
  if (e != cudaSuccess) return e;
  e = cudaMemcpyToSymbol(c_crc_x2n, x2n, sizeof(x2n));
  if (e == cudaSuccess && tracked) memo.fetch_or(1ull << dev, std::memory_order_release);
  return e;
}

constexpr int kCrcWarps = 8;

// batched: one warp per chunk
__global__ void __launch_bounds__(kCrcWarps * 32)
crc32_batch_kernel(const void* const* __restrict__ ptrs, const size_t* __restrict__ bytes, size_t batch,
                   uint32_t* __restrict__ crcs) {
  __shared__ uint32_t s_table[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_table[i] = c_crc_table[i];
  __syncthreads();
  const int lane = lane_id();
  const size_t warps_total = (size_t)gridDim.x * kCrcWarps;
  for (size_t c = (size_t)blockIdx.x * kCrcWarps + (threadIdx.x >> 5); c < batch; c += warps_total) {
    const uint8_t* p = (const uint8_t*)ptrs[c];
    const size_t n = bytes[c];
    const uint32_t c0 = crc0_warp(s_table, c_crc_x2n, p, n, lane);
    if (lane == 0) crcs[c] = crc_finish(c_crc_x2n, c0, n);
  }
}

// one contiguous buffer in pieces of kCrcPiece bytes: piece_crc0[i] = crc0 of piece i (0 for pieces past the end).
// The length comes from the host (n_host) or, when len_dev != nullptr, from device memory (*len_dev - skip).
__global__ void __launch_bounds__(kCrcWarps * 32)
crc32_pieces_kernel(const uint8_t* __restrict__ data, size_t n_host, const unsigned long long* len_dev, size_t skip,
                    size_t max_bytes, size_t max_pieces, uint32_t* __restrict__ piece_crc0) {
  __shared__ uint32_t s_table[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_table[i] = c_crc_table[i];
  __syncthreads();
  size_t n = n_host;
  if (len_dev) { const unsigned long long t = *len_dev; n = t > skip ? (size_t)(t - skip) : 0; }
  n = min(n, max_bytes);                        // a corrupt device-side length never reads past the bound
  const int lane = lane_id();
  const size_t warps_total = (size_t)gridDim.x * kCrcWarps;
  for (size_t i = (size_t)blockIdx.x * kCrcWarps + (threadIdx.x >> 5); i < max_pieces; i += warps_total) {
    const size_t lo = i * kCrcPiece;
    uint32_t c0 = 0;
    if (lo < n) c0 = crc0_warp(s_table, c_crc_x2n, data + lo, min(kCrcPiece, n - lo), lane);
    if (lane == 0) piece_crc0[i] = c0;
  }
}

// single CTA: fold the piece values in order.  Every piece but the last is kCrcPiece bytes, so a thread folds
// its contiguous group with one constant multiplier; groups merge in a shared-memory tree.
__global__ void __launch_bounds__(1024)
crc32_fold_kernel(const uint32_t* __restrict__ piece_crc0, size_t n_host, const unsigned long long* len_dev, size_t skip,
                  size_t max_bytes, uint32_t* __restrict__ result) {
  __shared__ uint32_t s_c[1024];
  __shared__ unsigned long long s_len[1024];
  size_t n = n_host;
  if (len_dev) { const unsigned long long t = *len_dev; n = t > skip ? (size_t)(t - skip) : 0; }
  n = min(n, max_bytes);
  const size_t pieces = (n + kCrcPiece - 1) / kCrcPiece;
  const size_t per = (pieces + blockDim.x - 1) / blockDim.x;
  const size_t p0 = min((size_t)threadIdx.x * per, pieces), p1 = min(p0 + per, pieces);
  const uint32_t xpiece = crc_x8n(c_crc_x2n, kCrcPiece);
  uint32_t c = 0;
  unsigned long long len = 0;
  for (size_t i = p0; i < p1; ++i) {
    const unsigned long long li = min((unsigned long long)kCrcPiece, (unsigned long long)(n - i * kCrcPiece));
    // appending piece i: c = c * x^(8 li) + crc0_i ; li == kCrcPiece except for the very last piece
    if (c) c = crc_mulmod(li == kCrcPiece ? xpiece : crc_x8n(c_crc_x2n, li), c);
    c ^= piece_crc0[i];
    len += li;
  }
  s_c[threadIdx.x] = c;
  s_len[threadIdx.x] = len;
  __syncthreads();
  for (unsigned stride = 1; stride < blockDim.x; stride <<= 1) {
    const unsigned i = threadIdx.x;
    if ((i & (2 * stride - 1)) == 0 && i + stride < blockDim.x) {
      const unsigned long long lr = s_len[i + stride];
      uint32_t cl = s_c[i];
      if (cl && lr) cl = crc_mulmod(crc_x8n(c_crc_x2n, lr), cl);
      s_c[i] = cl ^ s_c[i + stride];
      s_len[i] += lr;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *result = crc_finish(c_crc_x2n, s_c[0], n);
}

size_t crc_scratch_words(size_t max_bytes) { return (max_bytes + kCrcPiece - 1) / kCrcPiece + 1; }

cudaError_t crc32_buffer_async(const uint8_t* data, size_t n_host, const unsigned long long* len_dev, size_t skip,
                               size_t max_bytes, uint32_t* piece_scratch, uint32_t* result, cudaStream_t stream) {
  cudaError_t e = crc_init_tables();
  if (e != cudaSuccess) return e;
  const size_t max_pieces = (max_bytes + kCrcPiece - 1) / kCrcPiece;
  if (max_pieces) {
    const int grid = persistent_grid(8, max_pieces, kCrcWarps);
    crc32_pieces_kernel<<<grid, kCrcWarps * 32, 0, stream>>>(data, n_host, len_dev, skip, max_bytes, max_pieces, piece_scratch);
  }
  crc32_fold_kernel<<<1, 1024, 0, stream>>>(piece_scratch, n_host, len_dev, skip, max_bytes, result);
  return cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" nvcompStatus_t nvcompBatchedCRC32Async(
    const void* const* device_uncompressed_ptrs, const size_t* device_uncompressed_bytes, size_t batch_size,
    uint32_t* device_CRC32_ptr, cudaStream_t stream) {
  log_call("nvcompBatchedCRC32Async", batch_size, 0, stream);
  if (batch_size == 0) return nvcompSuccess;
  if (!device_uncompressed_ptrs || !device_uncompressed_bytes || !device_CRC32_ptr) return nvcompErrorInvalidValue;
  B200_CUDA_TRY(crc_init_tables());
  const int grid = persistent_grid(8, batch_size, kCrcWarps);
  crc32_batch_kernel<<<grid, kCrcWarps * 32, 0, stream>>>(device_uncompressed_ptrs, device_uncompressed_bytes,
                                                         batch_size, device_CRC32_ptr);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}
