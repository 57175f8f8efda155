// deflate.cu -- batched Deflate (RFC 1951) and Gzip (RFC 1952) decompression for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedDeflate{DecompressGetTempSize, GetDecompressSizeAsync, DecompressAsync} and
// nvcompBatchedGzip* entry points (include/nvcomp/deflate.h, gzip.h; reference call site
// examples/gzip_gpu_decompression.cu:110-164).  Decode only: Deflate compression and DeflateManager report
// nvcompErrorNotSupported (hlif.cu).  One warp decodes one chunk (inflate_decode.cuh); a persistent grid of 4-warp
// CTAs pulls chunks from a ticket counter in the workspace, or walks a static grid stride without one.
#include "common.cuh"
#include "crc32.cuh"
#include "inflate_decode.cuh"
#include "nvcomp/deflate.h"
#include "nvcomp/gzip.h"

namespace b200 {

constexpr int kInfWarps = 4;
// 4 x 10 368 B of decode tables + 1 152 B of CRC tables = 42 624 B per CTA: 5 CTAs per SM fit in shared memory
constexpr int kInfCtasPerSm = 5;

// kCount: the size query (walk without writing; actual_bytes receives the decoded lengths, out_caps / out_ptrs /
// statuses are unused)
template <bool kGzip, bool kCount>
__global__ void __launch_bounds__(kInfWarps * 32, kInfCtasPerSm)
inflate_kernel(const void* const* __restrict__ comp_ptrs, const size_t* __restrict__ comp_bytes,
               const size_t* out_caps, size_t* actual_bytes, size_t batch, void* const* __restrict__ out_ptrs,
               nvcompStatus_t* statuses, unsigned long long* ticket) {
  __shared__ __align__(16) uint8_t s_warp[kInfWarps][kInfWarpSmem];
  __shared__ uint32_t s_crc[kGzip ? 256 + 32 : 1];    // byte table, then x^(2^k)
  if (kGzip) {
    for (uint32_t i = threadIdx.x; i < 256u + 32u; i += blockDim.x)
      s_crc[i] = i < 256u ? crc_table_entry(i) : crc_x2n_entry((int)(i - 256u));
    __syncthreads();
  }
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const size_t warp_global = (size_t)blockIdx.x * kInfWarps + w;
  const size_t warps_total = (size_t)gridDim.x * kInfWarps;
  InflateWarp ws{smem_addr(s_warp[w]), false};
  WarpTicket sched(ticket, warp_global, warps_total);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap64 = kCount ? 0xffffffffull : (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = kCount ? nullptr : (uint8_t*)out_ptrs[c];
    uint32_t produced = 0;
    int r = kInflateBad;
    if (in_n64 <= 0xffffffffull && cap64 <= 0xffffffffull)
      r = inflate_chunk<kGzip, kCount>(in, (uint32_t)in_n64, out, (uint32_t)cap64, &produced, ws, s_crc,
                                       s_crc + (kGzip ? 256 : 0), lane);
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = r == kInflateOk ? (size_t)produced : 0;
      if (!kCount && statuses)
        statuses[c] = r == kInflateOk ? nvcompSuccess
                      : r == kInflateBadChecksum ? nvcompErrorBadChecksum : nvcompErrorCannotDecompress;
    }
    __syncwarp();
  }
}

template <bool kGzip>
static nvcompStatus_t inflate_size_async(const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
                                         size_t batch, cudaStream_t stream) {
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  const int grid = persistent_grid(kInfCtasPerSm, batch, kInfWarps);
  inflate_kernel<kGzip, true><<<grid, kInfWarps * 32, 0, stream>>>(comp_ptrs, comp_bytes, nullptr, out_sizes, batch,
                                                                   nullptr, nullptr, nullptr);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

template <bool kGzip>
static nvcompStatus_t inflate_async(const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
                                    size_t* actual_bytes, size_t batch, void* temp, size_t temp_bytes,
                                    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const int grid = persistent_grid(kInfCtasPerSm, batch, kInfWarps);
  inflate_kernel<kGzip, false><<<grid, kInfWarps * 32, 0, stream>>>(comp_ptrs, comp_bytes, out_caps, actual_bytes,
                                                                    batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedDeflateDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedDeflateGetDecompressSizeAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                          size_t* out_sizes, size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedDeflateGetDecompressSizeAsync", batch, 0, stream);
  return inflate_size_async<false>(comp_ptrs, comp_bytes, out_sizes, batch, stream);
}

nvcompStatus_t nvcompBatchedDeflateDecompressAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                   const size_t* out_caps, size_t* actual_bytes, size_t batch,
                                                   void* const temp, size_t temp_bytes, void* const* out_ptrs,
                                                   nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedDeflateDecompressAsync", batch, 0, stream);
  return inflate_async<false>(comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, temp, temp_bytes, out_ptrs,
                              statuses, stream);
}

nvcompStatus_t nvcompBatchedGzipDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedGzipGetDecompressSizeAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                       size_t* out_sizes, size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedGzipGetDecompressSizeAsync", batch, 0, stream);
  return inflate_size_async<true>(comp_ptrs, comp_bytes, out_sizes, batch, stream);
}

nvcompStatus_t nvcompBatchedGzipDecompressAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                const size_t* out_caps, size_t* actual_bytes, size_t batch,
                                                void* const temp, size_t temp_bytes, void* const* out_ptrs,
                                                nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedGzipDecompressAsync", batch, 0, stream);
  return inflate_async<true>(comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, temp, temp_bytes, out_ptrs,
                             statuses, stream);
}

}  // extern "C"
