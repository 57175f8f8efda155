// zstd.cu -- batched Zstandard (RFC 8878) decompression for H100 (sm_90a) + its C ABI (include/nvcomp/zstd.h).
//
// Replaces the closed nvcompBatchedZstd* decompression entry points.  One warp decodes one chunk (zstd_decode.cuh); a
// persistent grid of CTAs pulls chunks from a ticket counter in the workspace, or walks a static grid stride without
// one.  Compression is not provided (hlif.cu reports nvcompErrorNotSupported for it).
#include "common.cuh"
#include "nvcomp/zstd.h"
#include "zstd_decode.cuh"

namespace b200 {

constexpr int kZstdWarps = 4;
// 4 x 15 872 B of per-warp tables + 1 024 B of predefined tables = 64 512 B of dynamic shared memory per CTA: 3 CTAs
// per SM fit
constexpr int kZstdCtasPerSm = 3;
constexpr size_t kZstdSmem = (size_t)kZstdWarps * kZsWarpSmem + kZsPreSmem;

// kCount: the size query (walk without writing; actual_bytes receives the decoded lengths, out_caps / out_ptrs /
// statuses are unused)
template <bool kCount>
__global__ void __launch_bounds__(kZstdWarps * 32, kZstdCtasPerSm)
zstd_kernel(const void* const* __restrict__ comp_ptrs, const size_t* __restrict__ comp_bytes, const size_t* out_caps,
            size_t* actual_bytes, size_t batch, void* const* __restrict__ out_ptrs, nvcompStatus_t* statuses,
            unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const ZstdWarp ws{smem_addr(smem + kZsPreSmem + (size_t)w * kZsWarpSmem), smem_addr(smem)};
  if (w == 0) zstd_build_predefined(ws.predef, ws.smem, lane);
  __syncthreads();
  const size_t warp_global = (size_t)blockIdx.x * kZstdWarps + w;
  WarpTicket sched(ticket, warp_global, (size_t)gridDim.x * kZstdWarps);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap64 = kCount ? 0xffffffffull : (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = kCount ? nullptr : (uint8_t*)out_ptrs[c];
    uint32_t produced = 0;
    int r = kZstdBad;
    if (in_n64 <= 0xffffffffull && cap64 <= 0xffffffffull)
      r = zstd_chunk<kCount>(in, (uint32_t)in_n64, out, (uint32_t)cap64, &produced, ws, lane);
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = r == kZstdOk ? (size_t)produced : 0;
      if (!kCount && statuses)
        statuses[c] = r == kZstdOk ? nvcompSuccess
                      : r == kZstdBadChecksum ? nvcompErrorBadChecksum : nvcompErrorCannotDecompress;
    }
    __syncwarp();
  }
}

template <bool kCount>
static nvcompStatus_t zstd_launch(const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
                                  size_t* actual_bytes, size_t batch, void* const* out_ptrs, nvcompStatus_t* statuses,
                                  unsigned long long* ticket, cudaStream_t stream) {
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(zstd_kernel<kCount>, (int)kZstdSmem, smem_set));
  const int grid = persistent_grid(kZstdCtasPerSm, batch, kZstdWarps);
  zstd_kernel<kCount><<<grid, kZstdWarps * 32, kZstdSmem, stream>>>(comp_ptrs, comp_bytes, out_caps, actual_bytes,
                                                                    batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedZstdDecompressGetTempSize(size_t batch, size_t max_chunk, size_t* temp_bytes) {
  log_call("nvcompBatchedZstdDecompressGetTempSize", batch, max_chunk, nullptr);
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedZstdGetDecompressSizeAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                       size_t* out_sizes, size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedZstdGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  return zstd_launch<true>(comp_ptrs, comp_bytes, nullptr, out_sizes, batch, nullptr, nullptr, nullptr, stream);
}

nvcompStatus_t nvcompBatchedZstdDecompressAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                const size_t* out_caps, size_t* actual_bytes, size_t batch,
                                                void* const temp, size_t temp_bytes, void* const* out_ptrs,
                                                nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedZstdDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  return zstd_launch<false>(comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket, stream);
}

}  // extern "C"
