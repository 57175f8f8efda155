// lz4frame.cu -- batched LZ4 frame-format decompression for H100 (sm_90a) + its C ABI (include/nvcomp/lz4frame.h).
//
// One warp decodes one chunk of LZ4 frames (nvcomp/device/detail/lz4frame_decode.cuh); a persistent grid of CTAs pulls
// chunks from a ticket counter in the workspace, or walks a static grid stride without one.  Each warp owns the LZ4
// block decoder's shared-memory region (ring, staging buffers, mbarrier), initialised once and carried from block to
// block and chunk to chunk.
#include "common.cuh"
#include "nvcomp/lz4frame.h"
#include "lz_decode.cuh"
#include "nvcomp/device/detail/lz4frame_decode.cuh"

namespace b200 {

using nvcomp::device::lz4frame::detail::kLz4fBadChecksum;
using nvcomp::device::lz4frame::detail::kLz4fOk;
using nvcomp::device::lz4frame::detail::lz4f_chunk;

constexpr int kLz4fWarps = 4;
// 4 x 7 248 B of per-warp regions = 28 992 B of dynamic shared memory per CTA; 5 CTAs per SM, as the LZ4 dense kernel
constexpr int kLz4fCtasPerSm = 5;
constexpr size_t kLz4fSmem = (size_t)kLz4fWarps * kLzWarpSmem;

// kCount: the size query (walk without writing; actual_bytes receives the decoded lengths, out_caps / out_ptrs /
// statuses are unused)
template <bool kCount>
__global__ void __launch_bounds__(kLz4fWarps * 32, kLz4fCtasPerSm)
lz4frame_kernel(const void* const* __restrict__ comp_ptrs, const size_t* __restrict__ comp_bytes, const size_t* out_caps,
                size_t* actual_bytes, size_t batch, void* const* __restrict__ out_ptrs, nvcompStatus_t* statuses,
                unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  uint8_t* const ring = smem + (size_t)w * kLzWarpSmem;
  lz_warp_init(smem_addr(ring), lane);
  uint32_t parity = 0;
  const size_t warp_global = (size_t)blockIdx.x * kLz4fWarps + w;
  WarpTicket sched(ticket, warp_global, (size_t)gridDim.x * kLz4fWarps);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap64 = kCount ? 0xffffffffull : (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = kCount ? nullptr : (uint8_t*)out_ptrs[c];
    uint32_t produced = 0;
    int r = nvcomp::device::lz4frame::detail::kLz4fBad;
    if (in_n64 <= 0xffffffffull && cap64 <= 0xffffffffull)
      r = lz4f_chunk<kCount>(in, (uint32_t)in_n64, out, (uint32_t)cap64, &produced, ring, parity, lane);
    __syncwarp();
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = r == kLz4fOk ? (size_t)produced : 0;
      if (!kCount && statuses)
        statuses[c] = r == kLz4fOk ? nvcompSuccess
                      : r == kLz4fBadChecksum ? nvcompErrorBadChecksum : nvcompErrorCannotDecompress;
    }
    __syncwarp();
  }
}

template <bool kCount>
static nvcompStatus_t lz4frame_launch(const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
                                      size_t* actual_bytes, size_t batch, void* const* out_ptrs,
                                      nvcompStatus_t* statuses, unsigned long long* ticket, cudaStream_t stream) {
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(lz4frame_kernel<kCount>, (int)kLz4fSmem, smem_set));
  const int grid = persistent_grid(kLz4fCtasPerSm, batch, kLz4fWarps);
  lz4frame_kernel<kCount><<<grid, kLz4fWarps * 32, kLz4fSmem, stream>>>(comp_ptrs, comp_bytes, out_caps,
                                                                        actual_bytes, batch, out_ptrs, statuses,
                                                                        ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedLZ4FrameDecompressGetTempSize(size_t batch, size_t max_chunk, size_t* temp_bytes) {
  log_call("nvcompBatchedLZ4FrameDecompressGetTempSize", batch, max_chunk, nullptr);
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedLZ4FrameGetDecompressSizeAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                           size_t* out_sizes, size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedLZ4FrameGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  return lz4frame_launch<true>(comp_ptrs, comp_bytes, nullptr, out_sizes, batch, nullptr, nullptr, nullptr, stream);
}

nvcompStatus_t nvcompBatchedLZ4FrameDecompressAsync(const void* const* comp_ptrs, const size_t* comp_bytes,
                                                    const size_t* out_caps, size_t* actual_bytes, size_t batch,
                                                    void* const temp, size_t temp_bytes, void* const* out_ptrs,
                                                    nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedLZ4FrameDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  return lz4frame_launch<false>(comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket,
                                stream);
}

}  // extern "C"
