// common.cuh -- shared device/host helpers for the H100-native batched codecs.
//
// Everything here is internal to libnvcomp.so (sm_90a only).  The public
// boundary is include/nvcomp/*.h.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#include <atomic>

#include "nvcomp/shared_types.h"
#include <ptx.cuh>   // found through -I (csrc/ for the library; tests/emu shadows it for the host emulator)
#include "nvcomp/device/detail/lz_common.cuh"

namespace b200 {

// Warp-level helpers shared with the device API (nvcomp/device/detail/lz_common.cuh)
using nvcomp::device::lz::detail::kWarp;
using nvcomp::device::lz::detail::kFull;
using nvcomp::device::lz::detail::lane_id;
using nvcomp::device::lz::detail::load_u16;
using nvcomp::device::lz::detail::load_u32;
using nvcomp::device::lz::detail::realign16;
using nvcomp::device::lz::detail::warp_copy;
using nvcomp::device::lz::detail::warp_match_copy;
using nvcomp::device::lz::detail::lz_expand_period_from_window;

// Bytes at the head of every decompress/compress workspace reserved for the
// persistent chunk scheduler (one 64-bit ticket counter per launch, padded).
constexpr size_t kSchedBytes = 256;

// ---------------------------------------------------------------------------
// Persistent chunk scheduler: every warp (or CTA) pulls the next chunk index
// from a global ticket counter, so thousands of unequal chunks keep every
// SM busy until the batch drains (no static wave quantisation).
// ---------------------------------------------------------------------------
struct WarpTicket {
  unsigned long long* counter;  // nullptr -> static grid-stride assignment
  size_t static_next;
  size_t static_stride;
  __device__ __forceinline__ WarpTicket(unsigned long long* c, size_t warp_global, size_t warps_total)
      : counter(c), static_next(warp_global), static_stride(warps_total) {}
  __device__ __forceinline__ size_t next(int lane) {
    if (counter == nullptr) {
      size_t r = static_next;
      static_next += static_stride;
      return r;
    }
    unsigned long long t = 0;
    if (lane == 0) t = atomicAdd(counter, 1ull);
    return (size_t)__shfl_sync(kFull, t, 0);
  }
};

// SM count of the current device, queried once per device (log.cu); 0 when the query fails.
int sm_count_for_current_device();

// Host-side launch helper: number of CTAs for a persistent kernel (ctas_per_sm on every SM of the current device,
// fewer when there is less work).  Correctness does not depend on it: the kernels pull chunks from a ticket or a
// grid stride, whatever the grid.
inline int persistent_grid(int ctas_per_sm, size_t work_items, int work_per_cta) {
  size_t need = (work_items + (size_t)work_per_cta - 1) / (size_t)work_per_cta;
  const int sms = sm_count_for_current_device();
  size_t cap = (size_t)(sms > 0 ? sms : 1) * (size_t)ctas_per_sm;
  size_t g = need < cap ? need : cap;
  return (int)(g == 0 ? 1 : g);
}

// Opt-in dynamic shared memory of a kernel.  The attribute is per device (and per context), so the
// "already set" memo is a per-device bitmask, updated atomically: safe from several host threads and for
// one process driving several GPUs (reference benchmarks/benchmark_allgather.cpp:359-368 pattern).
template <class Kernel>
inline cudaError_t ensure_func_attribute(Kernel kernel, cudaFuncAttribute attr, int value,
                                         std::atomic<unsigned long long>& memo) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const bool tracked = dev >= 0 && dev < 64;
  if (tracked && ((memo.load(std::memory_order_acquire) >> dev) & 1ull)) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, attr, value);
  if (e == cudaSuccess && tracked) memo.fetch_or(1ull << dev, std::memory_order_release);
  return e;
}
template <class Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kernel, int bytes, std::atomic<unsigned long long>& memo) {
  return ensure_func_attribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes, memo);
}

// Fork / join around a second kernel that should run concurrently with work on the caller's stream (the light and
// the dense LZ decode kernels of one batch: as the dense kernel's persistent CTAs drain, CTAs of the light kernel
// take their place instead of leaving the tail of the batch to a few busy SMs).  The side stream is per device and
// lives for the process; the two events are per call (recorded once, destroyed right away: CUDA releases them when
// they complete), so concurrent callers on different streams never share an event.  Works under stream capture.
cudaError_t side_stream_for_current_device(cudaStream_t* side);
struct StreamFork {
  cudaStream_t main = nullptr, side = nullptr;
  cudaEvent_t fork_ev = nullptr, join_ev = nullptr;
  cudaError_t begin(cudaStream_t stream) {
    main = stream;
    cudaError_t e = side_stream_for_current_device(&side);
    if (e != cudaSuccess) return e;
    if ((e = cudaEventCreateWithFlags(&fork_ev, cudaEventDisableTiming)) != cudaSuccess) return e;
    if ((e = cudaEventCreateWithFlags(&join_ev, cudaEventDisableTiming)) != cudaSuccess) return e;
    if ((e = cudaEventRecord(fork_ev, main)) != cudaSuccess) return e;
    return cudaStreamWaitEvent(side, fork_ev, 0);
  }
  cudaError_t end() {
    cudaError_t e = cudaEventRecord(join_ev, side);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(main, join_ev, 0);
    return e;
  }
  ~StreamFork() {
    if (fork_ev) cudaEventDestroy(fork_ev);
    if (join_ev) cudaEventDestroy(join_ev);
  }
};

// call logging (log.cu): NVCOMP_LOG_LEVEL >= 3 logs every low-level API call
int log_level();
void log_call(const char* fn, size_t batch, size_t max_chunk, const void* stream);

}  // namespace b200
namespace b200 {

#define B200_CUDA_TRY(expr)                                  \
  do {                                                       \
    cudaError_t _e = (expr);                                 \
    if (_e != cudaSuccess) return nvcompErrorCudaError;      \
  } while (0)

}  // namespace b200
