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

namespace b200 {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;

// Bytes at the head of every decompress/compress workspace reserved for the
// persistent chunk scheduler (one 64-bit ticket counter per launch, padded).
constexpr size_t kSchedBytes = 256;

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

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

// Unaligned little-endian loads from byte pointers (no alignment assumed).
__device__ __forceinline__ uint32_t load_u16(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8);
}
__device__ __forceinline__ uint32_t load_u32(const uint8_t* p) {
  uintptr_t a = (uintptr_t)p;
  const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
  uint32_t sh = (uint32_t)(a & 3) * 8;
  uint32_t lo = w[0];
  if (sh == 0) return lo;
  uint32_t hi = w[1];
  return __funnelshift_r(lo, hi, sh);
}

// Select 4 consecutive words starting at word `ws` (0..3) of an 8-word window
// and byte-shift by `bs` bits; ws/bs are warp-uniform so the switch does not
// diverge.  This is the funnel-shift realignment that lets an arbitrarily
// aligned source feed 16-byte aligned destination stores.
__device__ __forceinline__ uint4 realign16(const uint4& a, const uint4& b, uint32_t ws, uint32_t bs) {
  uint32_t w0, w1, w2, w3, w4;
  switch (ws) {
    case 0: w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; break;
    case 1: w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; break;
    case 2: w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; break;
    default: w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; break;
  }
  uint4 r;
  r.x = __funnelshift_r(w0, w1, bs);
  r.y = __funnelshift_r(w1, w2, bs);
  r.z = __funnelshift_r(w2, w3, bs);
  r.w = __funnelshift_r(w3, w4, bs);
  return r;
}

// ---------------------------------------------------------------------------
// Warp-cooperative copy of n bytes, src and dst do not overlap within the span
// being copied.  Long spans move as 16-byte vectors: destination stores are
// 16-byte aligned, the source is re-aligned with funnel shifts.  RO selects the
// non-coherent path for sources that this kernel never writes (compressed
// input); sources inside the output buffer must use coherent loads.
// Reads may touch up to 15 bytes before/after [src, src+n) but never leave the
// 16-byte granules that contain valid bytes (so they cannot fault).
// ---------------------------------------------------------------------------
template <bool RO>
__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, uint32_t n, int lane) {
  if (n < 96) {
    for (uint32_t i = lane; i < n; i += kWarp) dst[i] = src[i];
    return;
  }
  uint32_t head = (16u - (uint32_t)((uintptr_t)dst & 15)) & 15u;
  if ((uint32_t)lane < head) dst[lane] = src[lane];
  dst += head; src += head; n -= head;
  const uint32_t nvec = n >> 4;
  const uint32_t mis = (uint32_t)((uintptr_t)src & 15);
  const uint4* s16 = (const uint4*)(src - mis);
  uint4* d16 = (uint4*)dst;
  if (mis == 0) {
    // 4 vectors in flight per lane: all loads of a round are issued before the stores
    uint32_t v = lane;
    for (; v + 3 * kWarp < nvec; v += 4 * kWarp) {
      uint4 a0 = RO ? ld_nc_v4(s16 + v) : ld_v4(s16 + v);
      uint4 a1 = RO ? ld_nc_v4(s16 + v + kWarp) : ld_v4(s16 + v + kWarp);
      uint4 a2 = RO ? ld_nc_v4(s16 + v + 2 * kWarp) : ld_v4(s16 + v + 2 * kWarp);
      uint4 a3 = RO ? ld_nc_v4(s16 + v + 3 * kWarp) : ld_v4(s16 + v + 3 * kWarp);
      st_v4(d16 + v, a0); st_v4(d16 + v + kWarp, a1);
      st_v4(d16 + v + 2 * kWarp, a2); st_v4(d16 + v + 3 * kWarp, a3);
    }
    for (; v < nvec; v += kWarp) {
      uint4 a = RO ? ld_nc_v4(s16 + v) : ld_v4(s16 + v);
      st_v4(d16 + v, a);
    }
  } else {
    const uint32_t ws = mis >> 2, bs = (mis & 3) * 8;
    uint32_t v = lane;
    for (; v + kWarp < nvec; v += 2 * kWarp) {
      uint4 a0 = RO ? ld_nc_v4(s16 + v) : ld_v4(s16 + v);
      uint4 b0 = RO ? ld_nc_v4(s16 + v + 1) : ld_v4(s16 + v + 1);
      uint4 a1 = RO ? ld_nc_v4(s16 + v + kWarp) : ld_v4(s16 + v + kWarp);
      uint4 b1 = RO ? ld_nc_v4(s16 + v + kWarp + 1) : ld_v4(s16 + v + kWarp + 1);
      st_v4(d16 + v, realign16(a0, b0, ws, bs));
      st_v4(d16 + v + kWarp, realign16(a1, b1, ws, bs));
    }
    for (; v < nvec; v += kWarp) {
      uint4 a = RO ? ld_nc_v4(s16 + v) : ld_v4(s16 + v);
      uint4 b = RO ? ld_nc_v4(s16 + v + 1) : ld_v4(s16 + v + 1);
      st_v4(d16 + v, realign16(a, b, ws, bs));
    }
  }
  const uint32_t done = nvec << 4;
  const uint32_t tail = n - done;
  if ((uint32_t)lane < tail) dst[done + lane] = src[done + lane];
}

// ---------------------------------------------------------------------------
// LZ77 match copy: dst[0..len) = dst[-off .. -off+len) with the usual
// byte-serial semantics (off may be smaller than len: the pattern repeats).
// All bytes before dst are already globally visible to the warp (caller did a
// __syncwarp after the last stores).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void warp_match_copy(uint8_t* dst, uint32_t off, uint32_t len, int lane) {
  const uint8_t* src = dst - off;
  if (off >= len) {
    warp_copy<false>(dst, src, len, lane);
    return;
  }
  if (off < 32) {
    // Every output byte j equals src[j mod off]; all of src lies before dst, so
    // the lanes are independent: no intra-copy hazard, no sync between rounds.
    const bool pow2 = (off & (off - 1)) == 0;   // off in {1,2,4,8,16}
    if (pow2 && len >= 64) {
      // Periodic run (typed RLE): the period divides 16, so every 16-byte
      // aligned vector of the run is identical.  Materialise the first aligned
      // vector bytewise, then broadcast it with 16-byte stores.
      uint32_t head = ((16u - (uint32_t)((uintptr_t)dst & 15)) & 15u) + 16u;  // 16..31
      if ((uint32_t)lane < head) dst[lane] = src[lane & (off - 1)];
      __syncwarp();
      uint8_t* a = dst + head - 16;
      uint4 pat = ld_v4((const uint4*)a);
      uint32_t nvec = (len - head) >> 4;
      uint4* d16 = (uint4*)(a + 16);
      for (uint32_t v = lane; v < nvec; v += kWarp) st_v4(d16 + v, pat);
      uint32_t done = head + (nvec << 4);
      uint32_t j = done + lane;
      if (j < len) dst[j] = src[j & (off - 1)];
      return;
    }
    if (pow2) {                                   // short periodic run: j mod off is a mask
      for (uint32_t j = lane; j < len; j += kWarp) dst[j] = src[j & (off - 1)];
      return;
    }
    uint32_t r = (uint32_t)lane % off;
    const uint32_t step = 32u % off;
    for (uint32_t j = lane; j < len; j += kWarp) {
      dst[j] = src[r];
      r += step;
      if (r >= off) r -= off;
    }
    return;
  }
  // off >= 32, overlapping: copy in doubling spans, each span's source is
  // complete before the span starts (span <= k*off).
  uint32_t done = 0, span = off;
  while (done < len) {
    uint32_t n = min(span, len - done);
    warp_copy<false>(dst + done, dst + done - span, n, lane);
    done += n;
    span <<= 1;
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// Run-length expansion from a register window (the direct LZ4 / Snappy loops): a match whose period `off` (1, 2, 4 or
// 8 bytes) lies in bytes the warp already holds -- byte k of the run is window byte `b` of lane first_lane + (k mod
// off) -- is written without reading the output back: the 8-byte period is rotated to the destination alignment
// and broadcast with 16-byte stores.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void lz_expand_period_from_window(uint8_t* dst, uint32_t ml, uint32_t off, uint32_t b,
                                                             uint32_t first_lane, uint32_t ul) {
  // 8-byte period P: byte k = window lane first_lane + (k mod off)
  const uint32_t pb = __shfl_sync(kFull, b, (int)(first_lane + (ul & (off - 1u))));
  const uint32_t placed = pb << (8u * (ul & 3u));
  const uint32_t plo = __reduce_or_sync(kFull, ul < 4u ? placed : 0u);
  const uint32_t phi = __reduce_or_sync(kFull, (ul & 28u) == 4u ? placed : 0u);
  // every 16-byte aligned vector of the run holds P rotated by (-dst) & 7 bytes, twice
  const uint32_t head = (16u - (uint32_t)((uintptr_t)dst & 15u)) & 15u;
  const uint32_t r0 = head & 7u;
  const uint32_t wa = (r0 & 4u) ? phi : plo, wb = (r0 & 4u) ? plo : phi, sh = 8u * (r0 & 3u);
  uint4 v;
  v.x = __funnelshift_r(wa, wb, sh);
  v.y = __funnelshift_r(wb, wa, sh);
  v.z = v.x; v.w = v.y;
  // byte j of the run, for lanes that write single bytes (j mod 8 selects a byte of P)
  const uint32_t mine = (((ul & 4u) ? phi : plo) >> (8u * (ul & 3u))) & 0xffu;   // P[lane & 7]
  if (ml < 16u + head) {
    // short: bytes only (ml < 31)
    if (ul < ml) dst[ul] = (uint8_t)mine;
  } else {
    if (ul < head) dst[ul] = (uint8_t)mine;
    const uint32_t nvec = (ml - head) >> 4;
    uint4* d16 = (uint4*)(dst + head);
    // nvec <= 64 for matches up to ~1 KB: two predicated stores, a loop only beyond that
    if (ul < nvec) st_v4(d16 + ul, v);
    if (ul + kWarp < nvec) st_v4(d16 + ul + kWarp, v);
#pragma unroll 1
    for (uint32_t k = ul + 2u * kWarp; k < nvec; k += kWarp) st_v4(d16 + k, v);
    // ragged end (< 16 bytes): position head + 16 nvec + lane; 16 nvec = 0 mod 8
    const uint32_t j = head + (nvec << 4) + ul;
    const uint32_t jb = (((j & 4u) ? phi : plo) >> (8u * (j & 3u))) & 0xffu;
    if (j < ml) dst[j] = (uint8_t)jb;
  }
}

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
