// lz_sched.cuh -- work distribution of the batched LZ4 / Snappy decoders.
//
// A batch is decoded by two kernels that run side by side (lz4.cu / snappy.cu): "light" chunks -- compressed >= 4x
// (long matches, typed run-length data) or practically incompressible (one long literal run) -- are streamed by the
// direct global-memory sequence loop at high occupancy, everything else is dense short-token data for the
// block-parallel decoder (lz_decode.cuh).  A classification pass first writes the two chunk-index lists into the
// caller's workspace; each kernel's persistent warps then pull from their own list with an atomic ticket, so a
// kernel whose list is empty retires at once instead of walking the whole batch.  Without a workspace (temp ==
// nullptr is legal for these codecs) both kernels stride over all chunks and skip the other kernel's.
//
// Each list is handed out longest first, so that no long chunk starts late and ends the call on its own.  The
// classification pass sorts the chunks into cost buckets (a counting order: one atomic per warp and bucket); a list is
// its buckets one after the other, costliest first.  Light list: run-length-like chunks (a serial chain of window
// iterations, one per run) before practically incompressible ones (a few long literal copies).  Dense list: by
// compressed bytes, the proxy for the token count, in steps of 16 KB (64 KB chunks: the price-walk column, ~34 KB,
// before the low-cardinality column, ~28 KB).
#pragma once

#include "common.cuh"
#include "nvcomp/device/detail/lz_decode.cuh"

namespace b200 {

// the light / dense rule, shared with the device API (nvcomp/device/detail/lz_decode.cuh)
using nvcomp::device::lz::detail::lz_chunk_is_light;

constexpr int kLzLightBuckets = 2;
constexpr int kLzDenseBuckets = 4;
constexpr int kLzBuckets = kLzLightBuckets + kLzDenseBuckets;   // light buckets first, then dense; costliest first
constexpr uint32_t kLzDenseBucketShift = 14;                    // dense bucket width: 16 KB of compressed input

__device__ __forceinline__ int lz_bucket(uint64_t cap, uint64_t in_n) {
  if (lz_chunk_is_light(cap, in_n)) return cap >= 4ull * in_n ? 0 : 1;
  const uint64_t q = in_n >> kLzDenseBucketShift;
  return kLzLightBuckets + (kLzDenseBuckets - 1) - (int)(q < (uint64_t)(kLzDenseBuckets - 1) ? q : kLzDenseBuckets - 1);
}

// workspace: kSchedBytes of counters | u32 bucket[kLzBuckets][batch]
struct LzLists {
  unsigned long long* ctr;      // [0] light ticket, [1] dense ticket, [2 + b] number of chunks in bucket b
  uint32_t* buckets;            // bucket b holds its chunk indices at buckets[b * batch ...]
};
constexpr size_t kLzCounterBytes = (2 + kLzBuckets) * sizeof(unsigned long long);   // what a call resets
static_assert(kLzCounterBytes <= kSchedBytes, "LZ scheduler counters exceed the reserved workspace head");
inline size_t lz_decode_temp_bytes(size_t batch) {
  return kSchedBytes + ((4 * (size_t)kLzBuckets * batch + 255) & ~(size_t)255);
}
inline LzLists lz_lists_in(void* temp, size_t temp_bytes, size_t batch) {
  LzLists l{nullptr, nullptr};
  if (temp && temp_bytes >= lz_decode_temp_bytes(batch) && batch <= 0xffffffffull) {
    l.ctr = (unsigned long long*)temp;
    l.buckets = (uint32_t*)((uint8_t*)temp + kSchedBytes);
  }
  return l;
}

// (static: one copy per translation unit that launches it)
static __global__ void __launch_bounds__(256)
lz_classify_kernel(const size_t* __restrict__ comp_bytes, const size_t* __restrict__ out_caps, size_t batch, LzLists l) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = lane_id();
  const int b = i < batch ? lz_bucket((uint64_t)out_caps[i], (uint64_t)comp_bytes[i]) : -1;
  // one atomic per warp and bucket: the lowest lane of each bucket reserves room for the warp's chunks of that
  // bucket, which are appended in lane order
  const unsigned peers = __match_any_sync(kFull, b);
  const int leader = __ffs(peers) - 1;
  unsigned long long base = 0;
  if (b >= 0 && lane == leader) base = atomicAdd(l.ctr + 2 + b, (unsigned long long)__popc(peers));
  base = __shfl_sync(kFull, base, leader);
  if (b >= 0) l.buckets[(size_t)b * batch + base + __popc(peers & ((1u << lane) - 1u))] = (uint32_t)i;
}

// A warp's source of chunk indices: its list (atomic ticket) or, without a workspace, a static stride over the batch
// filtered by class.
struct LzWork {
  const uint32_t* list;         // first bucket of this warp's list
  const unsigned long long* count;   // its bucket sizes
  unsigned long long* ticket;
  const size_t* comp_bytes;
  const size_t* out_caps;
  size_t batch, static_next, static_stride;
  bool want_light, first;
  __device__ __forceinline__ LzWork(const LzLists& l, bool light, const size_t* cb, const size_t* oc, size_t n,
                                    size_t warp_global, size_t warps_total)
      : list(l.ctr ? l.buckets + (light ? 0 : (size_t)kLzLightBuckets * n) : nullptr),
        count(l.ctr ? l.ctr + 2 + (light ? 0 : kLzLightBuckets) : nullptr),
        ticket(l.ctr ? l.ctr + (light ? 0 : 1) : nullptr), comp_bytes(cb), out_caps(oc), batch(n),
        static_next(warp_global), static_stride(warps_total), want_light(light), first(true) {}
  // next chunk of this warp, or batch when there is none
  __device__ __forceinline__ size_t next(int lane) {
    if (list) {
      // The first chunk of every warp is static (list entry = global warp index), the rest come from the ticket.  With
      // fewer chunks than resident warps this packs the work into whole CTAs -- the CTAs behind them retire at once --
      // instead of leaving every resident CTA half idle while it still holds its shared memory and registers.
      unsigned long long t;
      if (first) {
        first = false;
        t = static_next;
      } else {
        t = 0;
        if (lane == 0) t = atomicAdd(ticket, 1ull);
        t = __shfl_sync(kFull, t, 0) + static_stride;
      }
      // list entry t: walk the buckets (t is warp-uniform)
      const int nb = want_light ? kLzLightBuckets : kLzDenseBuckets;
      for (int k = 0; k < nb; ++k) {
        const unsigned long long c = count[k];
        if (t < c) return (size_t)list[(size_t)k * batch + t];
        t -= c;
      }
      return batch;
    }
    while (static_next < batch) {
      const size_t c = static_next;
      static_next += static_stride;
      if (lz_chunk_is_light((uint64_t)out_caps[c], (uint64_t)comp_bytes[c]) == want_light) return c;
    }
    return batch;
  }
};

// ---------------------------------------------------------------------------
// Schedule trace (compile with -DB200_LZ_TRACE; tools/lz_trace.py reads it).  Lane 0 of every warp records, per chunk,
// the list, the SM and the %globaltimer at the start and end of its decode, and per warp when it entered and left the
// kernel.  The records live in this translation unit's device buffers (indexed by chunk and by global warp index, so
// the last call overwrites them); B200_LZ_TRACE_EXPORT(name) adds extern "C" b200_lz_trace_{clear,fetch}_<name>.
// Without the switch every hook is empty and the decode kernels compile as if it did not exist.
// ---------------------------------------------------------------------------
#ifdef B200_LZ_TRACE
constexpr uint32_t kLzTraceChunks = 1u << 16;   // chunks beyond this index are not recorded
constexpr uint32_t kLzTraceWarps = 1u << 15;    // per list
struct LzTraceChunk { uint32_t list, smid; unsigned long long t0, t1; };        // list: 0 light, 1 dense
struct LzTraceWarp { uint32_t smid, chunks; unsigned long long t_enter, t_exit; };
static __device__ LzTraceChunk g_lz_trace_chunk[kLzTraceChunks];
static __device__ LzTraceWarp g_lz_trace_warp[2][kLzTraceWarps];

struct LzTrace {
  uint32_t list, chunks;
  unsigned long long t_enter, t0;
  __device__ __forceinline__ explicit LzTrace(bool light) : list(light ? 0u : 1u), chunks(0), t_enter(globaltimer_ns()), t0(0) {}
  __device__ __forceinline__ void chunk_begin() { t0 = globaltimer_ns(); }
  __device__ __forceinline__ void chunk_end(size_t c, int lane) {
    const unsigned long long t1 = globaltimer_ns();
    ++chunks;
    if (lane == 0 && c < kLzTraceChunks) g_lz_trace_chunk[c] = LzTraceChunk{list, sm_id(), t0, t1};
  }
  __device__ __forceinline__ void exit(size_t warp_global, int lane) {
    if (lane == 0 && warp_global < kLzTraceWarps)
      g_lz_trace_warp[list][warp_global] = LzTraceWarp{sm_id(), chunks, t_enter, globaltimer_ns()};
  }
};
#define B200_LZ_TRACE_BEGIN(light) LzTrace lz_trace_(light)
#define B200_LZ_TRACE_CHUNK_BEGIN() lz_trace_.chunk_begin()
#define B200_LZ_TRACE_CHUNK_END(c, lane) lz_trace_.chunk_end(c, lane)
#define B200_LZ_TRACE_EXIT(warp_global, lane) lz_trace_.exit(warp_global, lane)
#define B200_LZ_TRACE_EXPORT(name)                                                                              \
  extern "C" int b200_lz_trace_clear_##name() {                                                                 \
    void *c = nullptr, *w = nullptr;                                                                            \
    if (cudaGetSymbolAddress(&c, b200::g_lz_trace_chunk) != cudaSuccess) return -1;                            \
    if (cudaGetSymbolAddress(&w, b200::g_lz_trace_warp) != cudaSuccess) return -1;                             \
    if (cudaMemset(c, 0, sizeof(b200::g_lz_trace_chunk)) != cudaSuccess) return -1;                             \
    return cudaMemset(w, 0, sizeof(b200::g_lz_trace_warp)) == cudaSuccess ? 0 : -1;                             \
  }                                                                                                             \
  /* chunks: kLzTraceChunks records of 24 bytes; warps: 2 x kLzTraceWarps records of 24 bytes (light, dense) */ \
  extern "C" int b200_lz_trace_fetch_##name(void* chunks, void* warps) {                                        \
    if (cudaMemcpyFromSymbol(chunks, b200::g_lz_trace_chunk, sizeof(b200::g_lz_trace_chunk)) != cudaSuccess)    \
      return -1;                                                                                                \
    return cudaMemcpyFromSymbol(warps, b200::g_lz_trace_warp, sizeof(b200::g_lz_trace_warp)) == cudaSuccess     \
               ? 0 : -1;                                                                                        \
  }
#else
#define B200_LZ_TRACE_BEGIN(light) ((void)0)
#define B200_LZ_TRACE_CHUNK_BEGIN() ((void)0)
#define B200_LZ_TRACE_CHUNK_END(c, lane) ((void)0)
#define B200_LZ_TRACE_EXIT(warp_global, lane) ((void)0)
#define B200_LZ_TRACE_EXPORT(name)
#endif

}  // namespace b200
