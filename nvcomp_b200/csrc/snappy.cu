// snappy.cu -- batched Snappy raw-format codec for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedSnappy* entry points (include/nvcomp/snappy.h;
// reference call sites benchmarks/benchmark_snappy_synth.cpp:128-266,
// benchmarks/benchmark_snappy_chunked.cu:51-55).  The decoder accepts every legal
// Snappy stream: literal tags with 0..4 length bytes and copy-1 / copy-2 / copy-4
// elements (reference CHANGELOG.md:182-184).
#include "common.cuh"
#include "lz77_compress.cuh"
#include "nvcomp/device/detail/snappy_encode.cuh"
#include "snappy_decode.cuh"
#include "lz_sched.cuh"
#include "nvcomp/snappy.h"

namespace b200 {

#ifndef LZ_DEC_WARPS
#define LZ_DEC_WARPS 4
#endif
constexpr int kLzDecWarps = LZ_DEC_WARPS;
// dense kernel: 7 CTAs x 4 warps per SM -- shared memory (ring + staged block + token records per warp) sets the limit;
// on H100 it beats 6 and 5 CTAs (more registers, fewer spills) by 1-2 % on the Snappy workload
#ifndef LZ_DEC_CTAS
#define LZ_DEC_CTAS 7
#endif
constexpr int kLzDecCtasPerSm = LZ_DEC_CTAS;
// dense persistent grid, CTAs per SM.  Below LZ_DEC_CTAS it leaves registers for light CTAs from the start: 7 x 128
// threads x 72 registers fill the register file (64 512 of 65 536) and a light CTA needs 128 x 48 = 6 144, so at 7 no
// light CTA starts on an SM before a dense CTA there retires; at 6 (55 296) one does, at 5 three.  With the lists in
// cost order 7 is still the fastest (DESIGN §3.1): fewer dense warps stretch the dense list more than the early light
// CTAs shorten the light one.
#ifndef LZ_DEC_GRID_CTAS
#define LZ_DEC_GRID_CTAS LZ_DEC_CTAS
#endif
constexpr int kLzDecGridCtasPerSm = LZ_DEC_GRID_CTAS;
// light kernel: no shared memory, 10 CTAs x 4 warps per SM (long copies want many warps in flight)
#ifndef LZ_LIGHT_CTAS
#define LZ_LIGHT_CTAS 10
#endif
constexpr int kLzLightCtasPerSm = LZ_LIGHT_CTAS;

__global__ void __launch_bounds__(kLzDecWarps * 32, kLzLightCtasPerSm)
snappy_decompress_light_kernel(const void* const* __restrict__ comp_ptrs,
                            const size_t* __restrict__ comp_bytes,
                            const size_t* __restrict__ out_caps,
                            size_t* actual_bytes, size_t batch,
                            void* const* __restrict__ out_ptrs,
                            nvcompStatus_t* statuses,
                            LzLists lists) {
  const int lane = lane_id();
  const size_t warp_global = (size_t)blockIdx.x * kLzDecWarps + (threadIdx.x >> 5);
  const size_t warps_total = (size_t)gridDim.x * kLzDecWarps;
  LzWork sched(lists, true, comp_bytes, out_caps, batch, warp_global, warps_total);
  B200_LZ_TRACE_BEGIN(true);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    B200_LZ_TRACE_CHUNK_BEGIN();
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap = (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    uint32_t produced = 0;
    bool ok = in_n64 <= 0xffffffffull;
    if (ok) ok = snappy_decode_chunk(in, (uint32_t)in_n64, out, cap, &produced, lane);
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = ok ? (size_t)produced : 0;
      if (statuses) statuses[c] = ok ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    B200_LZ_TRACE_CHUNK_END(c, lane);
    __syncwarp();
  }
  B200_LZ_TRACE_EXIT(warp_global, lane);
}

__global__ void __launch_bounds__(kLzDecWarps * 32, kLzDecCtasPerSm)
snappy_decompress_v2_kernel(const void* const* __restrict__ comp_ptrs,
                         const size_t* __restrict__ comp_bytes,
                         const size_t* __restrict__ out_caps,
                         size_t* actual_bytes, size_t batch,
                         void* const* __restrict__ out_ptrs,
                         nvcompStatus_t* statuses,
                         LzLists lists) {
  __shared__ __align__(16) uint8_t s_ring[kLzDecWarps][kLzWarpSmem];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const size_t warp_global = (size_t)blockIdx.x * kLzDecWarps + w;
  const size_t warps_total = (size_t)gridDim.x * kLzDecWarps;
  lz_warp_init(smem_addr(s_ring[w]), lane);
  uint32_t tma_parity = 0;
  LzWork sched(lists, false, comp_bytes, out_caps, batch, warp_global, warps_total);
  B200_LZ_TRACE_BEGIN(false);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    B200_LZ_TRACE_CHUNK_BEGIN();
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap = (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    uint32_t produced = 0;
    bool ok = in_n64 <= 0xffffffffull;
    if (ok) ok = snappy_decode_chunk_v2(in, (uint32_t)in_n64, out, cap, &produced, s_ring[w], tma_parity, lane, false);
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = ok ? (size_t)produced : 0;
      if (statuses) statuses[c] = ok ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    B200_LZ_TRACE_CHUNK_END(c, lane);
    __syncwarp();
  }
  B200_LZ_TRACE_EXIT(warp_global, lane);
}


// Size query: only the varint preamble is read (one thread per chunk).
__global__ void snappy_size_kernel(const void* const* __restrict__ comp_ptrs,
                                   const size_t* __restrict__ comp_bytes,
                                   size_t* out_sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= batch) return;
  const uint8_t* in = (const uint8_t*)comp_ptrs[c];
  const size_t n = comp_bytes[c];
  uint32_t ip = 0;
  uint64_t ulen = 0;
  const bool ok = n <= 0xffffffffull && snappy_read_preamble(in, (uint32_t)n, ip, ulen);
  out_sizes[c] = ok ? (size_t)ulen : 0;
}

// ---------------------------------------------------------------------------
// Compression
// ---------------------------------------------------------------------------
// the Snappy emitter of the matcher, shared with the device API (nvcomp/device/detail/snappy_encode.cuh)
using nvcomp::device::lz::detail::SnappyEmitter;
using nvcomp::device::lz::detail::snappy_compress_chunk;

constexpr int kSnappyCompWarps = 4;

__global__ void __launch_bounds__(kSnappyCompWarps * 32)
snappy_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                       size_t max_chunk, size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                       unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  uint16_t* table = (uint16_t*)(smem + (size_t)w * kHashBytesPerWarp);
  const size_t warp_global = (size_t)blockIdx.x * kSnappyCompWarps + w;
  const size_t warps_total = (size_t)gridDim.x * kSnappyCompWarps;
  WarpTicket sched(ticket, warp_global, warps_total);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    // a chunk over max_chunk gets size 0 and nothing else: its stream could outgrow the output slot the caller
    // sized with GetMaxOutputChunkSize(max_chunk)
    SnappyEmitter em{(uint8_t*)out_ptrs[c], 0};
    if (in_bytes[c] <= max_chunk) {
      em.begin((uint32_t)in_bytes[c], lane);
      snappy_compress_chunk(in, (uint32_t)in_bytes[c], em, table, lane);
    }
    if (lane == 0) out_bytes[c] = em.op;
    __syncwarp();
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedSnappyCompressGetTempSize(
    size_t, size_t max_chunk, nvcompBatchedSnappyOpts_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompSnappyCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedSnappyCompressGetTempSizeEx(
    size_t b, size_t m, nvcompBatchedSnappyOpts_t o, size_t* t, const size_t) {
  return nvcompBatchedSnappyCompressGetTempSize(b, m, o, t);
}

nvcompStatus_t nvcompBatchedSnappyCompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedSnappyOpts_t, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompSnappyCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *max_compressed_bytes = 32 + max_chunk + max_chunk / 6;   // snappy::MaxCompressedLength
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedSnappyCompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedSnappyOpts_t, cudaStream_t stream) {
  log_call("nvcompBatchedSnappyCompressAsync", batch, max_chunk, stream);
  if (max_chunk > nvcompSnappyCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const size_t smem = (size_t)kSnappyCompWarps * kHashBytesPerWarp;
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(snappy_compress_kernel, (int)smem, smem_set));
  const int grid = persistent_grid(6, batch, kSnappyCompWarps);
  snappy_compress_kernel<<<grid, kSnappyCompWarps * 32, smem, stream>>>(
      in_ptrs, in_bytes, max_chunk, batch, out_ptrs, out_bytes, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedSnappyDecompressGetTempSize(size_t batch, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = lz_decode_temp_bytes(batch);     // ticket counters + the two chunk-index lists (lz_sched.cuh)
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedSnappyDecompressGetTempSizeEx(size_t n, size_t m, size_t* t, size_t) {
  return nvcompBatchedSnappyDecompressGetTempSize(n, m, t);
}

nvcompStatus_t nvcompBatchedSnappyGetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedSnappyGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  const int threads = 128;
  snappy_size_kernel<<<(unsigned)((batch + threads - 1) / threads), threads, 0, stream>>>(
      comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedSnappyDecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedSnappyDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  const LzLists lists = lz_lists_in(temp, temp_bytes, batch);
  if (lists.ctr) {
    B200_CUDA_TRY(cudaMemsetAsync(lists.ctr, 0, kLzCounterBytes, stream));
    lz_classify_kernel<<<(unsigned)((batch + 255) / 256), 256, 0, stream>>>(comp_bytes, out_caps, batch, lists);
  }
  // dense kernel on the caller's stream, light kernel beside it (see StreamFork): both are ordered after the ticket
  // reset above and before anything the caller enqueues next
  StreamFork fork;
  B200_CUDA_TRY(fork.begin(stream));
  const int grid = persistent_grid(kLzDecGridCtasPerSm, batch, kLzDecWarps);
  snappy_decompress_v2_kernel<<<grid, kLzDecWarps * 32, 0, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, lists);
  // both kernels ask for the same shared-memory carveout: an SM does not have to drain and reconfigure between a dense
  // CTA leaving and a light CTA arriving (or between back-to-back calls)
  static std::atomic<unsigned long long> carveout_set{0};
  B200_CUDA_TRY(ensure_func_attribute(snappy_decompress_light_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared, carveout_set));
  const int grid_l = persistent_grid(kLzLightCtasPerSm, batch, kLzDecWarps);
  snappy_decompress_light_kernel<<<grid_l, kLzDecWarps * 32, 0, fork.side>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, lists);
  B200_CUDA_TRY(fork.end());
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"

B200_LZ_TRACE_EXPORT(snappy)
