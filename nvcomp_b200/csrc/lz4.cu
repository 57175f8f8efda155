// lz4.cu -- batched LZ4 block codec for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedLZ4* entry points (include/nvcomp/lz4.h).
// Wire format: LZ4 block format, one block per chunk, interoperable with
// liblz4 1.9.4 in both directions (reference examples/lz4_cpu_compression.cu,
// examples/lz4_cpu_decompression.cu).
//
// Decode: one warp owns one chunk; chunks are handed out by a persistent two-pass ticket
// scheduler (dense chunks first).  Dense short-token chunks use the lane-parallel decoder of
// lz_decode.cuh; chunks that compressed >= 4x use the direct sequence loop below (the sequence is
// parsed from a 32-byte register window, run-length matches are expanded from registers, other
// matches are 16-byte vector copies: common.cuh warp_copy / warp_match_copy).
#include "common.cuh"
#include "lz77_compress.cuh"
#include "lz4_decode.cuh"
#include "lz_sched.cuh"
#include "nvcomp/lz4.h"

namespace b200 {

// Size query: one warp walks one chunk.
__global__ void __launch_bounds__(128)
lz4_size_kernel(const void* const* __restrict__ comp_ptrs, const size_t* __restrict__ comp_bytes,
                size_t* out_sizes, size_t batch) {
  const int lane = lane_id();
  const size_t warp_global = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t warps_total = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t c = warp_global; c < batch; c += warps_total) {
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    const size_t in_n64 = comp_bytes[c];
    uint32_t produced = 0;
    bool ok = in_n64 <= 0xffffffffull;
    if (ok) ok = lz4_walk_chunk(in, (uint32_t)in_n64, &produced, lane);
    if (lane == 0) out_sizes[c] = ok ? (size_t)produced : 0;
  }
}


#ifndef LZ_DEC_WARPS
#define LZ_DEC_WARPS 4
#endif
constexpr int kLzDecWarps = LZ_DEC_WARPS;
// dense kernel: 5 CTAs x 4 warps per SM (96 registers).  On H100 this decodes the LZ4 workload 4 % faster than 7 CTAs
// (72 registers, the most shared memory allows) or 6; Snappy's dense kernel is fastest at 7 (snappy.cu).
#ifndef LZ_DEC_CTAS
#define LZ_DEC_CTAS 5
#endif
constexpr int kLzDecCtasPerSm = LZ_DEC_CTAS;
// light kernel: no shared memory, 10 CTAs x 4 warps per SM (long copies want many warps in flight)
#ifndef LZ_LIGHT_CTAS
#define LZ_LIGHT_CTAS 10
#endif
constexpr int kLzLightCtasPerSm = LZ_LIGHT_CTAS;

__global__ void __launch_bounds__(kLzDecWarps * 32, kLzLightCtasPerSm)
lz4_decompress_light_kernel(const void* const* __restrict__ comp_ptrs,
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
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap = (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    uint32_t produced = 0;
    bool ok = in_n64 <= 0xffffffffull;
    if (ok) ok = lz4_decode_chunk_direct(in, (uint32_t)in_n64, out, cap, &produced, lane);
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = ok ? (size_t)produced : 0;
      if (statuses) statuses[c] = ok ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kLzDecWarps * 32, kLzDecCtasPerSm)
lz4_decompress_v2_kernel(const void* const* __restrict__ comp_ptrs,
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
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const size_t in_n64 = comp_bytes[c];
    const uint64_t cap = (uint64_t)out_caps[c];
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    uint32_t produced = 0;
    bool ok = in_n64 <= 0xffffffffull;
    if (ok) ok = lz4_decode_chunk_v2(in, (uint32_t)in_n64, out, cap, &produced, s_ring[w], tma_parity, lane, false);
    if (lane == 0) {
      if (actual_bytes) actual_bytes[c] = ok ? (size_t)produced : 0;
      if (statuses) statuses[c] = ok ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// Compression
// ---------------------------------------------------------------------------
struct Lz4Emitter {
  uint8_t* out;
  uint32_t op;

  __device__ __forceinline__ void ext(uint32_t rem, int lane) {   // rem = len - 15
    const uint32_t nb = rem / 255u + 1u;
    for (uint32_t i = lane; i < nb; i += kWarp)
      out[op + i] = (i + 1 < nb) ? (uint8_t)255 : (uint8_t)(rem - 255u * (nb - 1));
    op += nb;
  }
  __device__ __forceinline__ void sequence(const uint8_t* lit, uint32_t ll, uint32_t off,
                                           uint32_t ml, int lane) {
    const uint32_t mlc = ml - 4;
    if (lane == 0) out[op] = (uint8_t)((min(ll, 15u) << 4) | min(mlc, 15u));
    op += 1;
    if (ll >= 15) ext(ll - 15, lane);
    if (ll) warp_copy<true>(out + op, lit, ll, lane);
    op += ll;
    if (lane == 0) { out[op] = (uint8_t)(off & 255u); out[op + 1] = (uint8_t)(off >> 8); }
    op += 2;
    if (mlc >= 15) ext(mlc - 15, lane);
  }
  __device__ __forceinline__ void finish(const uint8_t* lit, uint32_t ll, int lane) {
    if (lane == 0) out[op] = (uint8_t)(min(ll, 15u) << 4);
    op += 1;
    if (ll >= 15) ext(ll - 15, lane);
    if (ll) warp_copy<true>(out + op, lit, ll, lane);
    op += ll;
  }
};

constexpr int kCompWarpsPerCta = 4;

__global__ void __launch_bounds__(kCompWarpsPerCta * 32)
lz4_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                    size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                    uint32_t step, unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  uint16_t* table = (uint16_t*)(smem + (size_t)w * kHashBytesPerWarp);
  const size_t warp_global = (size_t)blockIdx.x * kCompWarpsPerCta + w;
  const size_t warps_total = (size_t)gridDim.x * kCompWarpsPerCta;
  WarpTicket sched(ticket, warp_global, warps_total);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    const uint32_t n = (uint32_t)in_bytes[c];
    Lz4Emitter em{(uint8_t*)out_ptrs[c], 0};
    // LZ4 end-of-block rules: last 5 bytes are literals, the last match starts
    // at least 12 bytes before the end (reference CHANGELOG.md:195).
    lz77_compress_chunk(in, n, em, table, step, 5u, 12u, lane);
    if (lane == 0) out_bytes[c] = em.op;
    __syncwarp();
  }
}

inline uint32_t lz4_step_for(nvcompType_t t, bool* ok) {
  *ok = true;
  switch (t) {
    case NVCOMP_TYPE_CHAR: case NVCOMP_TYPE_UCHAR: case NVCOMP_TYPE_BITS: return 1;
    case NVCOMP_TYPE_SHORT: case NVCOMP_TYPE_USHORT: return 2;
    case NVCOMP_TYPE_INT: case NVCOMP_TYPE_UINT: return 4;
    default: *ok = false; return 1;
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedLZ4CompressGetTempSize(
    size_t, size_t max_chunk, nvcompBatchedLZ4Opts_t opts, size_t* temp_bytes) {
  bool ok; lz4_step_for(opts.data_type, &ok);
  if (!temp_bytes || !ok) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompLZ4CompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedLZ4CompressGetTempSizeEx(
    size_t batch, size_t max_chunk, nvcompBatchedLZ4Opts_t opts, size_t* temp_bytes, const size_t) {
  return nvcompBatchedLZ4CompressGetTempSize(batch, max_chunk, opts, temp_bytes);
}

nvcompStatus_t nvcompBatchedLZ4CompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedLZ4Opts_t, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompLZ4CompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  // LZ4_compressBound: n + n/255 + 16
  *max_compressed_bytes = max_chunk + max_chunk / 255 + 16;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedLZ4CompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedLZ4Opts_t opts, cudaStream_t stream) {
  log_call("nvcompBatchedLZ4CompressAsync", batch, max_chunk, stream);
  bool ok; const uint32_t step = lz4_step_for(opts.data_type, &ok);
  if (!ok) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompLZ4CompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const size_t smem = (size_t)kCompWarpsPerCta * kHashBytesPerWarp;
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(lz4_compress_kernel, (int)smem, smem_set));
  const int grid = persistent_grid(6, batch, kCompWarpsPerCta);
  lz4_compress_kernel<<<grid, kCompWarpsPerCta * 32, smem, stream>>>(
      in_ptrs, in_bytes, batch, out_ptrs, out_bytes, step, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedLZ4DecompressGetTempSize(
    size_t batch, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = lz_decode_temp_bytes(batch);     // ticket counters + the two chunk-index lists (lz_sched.cuh)
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedLZ4DecompressGetTempSizeEx(
    size_t n, size_t m, size_t* temp_bytes, size_t) {
  return nvcompBatchedLZ4DecompressGetTempSize(n, m, temp_bytes);
}

nvcompStatus_t nvcompBatchedLZ4GetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedLZ4GetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  const int grid = persistent_grid(8, batch, 4);
  lz4_size_kernel<<<grid, 128, 0, stream>>>(comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedLZ4DecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedLZ4DecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  const LzLists lists = lz_lists_in(temp, temp_bytes, batch);
  if (lists.ctr) {
    B200_CUDA_TRY(cudaMemsetAsync(lists.ctr, 0, 4 * sizeof(unsigned long long), stream));
    lz_classify_kernel<<<(unsigned)((batch + 255) / 256), 256, 0, stream>>>(comp_bytes, out_caps, batch, lists);
  }
  // dense kernel on the caller's stream, light kernel beside it (see StreamFork): both are ordered after the ticket
  // reset above and before anything the caller enqueues next
  StreamFork fork;
  B200_CUDA_TRY(fork.begin(stream));
  const int grid = persistent_grid(kLzDecCtasPerSm, batch, kLzDecWarps);
  lz4_decompress_v2_kernel<<<grid, kLzDecWarps * 32, 0, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, lists);
  // both kernels ask for the same shared-memory carveout: an SM does not have to drain and reconfigure between a dense
  // CTA leaving and a light CTA arriving (or between back-to-back calls)
  static std::atomic<unsigned long long> carveout_set{0};
  B200_CUDA_TRY(ensure_func_attribute(lz4_decompress_light_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared, carveout_set));
  const int grid_l = persistent_grid(kLzLightCtasPerSm, batch, kLzDecWarps);
  lz4_decompress_light_kernel<<<grid_l, kLzDecWarps * 32, 0, fork.side>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, lists);
  B200_CUDA_TRY(fork.end());
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"
