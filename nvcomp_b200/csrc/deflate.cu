// deflate.cu -- batched Deflate (RFC 1951) compression and decompression, and Gzip (RFC 1952) decompression, for
// H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedDeflate* and nvcompBatchedGzip* decompression entry points (include/nvcomp/deflate.h,
// gzip.h; reference call site examples/gzip_gpu_decompression.cu:110-164) and the Deflate compression ones.  One warp
// decodes one chunk (inflate_decode.cuh) or encodes one chunk (deflate_compress.cuh); a persistent grid of CTAs pulls
// chunks from a ticket counter in the workspace, or walks a static grid stride without one.
#include "common.cuh"
#include "crc32.cuh"
#include "deflate_compress.cuh"
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

// ---------------------------------------------------------------------------
// Compression.  Warps per CTA and CTAs per SM per algo: algo 0 and 2 take 11 152 B of shared memory per warp (5 CTAs
// of 4 warps fit an SM), algo 1's 64 KB hash table leaves room for one CTA of 3 warps (DESIGN §3.2).
// ---------------------------------------------------------------------------
template <int kAlgo> struct DeflateLaunch { static constexpr int kWarps = 4, kCtasPerSm = 5; };
template <> struct DeflateLaunch<1> { static constexpr int kWarps = 3, kCtasPerSm = 1; };

template <int kAlgo>
__global__ void __launch_bounds__(DeflateLaunch<kAlgo>::kWarps * 32, DeflateLaunch<kAlgo>::kCtasPerSm)
deflate_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes, size_t batch,
                        void* const* __restrict__ out_ptrs, size_t* out_bytes, unsigned long long* ticket) {
  constexpr int kWarps = DeflateLaunch<kAlgo>::kWarps;
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const DeflateWarp ws = DeflateWarp::carve<kAlgo>(smem + (size_t)w * kDeflateWarpSmem<kAlgo>);
  const size_t warp_global = (size_t)blockIdx.x * kWarps + w;
  WarpTicket sched(ticket, warp_global, (size_t)gridDim.x * kWarps);
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const size_t n = in_bytes[c];
    // a chunk over the 64 KB limit is not compressed: its output size is 0, which no decoder accepts
    const uint32_t produced = n <= kDeflateMaxChunk
        ? deflate_compress_chunk<kAlgo>((const uint8_t*)in_ptrs[c], (uint32_t)n, (uint8_t*)out_ptrs[c], ws, lane)
        : 0u;
    if (lane == 0) out_bytes[c] = produced;
    __syncwarp();
  }
}

template <int kAlgo>
static nvcompStatus_t deflate_compress_launch(const void* const* in_ptrs, const size_t* in_bytes, size_t batch,
                                              void* const* out_ptrs, size_t* out_bytes, unsigned long long* ticket,
                                              cudaStream_t stream) {
  constexpr int kWarps = DeflateLaunch<kAlgo>::kWarps;
  const size_t smem = (size_t)kWarps * kDeflateWarpSmem<kAlgo>;
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(deflate_compress_kernel<kAlgo>, (int)smem, smem_set));
  const int grid = persistent_grid(DeflateLaunch<kAlgo>::kCtasPerSm, batch, kWarps);
  deflate_compress_kernel<kAlgo><<<grid, kWarps * 32, smem, stream>>>(in_ptrs, in_bytes, batch, out_ptrs, out_bytes,
                                                                      ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

static nvcompStatus_t deflate_check_opts(size_t max_chunk, nvcompBatchedDeflateOpts_t opts) {
  if (opts.algo < 0 || opts.algo > 2) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompDeflateCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  return nvcompSuccess;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedDeflateCompressGetTempSize(size_t batch, size_t max_chunk, nvcompBatchedDeflateOpts_t opts,
                                                       size_t* temp_bytes) {
  log_call("nvcompBatchedDeflateCompressGetTempSize", batch, max_chunk, nullptr);
  const nvcompStatus_t st = deflate_check_opts(max_chunk, opts);
  if (st != nvcompSuccess) return st;
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedDeflateCompressGetTempSizeEx(size_t batch, size_t max_chunk,
                                                         nvcompBatchedDeflateOpts_t opts, size_t* temp_bytes,
                                                         const size_t) {
  return nvcompBatchedDeflateCompressGetTempSize(batch, max_chunk, opts, temp_bytes);
}

nvcompStatus_t nvcompBatchedDeflateCompressGetMaxOutputChunkSize(size_t max_chunk, nvcompBatchedDeflateOpts_t opts,
                                                                 size_t* max_compressed_bytes) {
  log_call("nvcompBatchedDeflateCompressGetMaxOutputChunkSize", 0, max_chunk, nullptr);
  const nvcompStatus_t st = deflate_check_opts(max_chunk, opts);
  if (st != nvcompSuccess) return st;
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  // the stored encoding: 5 header bytes per block of up to 65 535 bytes (the encoder never writes more)
  *max_compressed_bytes = max_chunk + 5 * (max_chunk / 65535 + 1);
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedDeflateCompressAsync(const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk,
                                                 size_t batch, void* temp, size_t temp_bytes, void* const* out_ptrs,
                                                 size_t* out_bytes, nvcompBatchedDeflateOpts_t opts,
                                                 cudaStream_t stream) {
  log_call("nvcompBatchedDeflateCompressAsync", batch, max_chunk, stream);
  const nvcompStatus_t st = deflate_check_opts(max_chunk, opts);
  if (st != nvcompSuccess) return st;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  switch (opts.algo) {
    case 0: return deflate_compress_launch<0>(in_ptrs, in_bytes, batch, out_ptrs, out_bytes, ticket, stream);
    case 1: return deflate_compress_launch<1>(in_ptrs, in_bytes, batch, out_ptrs, out_bytes, ticket, stream);
    default: return deflate_compress_launch<2>(in_ptrs, in_bytes, batch, out_ptrs, out_bytes, ticket, stream);
  }
}

nvcompStatus_t nvcompBatchedDeflateDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedDeflateDecompressGetTempSizeEx(size_t batch, size_t max_chunk, size_t* temp_bytes,
                                                           const size_t) {
  return nvcompBatchedDeflateDecompressGetTempSize(batch, max_chunk, temp_bytes);
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
