// ans.cu -- batched byte-wise rANS entropy codec for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedANS* entry points (include/nvcomp/ans.h; reference
// benchmarks/benchmark_ans_chunked.cu:68-72).  The reference bitstream is undocumented,
// so this library defines its own; the stream format and its coder (header parse, LUT
// build, segment decode and encode, normalisation, layout) live in
// include/nvcomp/device/detail/ans_impl.cuh, shared with the warp-level device API
// (include/nvcomp/device/ans.cuh).  This file holds the batched kernels' shape:
//
// Decode: one CTA (4 warps) per chunk, one warp per segment, 4096-entry decode LUT
// {symbol, freq, slot - cumfreq} in shared memory (16 KB), persistent ticket scheduling.
// Compress: one CTA per chunk, every warp encodes whole segments into the CTA's scratch.
#include "common.cuh"
#include "nvcomp/ans.h"
#include "nvcomp/device/ans.cuh"

namespace b200 {

using namespace nvcomp::device::ans::detail;
constexpr int kAnsWarps = 4;
constexpr int kAnsThreads = kAnsWarps * 32;

__global__ void __launch_bounds__(kAnsThreads)
ans_decompress_kernel(const void* const* __restrict__ comp_ptrs,
                      const size_t* __restrict__ comp_bytes,
                      const size_t* __restrict__ out_caps,
                      size_t* actual_bytes, size_t batch,
                      void* const* __restrict__ out_ptrs,
                      nvcompStatus_t* statuses,
                      unsigned long long* ticket) {
  __shared__ uint32_t s_lut[kM];
  __shared__ uint32_t s_cum[257];
  __shared__ __align__(1024) uint16_t s_wring[kAnsWarps][kRingWords];   // 1 KB per warp, 1 KB aligned
  __shared__ unsigned long long s_chunk;
  __shared__ int s_fail;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const uint32_t lut = (uint32_t)__cvta_generic_to_shared(s_lut);
  const uint32_t wring = (uint32_t)__cvta_generic_to_shared(&s_wring[w][0]);
  size_t static_next = blockIdx.x;
  while (true) {
    if (threadIdx.x == 0) {
      s_chunk = ticket ? atomicAdd(ticket, 1ull) : (unsigned long long)static_next;
      s_fail = 0;
    }
    static_next += gridDim.x;
    __syncthreads();
    const size_t c = (size_t)s_chunk;
    if (c >= batch) break;
    const uint8_t* in = (const uint8_t*)comp_ptrs[c];
    const size_t in_bytes = comp_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in));      // LDG/STG instead of generic LD/ST
    __builtin_assume(__isGlobal(out));
    Header h;
    bool ok = read_header(in, in_bytes, h);
    if (ok && h.n > out_caps[c]) ok = false;
    if (ok && h.mode == 1) {
      // stored: every warp copies one contiguous slice as 16-byte vectors
      const uint32_t slice = (((h.n + kAnsWarps - 1) / kAnsWarps) + 15u) & ~15u;
      const uint32_t b0 = min((uint32_t)w * slice, h.n), b1 = min(b0 + slice, h.n);
      if (b1 > b0) warp_copy<true>(out + b0, in + 16 + b0, b1 - b0, lane);
    } else if (ok && h.mode == 2) {
      const uint8_t sym = in[16];
      for (uint32_t i = threadIdx.x; i < h.n; i += kAnsThreads) out[i] = sym;
    } else if (ok) {
      if (w == 0 && !cum_scan((const uint16_t*)(in + 16), s_cum, lane) && lane == 0) s_fail = 1;
      __syncthreads();
      if (!s_fail) {
        // warp w owns symbols 64w .. 64w+63
        for (uint32_t half = 0; half < 2; ++half)
          if (!lut_fill32(s_cum, s_lut, 64u * (uint32_t)w + 32u * half, lane)) s_fail = 1;
      }
      __syncthreads();
      if (!s_fail) {
        for (uint32_t sg = w; sg < h.nseg; sg += kAnsWarps)
          if (!decode_segment(in, in_bytes, h.n, sg, out, lut, wring, lane) && lane == 0) s_fail = 1;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const bool good = ok && !s_fail;
      if (actual_bytes) actual_bytes[c] = good ? (size_t)h.n : 0;
      if (statuses) statuses[c] = good ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    __syncthreads();
  }
}

__global__ void ans_size_kernel(const void* const* __restrict__ comp_ptrs,
                                const size_t* __restrict__ comp_bytes,
                                size_t* out_sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= batch) return;
  Header h;
  const bool ok = read_header((const uint8_t*)comp_ptrs[c], comp_bytes[c], h);
  out_sizes[c] = ok ? (size_t)h.n : 0;
}

// Compression: one CTA per chunk.  Histogram -> 12-bit normalisation -> every warp encodes whole segments
// backwards into the CTA's scratch region -> offsets -> cooperative copy into the final stream.
__global__ void __launch_bounds__(kAnsThreads)
ans_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                    size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                    uint8_t* scratch_base, size_t scratch_per_cta, unsigned long long* ticket) {
  __shared__ uint32_t s_hist[256];
  __shared__ uint16_t s_freq[256];
  __shared__ uint16_t s_cum[256];
  __shared__ uint32_t s_seg_words[1024];     // words produced per segment (chunks up to 16 MB)
  __shared__ unsigned long long s_chunk;
  __shared__ uint32_t s_mode, s_total;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  uint8_t* scratch = scratch_base + (size_t)blockIdx.x * scratch_per_cta;
  size_t static_next = blockIdx.x;
  while (true) {
    if (threadIdx.x == 0) s_chunk = ticket ? atomicAdd(ticket, 1ull) : (unsigned long long)static_next;
    static_next += gridDim.x;
    __syncthreads();
    const size_t c = (size_t)s_chunk;
    if (c >= batch) break;
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    const uint32_t n = (uint32_t)in_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    const uint32_t nseg = (n + kSeg - 1) / kSeg;
    hist_clear(s_hist, threadIdx.x, kAnsThreads);
    __syncthreads();
    hist_add(in, n, s_hist, threadIdx.x, kAnsThreads);
    __syncthreads();
    if (threadIdx.x == 0) s_mode = normalize(s_hist, s_freq, s_cum, n);
    __syncthreads();
    uint32_t mode = s_mode;
    if (mode == 0) {
      for (uint32_t sg = w; sg < nseg; sg += kAnsWarps) {
        const uint32_t begin = sg * kSeg;
        const uint32_t nw = encode_segment(in + begin, min(kSeg, n - begin), s_freq, s_cum,
                                           scratch + (size_t)sg * scratch_per_seg(), lane);
        if (lane == 0) s_seg_words[sg] = nw;
      }
    }
    __syncthreads();
    // ---- layout
    if (threadIdx.x == 0 && mode == 0) {
      uint32_t off = header_bytes(nseg);
      uint32_t* seg_off = (uint32_t*)(out + 16 + 512);
      for (uint32_t sg = 0; sg < nseg; ++sg) {
        seg_off[sg] = off;
        off += seg_bytes(s_seg_words[sg]);
      }
      seg_off[nseg] = off;
      s_total = off;
      if (off >= 16u + n) s_mode = 1;       // incompressible: store raw
    }
    __syncthreads();
    mode = s_mode;
    if (threadIdx.x == 0) write_header(out, n, mode, nseg);
    if (mode == 0) {
      write_freq(out, s_freq, threadIdx.x, kAnsThreads);
      const uint32_t* seg_off = (const uint32_t*)(out + 16 + 512);
      for (uint32_t sg = 0; sg < nseg; ++sg)
        copy_segment(out + seg_off[sg], scratch + (size_t)sg * scratch_per_seg(), s_seg_words[sg], threadIdx.x,
                     kAnsThreads);
      if (threadIdx.x == 0) out_bytes[c] = s_total;
    } else if (mode == 1) {
      copy_stored(out, in, n, threadIdx.x, kAnsThreads);
      if (threadIdx.x == 0) out_bytes[c] = 16u + n;
    } else {
      if (threadIdx.x == 0) { out[16] = in[0]; out_bytes[c] = 17; }
    }
    __syncthreads();
  }
}

inline size_t ans_scratch_per_cta(size_t max_chunk) {
  const size_t nseg = (max_chunk + kSeg - 1) / kSeg;
  return (nseg ? nseg : 1) * scratch_per_seg();
}
constexpr int kAnsMaxCompCtas = 132 * 8;   // workspace cap: 8 CTAs on each of an H100 SXM's 132 SMs

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedANSCompressGetTempSize(
    size_t batch, size_t max_chunk, nvcompBatchedANSOpts_t opts, size_t* temp_bytes) {
  if (!temp_bytes || opts.type != nvcomp_rANS) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompANSCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  size_t ctas = batch < (size_t)kAnsMaxCompCtas ? batch : (size_t)kAnsMaxCompCtas;
  const size_t per = ans_scratch_per_cta(max_chunk);
  // keep the workspace under ~2 GB for very large chunks
  const size_t budget = (size_t)2 << 30;
  if (ctas * per > budget) ctas = budget / per;
  if (ctas < 1) ctas = 1;
  *temp_bytes = kSchedBytes + ctas * per;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedANSCompressGetTempSizeEx(
    size_t b, size_t m, nvcompBatchedANSOpts_t o, size_t* t, const size_t) {
  return nvcompBatchedANSCompressGetTempSize(b, m, o, t);
}

nvcompStatus_t nvcompBatchedANSCompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedANSOpts_t, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompANSCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *max_compressed_bytes = nvcomp::device::ans::max_compressed_bytes(max_chunk);
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedANSCompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedANSOpts_t opts, cudaStream_t stream) {
  log_call("nvcompBatchedANSCompressAsync", batch, max_chunk, stream);
  if (opts.type != nvcomp_rANS) return nvcompErrorInvalidValue;
  if (max_chunk > nvcompANSCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  const size_t per = ans_scratch_per_cta(max_chunk);
  if (!temp || temp_bytes < kSchedBytes + per) return nvcompErrorInvalidValue;
  size_t ctas = (temp_bytes - kSchedBytes) / per;
  if (ctas > (size_t)kAnsMaxCompCtas) ctas = kAnsMaxCompCtas;
  if (ctas > batch) ctas = batch;
  unsigned long long* ticket = (unsigned long long*)temp;
  B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  ans_compress_kernel<<<(unsigned)ctas, kAnsThreads, 0, stream>>>(
      in_ptrs, in_bytes, batch, out_ptrs, out_bytes, (uint8_t*)temp + kSchedBytes, per, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedANSDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedANSDecompressGetTempSizeEx(size_t n, size_t m, size_t* t, size_t) {
  return nvcompBatchedANSDecompressGetTempSize(n, m, t);
}

nvcompStatus_t nvcompBatchedANSGetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedANSGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  ans_size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedANSDecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedANSDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const int grid = persistent_grid(12, batch, 1);
  ans_decompress_kernel<<<grid, kAnsThreads, 0, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"
