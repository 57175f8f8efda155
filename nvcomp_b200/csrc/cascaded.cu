// cascaded.cu -- batched Cascaded codec (RLE x n, delta x m, frame-of-reference
// bit-packing) for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedCascaded* entry points
// (include/nvcomp/cascaded.h; reference benchmarks/benchmark_cascaded_chunked.cu:138-142).
// The stream and the per-partition coder live in include/nvcomp/device/detail/cascaded_impl.cuh,
// shared with the warp-level device API (include/nvcomp/device/cascaded.cuh).  This file holds the
// batched kernels' shape:
//
// Decode: one CTA per chunk (persistent ticket), one warp per partition; all
// layers run out of shared memory (unpack -> warp-tile prefix sums -> run
// expansion by head-flag scatter + max-scan) and the partition is written once
// with coalesced stores.
#include "common.cuh"
#include "nvcomp/cascaded.h"
#include "nvcomp/device/detail/cascaded_impl.cuh"

namespace b200 {

using namespace nvcomp::device::cascaded::detail;

constexpr int kCascWarps = 16;       // decode CTA: up to 16 warps, one partition each
#ifndef CASC_DEC_CTAS
#define CASC_DEC_CTAS 2
#endif
// decode CTAs per SM (96 KB of shared memory each).  2 CTAs cap the kernel at 64 registers and it spills; on H100 it
// is still 14 % faster than 1 CTA at 125 registers without spills
constexpr int kCascDecCtasPerSm = CASC_DEC_CTAS;
constexpr int kCascCompWarps = 4;    // compress CTA
// per-warp shared memory of the decoder: casc_decode_smem_bytes.  The CTA owns 96 KB and activates as many
// warps (<= 16) as fit: 16 for 4/8-byte elements with one layer pair and 4 KB partitions, ... 1 for a
// 16 KB partition of 1-byte elements.
constexpr uint32_t kCascSmem = 96 * 1024;

__global__ void __launch_bounds__(kCascWarps * 32, kCascDecCtasPerSm)
cascaded_decompress_kernel(const void* const* __restrict__ comp_ptrs,
                           const size_t* __restrict__ comp_bytes,
                           const size_t* __restrict__ out_caps,
                           size_t* actual_bytes, size_t batch,
                           void* const* __restrict__ out_ptrs,
                           nvcompStatus_t* statuses,
                           unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  // Chunk indices and failure flags live in a ring of three slots: thread 0 draws the ticket two chunks ahead while
  // this one decodes and parks it just before the one barrier per chunk, so no warp ever waits for the atomic.
  // The descriptor of a chunk (stream pointer and size, output pointer and capacity) is fetched one chunk ahead by
  // four lanes of warp 1 -- loads issued at the top of the loop, parked in shared memory before the barrier -- so the
  // sixteen warps do not start every chunk with a miss on the four descriptor arrays.
  __shared__ unsigned long long s_chunk[3];
  __shared__ unsigned long long s_desc[3][4];
  __shared__ int s_fail[3];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  auto load_desc = [&](size_t c, int which) -> unsigned long long {
    return which == 0 ? (unsigned long long)comp_ptrs[c] : which == 1 ? (unsigned long long)comp_bytes[c]
         : which == 2 ? (unsigned long long)out_ptrs[c] : (unsigned long long)out_caps[c];
  };
  unsigned long long static_next = blockIdx.x;
  if (threadIdx.x == 0) {
    s_chunk[0] = ticket ? atomicAdd(ticket, 1ull) : static_next;
    s_chunk[1] = ticket ? atomicAdd(ticket, 1ull) : static_next + gridDim.x;
    s_fail[0] = 0; s_fail[1] = 0;
  }
  static_next += 2ull * gridDim.x;
  __syncthreads();
  if (w == 1 && lane < 4 && s_chunk[0] < batch) s_desc[0][lane] = load_desc((size_t)s_chunk[0], lane);
  __syncthreads();
  for (uint32_t cur = 0, nxt = 1, nn = 2;; ) {
    const size_t c = (size_t)s_chunk[cur];
    if (c >= batch) break;
    // the ticket two chunks ahead is drawn now and parked before the barrier: warp 0 does not wait for the atomic
    unsigned long long drawn = static_next;
    if (threadIdx.x == 0 && ticket) drawn = atomicAdd(ticket, 1ull);
    static_next += gridDim.x;
    unsigned long long pre = 0;                        // the next chunk's descriptor word of this lane (warp 1)
    const bool pre_lane = w == 1 && lane < 4 && s_chunk[nxt] < batch;
    if (pre_lane) pre = load_desc((size_t)s_chunk[nxt], lane);
    const uint8_t* in = (const uint8_t*)s_desc[cur][0];
    const size_t in_bytes = (size_t)s_desc[cur][1];
    uint8_t* out = (uint8_t*)s_desc[cur][2];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    const size_t cap = (size_t)s_desc[cur][3];
    // the chunk header and the first 27 partition offsets in one coalesced load (lane l holds word l of the chunk);
    // fields are broadcast with shuffles: one miss instead of a header miss followed by an offset miss
    CascHeader h;
    bool ok = in_bytes >= 20 && ((uintptr_t)in & 7) == 0;
    uint32_t cw = 0;
    if (ok && 4u * (uint32_t)lane + 4u <= in_bytes) cw = __ldg((const uint32_t*)in + lane);
    ok = ok && casc_parse_header(__shfl_sync(kFull, cw, 0), __shfl_sync(kFull, cw, 1), __shfl_sync(kFull, cw, 2),
                                 __shfl_sync(kFull, cw, 3), __shfl_sync(kFull, cw, 4), in_bytes, h);
    if (ok && (h.uncompressed > cap || ((uintptr_t)out & (casc_type_size(h.type) - 1)))) ok = false;
    if (ok) {
      const uint32_t* part_off = (const uint32_t*)(in + 20);
      const uint32_t ts0 = casc_type_size(h.type);
      const uint32_t P = h.part_bytes;
      const bool two_bufs = (h.R > h.D ? h.R : h.D) > 1;
      const uint32_t need = casc_decode_smem_bytes(P, (uint32_t)(__ffs((int)ts0) - 1), two_bufs);
      const int nw = 16u * need <= kCascSmem ? kCascWarps : (int)(kCascSmem / need);   // (kCascWarps == 16)
      uint8_t* sm = smem + (size_t)w * need;
      if (w < nw) {
        for (uint32_t p = w; p < h.num_parts; p += nw) {
          uint32_t o0, o1;
          if (p + 6u < 32u) { o0 = __shfl_sync(kFull, cw, (int)(p + 5u)); o1 = __shfl_sync(kFull, cw, (int)(p + 6u)); }
          else { o0 = part_off[p]; o1 = part_off[p + 1]; }
          bool pok = casc_part_span_ok(o0, o1, in_bytes);
          if (pok) {
            const uint32_t begin = p * h.part_bytes;
            const uint32_t nbytes = min(h.part_bytes, h.uncompressed - h.uncompressed % ts0 - begin);
            switch (ts0) {
              case 1: pok = casc_decode_part<1>(in + o0, o1 - o0, out + begin, nbytes, h.R, h.D, sm, P, two_bufs, lane); break;
              case 2: pok = casc_decode_part<2>(in + o0, o1 - o0, out + begin, nbytes / 2, h.R, h.D, sm, P, two_bufs, lane); break;
              case 4: pok = casc_decode_part<4>(in + o0, o1 - o0, out + begin, nbytes / 4, h.R, h.D, sm, P, two_bufs, lane); break;
              default: pok = casc_decode_part<8>(in + o0, o1 - o0, out + begin, nbytes / 8, h.R, h.D, sm, P, two_bufs, lane); break;
            }
          }
          if (!pok && lane == 0) s_fail[cur] = 1;
          __syncwarp();
        }
      }
      // trailing bytes of a chunk whose length is not a multiple of the element size
      const uint32_t tail = h.uncompressed % ts0;
      if (tail && w == 0) {
        const uint32_t to = part_off[h.num_parts];
        if ((uint64_t)to + 8u > in_bytes) { if (lane == 0) s_fail[cur] = 1; }
        else if ((uint32_t)lane < tail) out[h.uncompressed - tail + lane] = in[to + lane];
      }
    }
    if (threadIdx.x == 0) { s_chunk[nn] = drawn; s_fail[nn] = 0; }
    if (pre_lane) s_desc[nxt][lane] = pre;
    __syncthreads();                                   // every partition of chunk c is done; the tickets are visible
    if (threadIdx.x == 0) {
      const bool good = ok && !s_fail[cur];
      const size_t c2 = (size_t)s_chunk[cur];
      if (actual_bytes) actual_bytes[c2] = good ? (size_t)h.uncompressed : 0;
      if (statuses) statuses[c2] = good ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    const uint32_t t = cur; cur = nxt; nxt = nn; nn = t;
  }
}

__global__ void cascaded_size_kernel(const void* const* __restrict__ comp_ptrs,
                                     const size_t* __restrict__ comp_bytes,
                                     size_t* out_sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= batch) return;
  CascHeader h;
  const bool ok = casc_read_header((const uint8_t*)comp_ptrs[c], comp_bytes[c], h);
  out_sizes[c] = ok ? (size_t)h.uncompressed : 0;
}

__global__ void __launch_bounds__(kCascCompWarps * 32)
cascaded_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                         size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                         nvcompBatchedCascadedOpts_t opts, uint32_t smem_per_warp,
                         unsigned long long* ticket) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  uint8_t* sm = smem + (size_t)w * smem_per_warp;
  const size_t warp_global = (size_t)blockIdx.x * (blockDim.x >> 5) + w;
  const size_t warps_total = (size_t)gridDim.x * (blockDim.x >> 5);
  WarpTicket sched(ticket, warp_global, warps_total);
  const uint32_t ts = casc_type_size(opts.type);
  const uint32_t P = (uint32_t)opts.chunk_size;
  // The chunk framing below (header words, offset table, pad word, trailing word) is repeated in the device API's
  // compress_chunk (include/nvcomp/device/cascaded.cuh); a change to the stream format changes both.
  for (size_t c = sched.next(lane); c < batch; c = sched.next(lane)) {
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    const uint32_t n = (uint32_t)in_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    const uint32_t tail = n % ts, whole = n - tail;
    const uint32_t num_parts = (whole + P - 1) / P;
    if (lane == 0) {
      uint32_t* hw = (uint32_t*)out;
      hw[0] = kCascMagic;
      hw[1] = (uint32_t)(opts.type & 0xff) | ((uint32_t)opts.num_RLEs << 8) | ((uint32_t)opts.num_deltas << 16)
              | ((uint32_t)(opts.use_bp ? 1 : 0) << 24);
      hw[2] = n; hw[3] = P; hw[4] = num_parts;
    }
    uint32_t* part_off = (uint32_t*)(out + 20);
    uint32_t off = (20u + 4u * (num_parts + 1) + 7u) & ~7u;
    // pad bytes are zero: an odd partition count leaves one word between the offset table and the first partition
    if (lane == 0 && (num_parts & 1u)) part_off[num_parts + 1] = 0u;
    for (uint32_t p = 0; p < num_parts; ++p) {
      if (lane == 0) part_off[p] = off;
      const uint32_t begin = p * P;
      const uint32_t nb = min(P, whole - begin);
      uint32_t sz;
      switch (ts) {
        case 1: sz = casc_encode_part<1>(in + begin, nb, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                         casc_type_signed(opts.type), out + off, sm, P, lane); break;
        case 2: sz = casc_encode_part<2>(in + begin, nb / 2, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                         casc_type_signed(opts.type), out + off, sm, P, lane); break;
        case 4: sz = casc_encode_part<4>(in + begin, nb / 4, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                         casc_type_signed(opts.type), out + off, sm, P, lane); break;
        default: sz = casc_encode_part<8>(in + begin, nb / 8, opts.num_RLEs, opts.num_deltas, opts.use_bp != 0,
                                          casc_type_signed(opts.type), out + off, sm, P, lane); break;
      }
      off += (sz + 7u) & ~7u;
    }
    if (lane == 0) { part_off[num_parts] = off; out_bytes[c] = off + (tail ? 8u : 0u); }
    if (tail && lane < 8) out[off + lane] = (uint32_t)lane < tail ? in[whole + lane] : (uint8_t)0;
    __syncwarp();
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedCascadedCompressGetTempSize(
    size_t, size_t max_chunk, nvcompBatchedCascadedOpts_t opts, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = casc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompCascadedCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedCompressGetTempSizeEx(
    size_t b, size_t m, nvcompBatchedCascadedOpts_t o, size_t* t, const size_t) {
  return nvcompBatchedCascadedCompressGetTempSize(b, m, o, t);
}

nvcompStatus_t nvcompBatchedCascadedCompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedCascadedOpts_t opts, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = casc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompCascadedCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *max_compressed_bytes = casc_max_output_bytes(max_chunk, opts);
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedCompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedCascadedOpts_t opts, cudaStream_t stream) {
  log_call("nvcompBatchedCascadedCompressAsync", batch, max_chunk, stream);
  const nvcompStatus_t st = casc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompCascadedCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const uint32_t per_warp = (kCascCompSmemPerWarp((uint32_t)opts.chunk_size) + 15u) & ~15u;
  int nw = (int)((220u * 1024u) / per_warp);
  if (nw > kCascCompWarps) nw = kCascCompWarps;
  if (nw < 1) return nvcompErrorInvalidValue;
  const size_t smem = (size_t)nw * per_warp;
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(cascaded_compress_kernel, 227 * 1024, smem_set));
  const int ctas_per_sm = (int)((227 * 1024) / (smem + 1024));
  const int grid = persistent_grid(ctas_per_sm < 1 ? 1 : (ctas_per_sm > 8 ? 8 : ctas_per_sm), batch, nw);
  cascaded_compress_kernel<<<grid, nw * 32, smem, stream>>>(
      in_ptrs, in_bytes, batch, out_ptrs, out_bytes, opts, per_warp, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedDecompressGetTempSizeEx(size_t n, size_t m, size_t* t, size_t) {
  return nvcompBatchedCascadedDecompressGetTempSize(n, m, t);
}

nvcompStatus_t nvcompBatchedCascadedGetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedCascadedGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  cascaded_size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedCascadedDecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedCascadedDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  static std::atomic<unsigned long long> smem_set{0};
  B200_CUDA_TRY(ensure_dynamic_smem(cascaded_decompress_kernel, (int)kCascSmem, smem_set));
  const int grid = persistent_grid(kCascDecCtasPerSm, batch, 1);
  cascaded_decompress_kernel<<<grid, kCascWarps * 32, kCascSmem, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"
