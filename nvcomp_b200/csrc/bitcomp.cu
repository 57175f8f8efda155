// bitcomp.cu -- batched Bitcomp-style typed bit-packing codec for H100 (sm_90a) + C ABI.
//
// Replaces the closed nvcompBatchedBitcomp* entry points (include/nvcomp/bitcomp.h;
// reference benchmarks/benchmark_bitcomp_chunked.cu:114-118).  The stream and the per-block
// coder live in include/nvcomp/device/detail/bitcomp_impl.cuh, shared with the warp-level
// device API (include/nvcomp/device/bitcomp.cuh).  This file holds the batched kernels' shape:
//
// Decode: one CTA per chunk; block payload offsets come from a block-wide scan of the
// descriptor table, 512 blocks per tile; every warp then decodes whole blocks (4
// consecutive elements per lane, warp-scan for the delta prefix) -- pure streaming.
#include "common.cuh"
#include "nvcomp/bitcomp.h"
#include "nvcomp/device/detail/bitcomp_impl.cuh"

namespace b200 {

using namespace nvcomp::device::bitcomp::detail;

constexpr int kBtcWarps = 4;
constexpr int kBtcThreads = kBtcWarps * 32;
constexpr uint32_t kBtcTile = 512;           // blocks per offset tile (4 per thread)
constexpr uint32_t kBtcStage = 12288;        // bytes of packed payload staged per tile by one TMA bulk copy

// block-wide exclusive scan of 4 values per thread; returns tile total.  scratch: kBtcWarps+1 u32
__device__ __forceinline__ uint32_t btc_block_scan4(uint32_t v[4], uint32_t excl[4], uint32_t* scratch) {
  const int lane = lane_id(), w = threadIdx.x >> 5;
  uint32_t local = v[0] + v[1] + v[2] + v[3];
  uint32_t incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t o = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) scratch[w] = incl;
  __syncthreads();
  uint32_t wbase = 0, total = 0;
#pragma unroll
  for (int i = 0; i < kBtcWarps; ++i) {
    const uint32_t s = scratch[i];
    if (i < w) wbase += s;
    total += s;
  }
  uint32_t e = wbase + incl - local;
  excl[0] = e; excl[1] = e + v[0]; excl[2] = excl[1] + v[1]; excl[3] = excl[2] + v[2];
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(kBtcThreads)
bitcomp_decompress_kernel(const void* const* __restrict__ comp_ptrs,
                          const size_t* __restrict__ comp_bytes,
                          const size_t* __restrict__ out_caps,
                          size_t* actual_bytes, size_t batch,
                          void* const* __restrict__ out_ptrs,
                          nvcompStatus_t* statuses,
                          unsigned long long* ticket) {
  __shared__ uint32_t s_off[kBtcTile];
  __shared__ uint16_t s_desc[kBtcTile];
  __shared__ uint32_t s_scratch[kBtcWarps + 1];
  __shared__ unsigned long long s_chunk;
  __shared__ int s_fail;
  // packed payload of one tile, staged by a TMA bulk copy (cp.async.bulk -> mbarrier): the unpack
  // loads then hit shared memory instead of stalling on global memory (long-scoreboard was the top stall)
  __shared__ __align__(128) uint8_t s_stage[kBtcStage];
  __shared__ __align__(8) unsigned long long s_mbar;
  const uint32_t mbar = (uint32_t)__cvta_generic_to_shared(&s_mbar);
  const uint32_t stage_s = (uint32_t)__cvta_generic_to_shared(s_stage);
  uint32_t parity = 0;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  if (threadIdx.x == 0) mbar_init(mbar, 1);
  __syncthreads();
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
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    BtcHeader h;
    bool ok = btc_read_header(in, in_bytes, h);
    const uint32_t ts = ok ? btc_type_size(h.type) : 1;
    if (ok && (h.uncompressed > out_caps[c] || ((uintptr_t)out & (ts - 1)))) ok = false;
    if (ok) {
      const uint16_t* desc = (const uint16_t*)(in + 16);
      const uint32_t n_elems = h.uncompressed / ts;
      uint32_t base_off = (16u + 2u * h.nblocks + 7u) & ~7u;
      for (uint32_t tile = 0; tile < h.nblocks; tile += kBtcTile) {
        uint32_t sz[4], ex[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t b = tile + 4 * threadIdx.x + j;
          uint32_t d = 0;
          if (b < h.nblocks) d = desc[b];
          sz[j] = (b < h.nblocks) ? btc_block_bytes(h.algo, d) : 0u;
          if (btc_desc_bad(h.algo, d)) s_fail = 1;
          s_desc[4 * threadIdx.x + j] = (uint16_t)d;
        }
        const uint32_t total = btc_block_scan4(sz, ex, s_scratch);
#pragma unroll
        for (int j = 0; j < 4; ++j) s_off[4 * threadIdx.x + j] = base_off + ex[j];
        if ((uint64_t)base_off + total > in_bytes) s_fail = 1;
        __syncthreads();
        if (!s_fail) {
          const uint32_t nb = min(kBtcTile, h.nblocks - tile);
          // stage [base_off, base_off + total) (16-byte aligned span around it) if it fits
          const uint8_t* tile_src = in + base_off;
          const uint32_t delta = (uint32_t)((uintptr_t)tile_src & 15u);
          const uint32_t span = (delta + total + 15u) & ~15u;
          const bool staged = total != 0u && span <= kBtcStage;
          if (staged) {
            if (threadIdx.x == 0) {
              fence_proxy_async_smem();
              mbar_expect_tx(mbar, span);
              tma_bulk_g2s(stage_s, tile_src - delta, span, mbar);
            }
            mbar_wait(mbar, parity);
            parity ^= 1u;
          }
          const uint8_t* pay_base = staged ? (const uint8_t*)s_stage + delta - base_off : in;
          for (uint32_t b = w; b < nb; b += kBtcWarps) {
            const uint32_t blk = tile + b;
            const uint32_t e0 = blk * kBtcBlock;
            const uint32_t nv = min(kBtcBlock, n_elems - e0);
            const uint8_t* payload = pay_base + s_off[b];
            const uint32_t d = s_desc[b];
            bool bok;
            switch (ts) {
              case 1: bok = btc_decode_block<1>(h.algo, d, payload, (uint8_t*)out + e0, nv, lane); break;
              case 2: bok = btc_decode_block<2>(h.algo, d, payload, (uint16_t*)out + e0, nv, lane); break;
              case 4: bok = btc_decode_block<4>(h.algo, d, payload, (uint32_t*)out + e0, nv, lane); break;
              default: bok = btc_decode_block<8>(h.algo, d, payload, (uint64_t*)out + e0, nv, lane); break;
            }
            if (!bok && lane == 0) s_fail = 1;
          }
        }
        base_off += total;
        __syncthreads();
      }
      // trailing bytes of a chunk whose length is not a multiple of the element size: stored verbatim
      const uint32_t tail = h.uncompressed - n_elems * ts;
      if (tail) {
        if ((uint64_t)base_off + 8u > in_bytes) s_fail = 1;
        else if (threadIdx.x < tail && !s_fail) out[n_elems * ts + threadIdx.x] = in[base_off + threadIdx.x];
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const bool good = ok && !s_fail;
      if (actual_bytes) actual_bytes[c] = good ? (size_t)h.uncompressed : 0;
      if (statuses) statuses[c] = good ? nvcompSuccess : nvcompErrorCannotDecompress;
    }
    __syncthreads();
  }
}

__global__ void bitcomp_size_kernel(const void* const* __restrict__ comp_ptrs,
                                    const size_t* __restrict__ comp_bytes,
                                    size_t* out_sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= batch) return;
  BtcHeader h;
  const bool ok = btc_read_header((const uint8_t*)comp_ptrs[c], comp_bytes[c], h);
  out_sizes[c] = ok ? (size_t)h.uncompressed : 0;
}

// ---------------------------------------------------------------------------
// Compression: one CTA per chunk, two passes per 512-block tile
//   pass 1: every warp analyses whole blocks -> descriptor (bits / nz)
//   scan  : block-wide scan of payload sizes -> offsets
//   pass 2: every warp packs its blocks at their final offsets
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBtcThreads)
bitcomp_compress_kernel(const void* const* __restrict__ in_ptrs, const size_t* __restrict__ in_bytes,
                        size_t batch, void* const* __restrict__ out_ptrs, size_t* out_bytes,
                        int algo, int type, unsigned long long* ticket) {
  __shared__ uint32_t s_off[kBtcTile];
  __shared__ uint16_t s_desc[kBtcTile];
  __shared__ uint32_t s_scratch[kBtcWarps + 1];
  __shared__ unsigned long long s_words[kBtcWarps][kBtcPackWords];
  __shared__ unsigned long long s_chunk;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const uint32_t ts = btc_type_size(type);
  size_t static_next = blockIdx.x;
  while (true) {
    if (threadIdx.x == 0) s_chunk = ticket ? atomicAdd(ticket, 1ull) : (unsigned long long)static_next;
    static_next += gridDim.x;
    __syncthreads();
    const size_t c = (size_t)s_chunk;
    if (c >= batch) break;
    const uint8_t* in = (const uint8_t*)in_ptrs[c];
    const uint32_t n_bytes = (uint32_t)in_bytes[c];
    uint8_t* out = (uint8_t*)out_ptrs[c];
    __builtin_assume(__isGlobal(in)); __builtin_assume(__isGlobal(out));
    const uint32_t n_elems = n_bytes / ts;
    const uint32_t nblocks = (n_elems + kBtcBlock - 1) / kBtcBlock;
    if (threadIdx.x == 0) {
      uint32_t* hw = (uint32_t*)out;
      hw[0] = kBtcMagic; hw[1] = (uint32_t)algo | ((uint32_t)type << 8); hw[2] = n_bytes; hw[3] = nblocks;
    }
    uint16_t* desc = (uint16_t*)(out + 16);
    uint32_t base_off = (16u + 2u * nblocks + 7u) & ~7u;
    // clear the descriptor pad so the stream is deterministic
    if (threadIdx.x < 4) { const uint32_t i = nblocks + threadIdx.x; if (16u + 2u * i < base_off) desc[i] = 0; }
    for (uint32_t tile = 0; tile < nblocks; tile += kBtcTile) {
      const uint32_t nb = min(kBtcTile, nblocks - tile);
      for (uint32_t b = w; b < nb; b += kBtcWarps) {
        const uint32_t e0 = (tile + b) * kBtcBlock;
        const uint32_t nv = min(kBtcBlock, n_elems - e0);
        uint32_t d;
        switch (ts) {
          case 1: d = btc_analyse_block<1>(algo, (const uint8_t*)in + e0, nv, lane); break;
          case 2: d = btc_analyse_block<2>(algo, (const uint16_t*)in + e0, nv, lane); break;
          case 4: d = btc_analyse_block<4>(algo, (const uint32_t*)in + e0, nv, lane); break;
          default: d = btc_analyse_block<8>(algo, (const uint64_t*)in + e0, nv, lane); break;
        }
        if (lane == 0) { s_desc[b] = (uint16_t)d; desc[tile + b] = (uint16_t)d; }
      }
      __syncthreads();
      uint32_t sz[4], ex[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t b = 4 * threadIdx.x + j;
        sz[j] = (b < nb) ? btc_block_bytes(algo, s_desc[b]) : 0u;
      }
      const uint32_t total = btc_block_scan4(sz, ex, s_scratch);
#pragma unroll
      for (int j = 0; j < 4; ++j) s_off[4 * threadIdx.x + j] = base_off + ex[j];
      __syncthreads();
      for (uint32_t b = w; b < nb; b += kBtcWarps) {
        const uint32_t e0 = (tile + b) * kBtcBlock;
        const uint32_t nv = min(kBtcBlock, n_elems - e0);
        uint8_t* payload = out + s_off[b];
        const uint32_t d = s_desc[b];
        switch (ts) {
          case 1: btc_pack_block<1>(algo, d, (const uint8_t*)in + e0, nv, payload, s_words[w], lane); break;
          case 2: btc_pack_block<2>(algo, d, (const uint16_t*)in + e0, nv, payload, s_words[w], lane); break;
          case 4: btc_pack_block<4>(algo, d, (const uint32_t*)in + e0, nv, payload, s_words[w], lane); break;
          default: btc_pack_block<8>(algo, d, (const uint64_t*)in + e0, nv, payload, s_words[w], lane); break;
        }
      }
      base_off += total;
      __syncthreads();
    }
    const uint32_t tail = n_bytes - n_elems * ts;
    if (tail && threadIdx.x < 8) out[base_off + threadIdx.x] = threadIdx.x < tail ? in[n_elems * ts + threadIdx.x] : (uint8_t)0;
    if (threadIdx.x == 0) out_bytes[c] = base_off + (tail ? 8u : 0u);
    __syncthreads();
  }
}

inline nvcompStatus_t btc_check_opts(const nvcompBatchedBitcompFormatOpts& o) {
  if (btc_type_size(o.data_type) == 0) return nvcompErrorInvalidValue;
  if (o.algorithm_type < 0 || o.algorithm_type > 1) return nvcompErrorInvalidValue;
  return nvcompSuccess;
}

}  // namespace b200

using namespace b200;

extern "C" {

nvcompStatus_t nvcompBatchedBitcompCompressGetTempSize(
    size_t, size_t max_chunk, nvcompBatchedBitcompFormatOpts opts, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = btc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompBitcompCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompCompressGetTempSizeEx(
    size_t b, size_t m, nvcompBatchedBitcompFormatOpts o, size_t* t, const size_t) {
  return nvcompBatchedBitcompCompressGetTempSize(b, m, o, t);
}

nvcompStatus_t nvcompBatchedBitcompCompressGetMaxOutputChunkSize(
    size_t max_chunk, nvcompBatchedBitcompFormatOpts opts, size_t* max_compressed_bytes) {
  if (!max_compressed_bytes) return nvcompErrorInvalidValue;
  const nvcompStatus_t st = btc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompBitcompCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  const size_t ts = btc_type_size(opts.data_type);
  const size_t n = max_chunk / ts;
  const size_t nblocks = (n + kBtcBlock - 1) / kBtcBlock;
  // header + descriptors + per block: 16 bytes of header/mask + 128 elements at full width
  // (+ the trailing-bytes word)
  *max_compressed_bytes = 16 + ((2 * nblocks + 7) & ~(size_t)7) + nblocks * (16 + kBtcBlock * ts) + 16;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompCompressAsync(
    const void* const* in_ptrs, const size_t* in_bytes, size_t max_chunk, size_t batch,
    void* temp, size_t temp_bytes, void* const* out_ptrs, size_t* out_bytes,
    nvcompBatchedBitcompFormatOpts opts, cudaStream_t stream) {
  log_call("nvcompBatchedBitcompCompressAsync", batch, max_chunk, stream);
  const nvcompStatus_t st = btc_check_opts(opts);
  if (st != nvcompSuccess) return st;
  if (max_chunk > nvcompBitcompCompressionMaxAllowedChunkSize) return nvcompErrorChunkSizeTooLarge;
  if (batch == 0) return nvcompSuccess;
  if (!in_ptrs || !in_bytes || !out_ptrs || !out_bytes) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const int grid = persistent_grid(8, batch, 1);
  bitcomp_compress_kernel<<<grid, kBtcThreads, 0, stream>>>(
      in_ptrs, in_bytes, batch, out_ptrs, out_bytes, opts.algorithm_type, (int)opts.data_type, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompDecompressGetTempSize(size_t, size_t, size_t* temp_bytes) {
  if (!temp_bytes) return nvcompErrorInvalidValue;
  *temp_bytes = kSchedBytes;
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompDecompressGetTempSizeEx(size_t n, size_t m, size_t* t, size_t) {
  return nvcompBatchedBitcompDecompressGetTempSize(n, m, t);
}

nvcompStatus_t nvcompBatchedBitcompGetDecompressSizeAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, size_t* out_sizes,
    size_t batch, cudaStream_t stream) {
  log_call("nvcompBatchedBitcompGetDecompressSizeAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_sizes) return nvcompErrorInvalidValue;
  bitcomp_size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp_ptrs, comp_bytes, out_sizes, batch);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

nvcompStatus_t nvcompBatchedBitcompDecompressAsync(
    const void* const* comp_ptrs, const size_t* comp_bytes, const size_t* out_caps,
    size_t* actual_bytes, size_t batch, void* const temp, size_t temp_bytes,
    void* const* out_ptrs, nvcompStatus_t* statuses, cudaStream_t stream) {
  log_call("nvcompBatchedBitcompDecompressAsync", batch, 0, stream);
  if (batch == 0) return nvcompSuccess;
  if (!comp_ptrs || !comp_bytes || !out_caps || !out_ptrs) return nvcompErrorInvalidValue;
  unsigned long long* ticket = nullptr;
  if (temp && temp_bytes >= kSchedBytes) {
    ticket = (unsigned long long*)temp;
    B200_CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream));
  }
  const int grid = persistent_grid(12, batch, 1);
  bitcomp_decompress_kernel<<<grid, kBtcThreads, 0, stream>>>(
      comp_ptrs, comp_bytes, out_caps, actual_bytes, batch, out_ptrs, statuses, ticket);
  B200_CUDA_TRY(cudaGetLastError());
  return nvcompSuccess;
}

}  // extern "C"
