// ans.cu -- batched byte-wise rANS entropy codec for H100 (sm_90a) + its C ABI.
//
// Replaces the closed nvcompBatchedANS* entry points (include/nvcomp/ans.h; reference
// benchmarks/benchmark_ans_chunked.cu:68-72).  The reference bitstream is undocumented,
// so this library defines its own:
//
// Chunk stream (8-byte aligned):
//   u32 magic 'ANS1', u32 uncompressed_bytes n, u32 mode, u32 nseg
//   mode 0 (rANS):   u16 freq[256] (sum 4096, 12-bit model), u32 seg_off[nseg+1],
//                    segments (4-byte aligned): u32 state[32], then u16 words
//   mode 1 (stored): n raw bytes            (incompressible chunk)
//   mode 2 (const):  u8 symbol              (single-symbol chunk)
// A segment covers 16384 consecutive symbols; symbol i of a segment belongs to lane
// i % 32, each lane runs its own 32-bit rANS state (16-bit renormalisation), and the
// 32 states share one word stream: in every round the lanes that must renormalise
// take consecutive words in lane order (ballot + popc rank) -- the decoder never
// branches per lane and reads the stream strictly forward.
//
// Decode: one CTA (4 warps) per chunk, one warp per segment, 4096-entry decode LUT
// {symbol, freq, slot - cumfreq} in shared memory (16 KB).
#include "common.cuh"
#include "nvcomp/ans.h"

namespace b200 {

constexpr uint32_t kAnsMagic = 0x31534e41u;   // "ANS1"
constexpr int kAnsWarps = 4;
constexpr int kAnsThreads = kAnsWarps * 32;
constexpr uint32_t kAnsLog = 12;
constexpr uint32_t kAnsM = 1u << kAnsLog;
constexpr uint32_t kAnsSeg = 16384;
constexpr uint32_t kAnsLow = 1u << 16;        // state lower bound

struct AnsHeader { uint32_t n, mode, nseg; };

__device__ __forceinline__ bool ans_read_header(const uint8_t* in, size_t in_bytes, AnsHeader& h) {
  if (in_bytes < 16 || ((uintptr_t)in & 7)) return false;
  const uint32_t* w = (const uint32_t*)in;
  if (w[0] != kAnsMagic) return false;
  h.n = w[1]; h.mode = w[2]; h.nseg = w[3];
  if (h.mode > 2) return false;
  if (h.mode == 0) {
    if (h.nseg != (h.n + kAnsSeg - 1) / kAnsSeg) return false;
    if (16ull + 512ull + 4ull * (h.nseg + 1ull) > in_bytes) return false;
  } else if (h.mode == 1) {
    if (16ull + h.n > in_bytes) return false;
  } else {
    if (17 > in_bytes) return false;
  }
  return true;
}

__device__ __forceinline__ uint32_t ans_lds(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}

constexpr uint32_t kAnsRingBlocks = 8;                      // 64-word (128-byte) blocks per warp ring
constexpr uint32_t kAnsRingWords = kAnsRingBlocks * 64;     // 512 words = 1 KB per warp

__device__ __forceinline__ uint32_t ans_lds_u16(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ans_mad(uint32_t a, uint32_t b, uint32_t c) {   // one IMAD
  uint32_t d;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ void ans_cp_async4(uint32_t saddr, const void* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void ans_cp_async_wait_all() {
  asm volatile("cp.async.wait_all;" ::: "memory");
}

__global__ void __launch_bounds__(kAnsThreads)
ans_decompress_kernel(const void* const* __restrict__ comp_ptrs,
                      const size_t* __restrict__ comp_bytes,
                      const size_t* __restrict__ out_caps,
                      size_t* actual_bytes, size_t batch,
                      void* const* __restrict__ out_ptrs,
                      nvcompStatus_t* statuses,
                      unsigned long long* ticket) {
  __shared__ uint32_t s_lut[kAnsM];
  __shared__ uint32_t s_cum[257];
  __shared__ __align__(1024) uint16_t s_wring[kAnsWarps][kAnsRingWords];   // 1 KB per warp, 1 KB aligned
  __shared__ unsigned long long s_chunk;
  __shared__ int s_fail;
  const int lane = lane_id();
  const int w = threadIdx.x >> 5;
  const uint32_t lut = (uint32_t)__cvta_generic_to_shared(s_lut);
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(&s_wring[0][0]);
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
    AnsHeader h;
    bool ok = ans_read_header(in, in_bytes, h);
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
      const uint16_t* freq = (const uint16_t*)(in + 16);
      // cumulative frequencies (256 entries): warp 0 scans 8 per lane
      if (w == 0) {
        uint32_t f[8], local = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) { f[j] = freq[8 * lane + j]; local += f[j]; }
        uint32_t incl = local;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t o = __shfl_up_sync(kFull, incl, d);
          if (lane >= d) incl += o;
        }
        uint32_t e = incl - local;
#pragma unroll
        for (int j = 0; j < 8; ++j) { s_cum[8 * lane + j] = e; e += f[j]; }
        if (lane == 31) { s_cum[256] = e; if (e != kAnsM) s_fail = 1; }
      }
      __syncthreads();
      if (!s_fail) {
        // fill the LUT: warp w owns symbols 64w .. 64w+63; a ballot finds the symbols that occur (a
        // low-entropy chunk uses a few dozen of the 256), then the lanes stride over each one's slots
        for (uint32_t half = 0; half < 2; ++half) {
          const uint32_t my_sym = 64u * (uint32_t)w + 32u * half + (uint32_t)lane;
          const uint32_t my_c0 = s_cum[my_sym], my_f = s_cum[my_sym + 1] - my_c0;
          if (my_f > 4095u) s_fail = 1;
          unsigned present = __ballot_sync(kFull, my_f != 0u);
          while (present) {
            const int k = __ffs(present) - 1;
            present &= present - 1u;
            const uint32_t c0 = __shfl_sync(kFull, my_c0, k), f = __shfl_sync(kFull, my_f, k);
            const uint32_t base = (64u * (uint32_t)w + 32u * half + (uint32_t)k) | ((f & 0xfffu) << 8);
            for (uint32_t i = lane; i < f; i += kWarp) s_lut[c0 + i] = base | (i << 20);
          }
        }
      }
      __syncthreads();
      if (!s_fail) {
        const uint32_t* seg_off = (const uint32_t*)(in + 16 + 512);
        for (uint32_t sg = w; sg < h.nseg; sg += kAnsWarps) {
          const uint32_t o0 = seg_off[sg], o1 = seg_off[sg + 1];
          bool sok = (o0 & 3) == 0 && o0 <= o1 && o1 <= in_bytes && o1 - o0 >= 128u;   // no 32-bit wrap
          if (sok) {
            const uint32_t begin = sg * kAnsSeg;
            const uint32_t ns = min(kAnsSeg, h.n - begin);
            uint32_t x = ((const uint32_t*)(in + o0))[lane];
            const uint32_t nwords = (o1 - o0 - 128u) >> 1;
            uint32_t wpos = 0;
            uint8_t* o = out + begin + lane;
            const unsigned lt = (1u << lane) - 1u;
            // The renormalisation words stream through a per-warp shared-memory ring (8 blocks of 64
            // words, filled by 4-byte cp.async several blocks ahead of the read position), so the
            // per-round dependent chain holds an LDS instead of a global load that misses L1 every
            // fourth round.  A malformed stream that asks for more words than it has reads stale ring
            // contents (never out of bounds) and fails the integrity check below.
            const uint32_t wring = ring0 + (uint32_t)w * (kAnsRingWords * 2u);
            const uint8_t* wbytes = in + o0 + 128;
            const uint32_t wbytes_n = nwords * 2u;
            uint32_t issued = 0;                      // 64-word blocks requested so far
            bool in_flight = false;                   // cp.async issued and not yet waited for
            auto ring_top = [&]() {
              // before a group of <= 8 rounds (<= 256 words): blocks kb .. kb+4 must be resident.
              // Common case: nothing to wait for, nothing to issue (a block lasts ~16 rounds).
              const uint32_t kb = wpos >> 6;
              if (in_flight) { ans_cp_async_wait_all(); __syncwarp(); in_flight = false; }
              if (issued < kb + kAnsRingBlocks && issued * 128u < wbytes_n) {
                bool urgent = false;
                do {
                  const uint32_t boff = issued * 128u + (uint32_t)lane * 4u;
                  if (boff < wbytes_n) ans_cp_async4(wring + (boff & (kAnsRingWords * 2u - 1u)), wbytes + boff);
                  urgent |= issued < kb + 5u;
                  ++issued;
                } while (issued < kb + kAnsRingBlocks);
                in_flight = true;
                if (urgent) { ans_cp_async_wait_all(); __syncwarp(); in_flight = false; }
              }
            };
            // full rounds: every lane decodes one symbol; straight-line, nothing predicated
            const uint32_t full = ns >> 5;
#define B200_ANS_ROUND(OFF)                                                              \
  {                                                                                      \
    const uint32_t e = ans_lds(ans_mad(x & (kAnsM - 1), 4u, lut));                       \
    o[OFF] = (uint8_t)e;                                                                 \
    x = ((e >> 8) & 0xfffu) * (x >> kAnsLog) + (e >> 20);                                \
    const bool need = x < kAnsLow;                                                       \
    const unsigned m = __ballot_sync(kFull, need);                                       \
    /* byte offset of this lane's word in the ring; the ring is 1 KB aligned: (off & mask) | base */ \
    const uint32_t boff = ans_mad(__popc(m & lt), 2u, wpos2);                            \
    const uint32_t wd = ans_lds_u16((boff & (kAnsRingWords * 2u - 2u)) | wring);         \
    x = need ? __byte_perm(wd, x, 0x5410) : x;                                           \
    wpos2 = ans_mad(__popc(m), 2u, wpos2);                                               \
  }
            uint32_t r = 0;
            uint32_t wpos2 = 0;                       // 2 * wpos (byte position in the word stream)
            for (; r + 8 <= full; r += 8) {
              wpos = wpos2 >> 1;
              ring_top();
              B200_ANS_ROUND(0) B200_ANS_ROUND(32) B200_ANS_ROUND(64) B200_ANS_ROUND(96)
              B200_ANS_ROUND(128) B200_ANS_ROUND(160) B200_ANS_ROUND(192) B200_ANS_ROUND(224)
              o += 256;
            }
            wpos = wpos2 >> 1;
            ring_top();                                // covers the < 8 remaining rounds + the tail round
            for (; r < full; ++r) {
              B200_ANS_ROUND(0)
              o += 32;
            }
            wpos = wpos2 >> 1;
#undef B200_ANS_ROUND
            // tail round (ns % 32 symbols)
            if (ns & 31u) {
              const bool active = (uint32_t)lane < (ns & 31u);
              bool need = false;
              if (active) {
                const uint32_t e = s_lut[x & (kAnsM - 1)];
                o[0] = (uint8_t)e;
                x = ((e >> 8) & 0xfffu) * (x >> kAnsLog) + (e >> 20);
                need = x < kAnsLow;
              }
              const unsigned m = __ballot_sync(kFull, need);
              const uint32_t idx = wpos + __popc(m & lt);
              const uint32_t wd = ans_lds_u16(wring + ((idx & (kAnsRingWords - 1u)) << 1));
              if (need) x = (x << 16) | wd;
              wpos += __popc(m);
            }
            ans_cp_async_wait_all();                   // nothing in flight when the ring is reused
            __syncwarp();
            // integrity: the stream must be consumed exactly and all states return to L
            const bool good = (nwords - wpos <= 1u) && (x == kAnsLow);   // <= 1: 4-byte pad word
            if (!__all_sync(kFull, good)) sok = false;
          }
          if (!sok && lane == 0) s_fail = 1;
        }
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
  AnsHeader h;
  const bool ok = ans_read_header((const uint8_t*)comp_ptrs[c], comp_bytes[c], h);
  out_sizes[c] = ok ? (size_t)h.n : 0;
}

// ---------------------------------------------------------------------------
// Compression: one CTA per chunk.  Histogram -> 12-bit normalisation -> every warp
// encodes whole segments backwards into the CTA's scratch region -> offsets ->
// cooperative copy into the final stream.
// ---------------------------------------------------------------------------
__host__ __device__ inline size_t ans_scratch_per_seg() { return 2 * (size_t)kAnsSeg + 256; }

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
    const uint32_t nseg = (n + kAnsSeg - 1) / kAnsSeg;
    // ---- histogram
    for (int i = threadIdx.x; i < 256; i += kAnsThreads) s_hist[i] = 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += kAnsThreads) atomicAdd(&s_hist[in[i]], 1u);
    __syncthreads();
    // ---- normalise to 4096 (thread 0; 256 symbols)
    if (threadIdx.x == 0) {
      uint32_t present = 0, sum = 0, best = 0, bestc = 0;
      for (int s = 0; s < 256; ++s) {
        const uint32_t cnt = s_hist[s];
        uint32_t f = 0;
        if (cnt) {
          ++present;
          f = (uint32_t)(((uint64_t)cnt * kAnsM) / n);
          if (f == 0) f = 1;
          if (cnt > bestc) { bestc = cnt; best = s; }
        }
        s_freq[s] = (uint16_t)f;
        sum += f;
      }
      uint32_t mode = 0;
      if (n == 0 || present <= 1) mode = (n == 0) ? 1u : 2u;
      else {
        if (sum < kAnsM) s_freq[best] = (uint16_t)(s_freq[best] + (kAnsM - sum));
        while (sum > kAnsM) {
          uint32_t bi = 0, bf = 0;
          for (int s = 0; s < 256; ++s) if (s_freq[s] > bf) { bf = s_freq[s]; bi = s; }
          const uint32_t dec = min(sum - kAnsM, bf - 1u);
          s_freq[bi] = (uint16_t)(bf - dec);
          sum -= dec;
        }
        uint32_t cum = 0;
        for (int s = 0; s < 256; ++s) { s_cum[s] = (uint16_t)cum; cum += s_freq[s]; }
      }
      s_mode = mode;
    }
    __syncthreads();
    uint32_t mode = s_mode;
    if (mode == 0) {
      // ---- encode segments backwards into scratch
      for (uint32_t sg = w; sg < nseg; sg += kAnsWarps) {
        const uint32_t begin = sg * kAnsSeg;
        const uint32_t ns = min(kAnsSeg, n - begin);
        uint8_t* sbase = scratch + (size_t)sg * ans_scratch_per_seg();
        uint16_t* wbuf = (uint16_t*)(sbase + 128);
        uint32_t wp = kAnsSeg;             // capacity in words: <= 1 word per symbol
        uint32_t x = kAnsLow;
        const uint32_t rounds = (ns + 31) >> 5;
        for (uint32_t r = rounds; r-- > 0;) {
          const uint32_t i = (r << 5) + lane;
          const bool active = i < ns;
          uint32_t f = 1, cm = 0;
          bool emit = false;
          if (active) {
            const uint32_t s = in[begin + i];
            f = s_freq[s]; cm = s_cum[s];
            emit = x >= (f << 20);         // x_max = ((L >> 12) << 16) * f
          }
          const unsigned m = __ballot_sync(kFull, emit);
          wp -= __popc(m);
          if (emit) {
            wbuf[wp + __popc(m & ((1u << lane) - 1u))] = (uint16_t)(x & 0xffffu);
            x >>= 16;
          }
          if (active) x = ((x / f) << kAnsLog) + (x % f) + cm;
        }
        ((uint32_t*)sbase)[lane] = x;      // final states = decoder's initial states
        if (lane == 0) {
          s_seg_words[sg] = kAnsSeg - wp;
        }
        __syncwarp();
      }
    }
    __syncthreads();
    // ---- layout
    const uint32_t hdr = 16u + 512u + 4u * (nseg + 1u);
    if (threadIdx.x == 0 && mode == 0) {
      uint32_t off = (hdr + 3u) & ~3u;
      uint32_t* seg_off = (uint32_t*)(out + 16 + 512);
      for (uint32_t sg = 0; sg < nseg; ++sg) {
        seg_off[sg] = off;
        off += 128u + ((2u * s_seg_words[sg] + 3u) & ~3u);
      }
      seg_off[nseg] = off;
      s_total = off;
      if (off >= 16u + n) s_mode = 1;       // incompressible: store raw
    }
    __syncthreads();
    mode = s_mode;
    if (threadIdx.x == 0) {
      uint32_t* hw = (uint32_t*)out;
      hw[0] = kAnsMagic; hw[1] = n; hw[2] = mode; hw[3] = (mode == 0) ? nseg : 0u;
    }
    if (mode == 0) {
      for (int i = threadIdx.x; i < 256; i += kAnsThreads) ((uint16_t*)(out + 16))[i] = s_freq[i];
      const uint32_t* seg_off = (const uint32_t*)(out + 16 + 512);
      for (uint32_t sg = 0; sg < nseg; ++sg) {
        const uint8_t* sbase = scratch + (size_t)sg * ans_scratch_per_seg();
        const uint32_t nw = s_seg_words[sg];
        const uint32_t o0 = seg_off[sg];
        // states
        if (threadIdx.x < 32) ((uint32_t*)(out + o0))[threadIdx.x] = ((const uint32_t*)sbase)[threadIdx.x];
        const uint16_t* src = (const uint16_t*)(sbase + 128) + (kAnsSeg - nw);
        uint16_t* dst = (uint16_t*)(out + o0 + 128);
        for (uint32_t i = threadIdx.x; i < nw; i += kAnsThreads) dst[i] = src[i];
        if ((nw & 1u) && threadIdx.x == 0) dst[nw] = 0;   // deterministic pad
      }
      if (threadIdx.x == 0) out_bytes[c] = s_total;
    } else if (mode == 1) {
      for (uint32_t i = threadIdx.x; i < n; i += kAnsThreads) out[16 + i] = in[i];
      if (threadIdx.x == 0) out_bytes[c] = 16u + n;
    } else {
      if (threadIdx.x == 0) { out[16] = in[0]; out_bytes[c] = 17; }
    }
    __syncthreads();
  }
}

inline size_t ans_scratch_per_cta(size_t max_chunk) {
  const size_t nseg = (max_chunk + kAnsSeg - 1) / kAnsSeg;
  return (nseg ? nseg : 1) * ans_scratch_per_seg();
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
  const size_t nseg = (max_chunk + kAnsSeg - 1) / kAnsSeg;
  // the encoder falls back to stored mode (16 + n) whenever rANS would be larger, but the
  // rANS attempt is laid out in the output's header area first
  // multiple of 8: callers lay output chunks out at i * max_compressed_bytes (reference
  // benchmarks/benchmark_template_chunked.cuh:217-232) and ANS streams must be 8-byte aligned
  *max_compressed_bytes = (16 + 512 + 4 * (nseg + 1) + max_chunk + 16 + 7) & ~(size_t)7;
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
