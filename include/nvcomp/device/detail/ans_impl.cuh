// nvcomp/device/detail/ans_impl.cuh -- the ANS stream coder, shared by the batched kernels (nvcomp_b200/csrc/ans.cu)
// and the warp-level device API (nvcomp/device/ans.cuh).  Header-only device code for sm_90a; not a public interface.
//
// Chunk stream (8-byte aligned; this library's own format, the reference's is undocumented):
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
// Every function here is called by whole warps; the callers own the shared memory (passed as pointers or as
// shared-window addresses) and the barriers between the phases.  `tid` / `nthreads` name the cooperating threads of
// the cooperative loops (a CTA in the batched kernels, one warp in the device API).
#pragma once

#include <stddef.h>
#include <stdint.h>

namespace nvcomp {
namespace device {
namespace ans {
namespace detail {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr uint32_t kMagic = 0x31534e41u;   // "ANS1"
constexpr uint32_t kLog = 12;
constexpr uint32_t kM = 1u << kLog;
constexpr uint32_t kSeg = 16384;
constexpr uint32_t kLow = 1u << 16;        // state lower bound
constexpr uint32_t kRingBlocks = 8;                   // 64-word (128-byte) blocks per warp ring
constexpr uint32_t kRingWords = kRingBlocks * 64;     // 512 words
constexpr uint32_t kRingBytes = kRingWords * 2;       // 1 KB per warp; the ring must be kRingBytes aligned

struct Header { uint32_t n, mode, nseg; };

// Bytes before the first segment of a mode-0 stream.
__host__ __device__ constexpr uint32_t header_bytes(uint32_t nseg) { return 16u + 512u + 4u * (nseg + 1u); }
// Bytes of a segment holding `words` renormalisation words (states, words, pad to 4 bytes).
__host__ __device__ constexpr uint32_t seg_bytes(uint32_t words) { return 128u + ((2u * words + 3u) & ~3u); }
// Encoder scratch of one segment: 32 states, then room for one word per symbol.
__host__ __device__ constexpr size_t scratch_per_seg() { return 2 * (size_t)kSeg + 256; }

__device__ __forceinline__ bool read_header(const uint8_t* in, size_t in_bytes, Header& h) {
  if (in_bytes < 16 || ((uintptr_t)in & 7)) return false;
  const uint32_t* w = (const uint32_t*)in;
  if (w[0] != kMagic) return false;
  h.n = w[1]; h.mode = w[2]; h.nseg = w[3];
  if (h.mode > 2) return false;
  if (h.mode == 0) {
    if (h.nseg != (h.n + kSeg - 1) / kSeg) return false;
    if (16ull + 512ull + 4ull * (h.nseg + 1ull) > in_bytes) return false;
  } else if (h.mode == 1) {
    if (16ull + h.n > in_bytes) return false;
  } else {
    if (17 > in_bytes) return false;
  }
  return true;
}

__device__ __forceinline__ uint32_t lds(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t mad(uint32_t a, uint32_t b, uint32_t c) {   // one IMAD
  uint32_t d;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ void cp_async4(uint32_t saddr, const void* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.wait_all;" ::: "memory");
}

// ---------------------------------------------------------------------------
// Decode
// ---------------------------------------------------------------------------

// Cumulative frequencies of the 256-entry table `freq` into s_cum[0..256], 8 symbols per lane.  One warp.
// Returns (warp-uniform) whether the frequencies sum to 4096.
__device__ __forceinline__ bool cum_scan(const uint16_t* freq, uint32_t* s_cum, int lane) {
  uint32_t f[8], local = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) { f[j] = freq[8 * lane + j]; local += f[j]; }
  uint32_t incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(kFullMask, incl, d);
    if (lane >= d) incl += o;
  }
  uint32_t e = incl - local;
#pragma unroll
  for (int j = 0; j < 8; ++j) { s_cum[8 * lane + j] = e; e += f[j]; }
  if (lane == 31) s_cum[256] = e;
  return __shfl_sync(kFullMask, e, 31) == kM;
}

// Decode-LUT entries {symbol, freq, slot - cumfreq} of symbols sym0 .. sym0+31.  One warp: a ballot finds the
// symbols that occur (a low-entropy chunk uses a few dozen of the 256), then the lanes stride over each one's
// slots.  Returns false in the lane whose symbol has a frequency above 4095 (not warp-uniform).
__device__ __forceinline__ bool lut_fill32(const uint32_t* s_cum, uint32_t* s_lut, uint32_t sym0, int lane) {
  const uint32_t my_sym = sym0 + (uint32_t)lane;
  const uint32_t my_c0 = s_cum[my_sym], my_f = s_cum[my_sym + 1] - my_c0;
  unsigned present = __ballot_sync(kFullMask, my_f != 0u);
  while (present) {
    const int k = __ffs(present) - 1;
    present &= present - 1u;
    const uint32_t c0 = __shfl_sync(kFullMask, my_c0, k), f = __shfl_sync(kFullMask, my_f, k);
    const uint32_t base = (sym0 + (uint32_t)k) | ((f & 0xfffu) << 8);
    for (uint32_t i = lane; i < f; i += 32) s_lut[c0 + i] = base | (i << 20);
  }
  return my_f <= 4095u;
}

// Decode segment `sg` of the mode-0 stream `in` (header already validated, LUT built) into out + sg * kSeg.  One
// warp.  `lut` is the shared-window address of the 4096-entry LUT, `wring` that of this warp's kRingBytes-aligned
// word ring.  `in` and `out` are global memory.  Returns (warp-uniform) whether the segment is intact: offsets in
// bounds, the word stream consumed exactly and every state back at kLow.  Reads stay inside [in, in + in_bytes);
// writes stay inside the segment's own n bytes of output.
__device__ __forceinline__ bool decode_segment(const uint8_t* in, size_t in_bytes, uint32_t n, uint32_t sg,
                                               uint8_t* out, uint32_t lut, uint32_t wring, int lane) {
  __builtin_assume(__isGlobal(in));      // LDG/STG instead of generic LD/ST
  __builtin_assume(__isGlobal(out));
  const uint32_t* seg_off = (const uint32_t*)(in + 16 + 512);
  const uint32_t o0 = seg_off[sg], o1 = seg_off[sg + 1];
  if (!((o0 & 3) == 0 && o0 <= o1 && o1 <= in_bytes && o1 - o0 >= 128u)) return false;   // no 32-bit wrap
  const uint32_t begin = sg * kSeg;
  const uint32_t ns = min(kSeg, n - begin);
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
  const uint8_t* wbytes = in + o0 + 128;
  const uint32_t wbytes_n = nwords * 2u;
  uint32_t issued = 0;                      // 64-word blocks requested so far
  bool in_flight = false;                   // cp.async issued and not yet waited for
  auto ring_top = [&]() {
    // before a group of <= 8 rounds (<= 256 words): blocks kb .. kb+4 must be resident.
    // Common case: nothing to wait for, nothing to issue (a block lasts ~16 rounds).
    const uint32_t kb = wpos >> 6;
    if (in_flight) { cp_async_wait_all(); __syncwarp(); in_flight = false; }
    if (issued < kb + kRingBlocks && issued * 128u < wbytes_n) {
      bool urgent = false;
      do {
        const uint32_t boff = issued * 128u + (uint32_t)lane * 4u;
        if (boff < wbytes_n) cp_async4(wring + (boff & (kRingBytes - 1u)), wbytes + boff);
        urgent |= issued < kb + 5u;
        ++issued;
      } while (issued < kb + kRingBlocks);
      in_flight = true;
      if (urgent) { cp_async_wait_all(); __syncwarp(); in_flight = false; }
    }
  };
  // full rounds: every lane decodes one symbol; straight-line, nothing predicated
  const uint32_t full = ns >> 5;
#define NVCOMP_ANS_ROUND(OFF)                                                            \
  {                                                                                      \
    const uint32_t e = lds(mad(x & (kM - 1), 4u, lut));                                  \
    o[OFF] = (uint8_t)e;                                                                 \
    x = ((e >> 8) & 0xfffu) * (x >> kLog) + (e >> 20);                                   \
    const bool need = x < kLow;                                                          \
    const unsigned m = __ballot_sync(kFullMask, need);                                   \
    /* byte offset of this lane's word in the ring; the ring is 1 KB aligned: (off & mask) | base */ \
    const uint32_t boff = mad(__popc(m & lt), 2u, wpos2);                                \
    const uint32_t wd = lds_u16((boff & (kRingBytes - 2u)) | wring);                     \
    x = need ? __byte_perm(wd, x, 0x5410) : x;                                           \
    wpos2 = mad(__popc(m), 2u, wpos2);                                                   \
  }
  uint32_t r = 0;
  uint32_t wpos2 = 0;                       // 2 * wpos (byte position in the word stream)
  for (; r + 8 <= full; r += 8) {
    wpos = wpos2 >> 1;
    ring_top();
    NVCOMP_ANS_ROUND(0) NVCOMP_ANS_ROUND(32) NVCOMP_ANS_ROUND(64) NVCOMP_ANS_ROUND(96)
    NVCOMP_ANS_ROUND(128) NVCOMP_ANS_ROUND(160) NVCOMP_ANS_ROUND(192) NVCOMP_ANS_ROUND(224)
    o += 256;
  }
  wpos = wpos2 >> 1;
  ring_top();                                // covers the < 8 remaining rounds + the tail round
  for (; r < full; ++r) {
    NVCOMP_ANS_ROUND(0)
    o += 32;
  }
  wpos = wpos2 >> 1;
#undef NVCOMP_ANS_ROUND
  // tail round (ns % 32 symbols)
  if (ns & 31u) {
    const bool active = (uint32_t)lane < (ns & 31u);
    bool need = false;
    if (active) {
      const uint32_t e = lds(mad(x & (kM - 1), 4u, lut));
      o[0] = (uint8_t)e;
      x = ((e >> 8) & 0xfffu) * (x >> kLog) + (e >> 20);
      need = x < kLow;
    }
    const unsigned m = __ballot_sync(kFullMask, need);
    const uint32_t idx = wpos + __popc(m & lt);
    const uint32_t wd = lds_u16(wring + ((idx & (kRingWords - 1u)) << 1));
    if (need) x = (x << 16) | wd;
    wpos += __popc(m);
  }
  cp_async_wait_all();                       // nothing in flight when the ring is reused
  __syncwarp();
  // integrity: the stream must be consumed exactly and all states return to L
  const bool good = (nwords - wpos <= 1u) && (x == kLow);   // <= 1: 4-byte pad word
  return __all_sync(kFullMask, good);
}

// ---------------------------------------------------------------------------
// Encode: histogram -> 12-bit normalisation (which also picks the mode) -> each segment encoded backwards into
// scratch -> segment offsets -> stream assembly.
// ---------------------------------------------------------------------------

__device__ __forceinline__ void hist_clear(uint32_t* s_hist, int tid, int nthreads) {
  for (int i = tid; i < 256; i += nthreads) s_hist[i] = 0;
}
__device__ __forceinline__ void hist_add(const uint8_t* in, uint32_t n, uint32_t* s_hist, int tid, int nthreads) {
  for (uint32_t i = tid; i < n; i += nthreads) atomicAdd(&s_hist[in[i]], 1u);
}

// Normalise the histogram of n bytes to frequencies summing to 4096 and their cumulative sums.  One thread.
// Returns the stream mode the histogram allows: 0 (rANS), 1 (stored; only for n == 0 here -- the caller
// switches to 1 when the rANS stream turns out no smaller), 2 (one symbol).
__device__ __forceinline__ uint32_t normalize(const uint32_t* s_hist, uint16_t* s_freq, uint16_t* s_cum, uint32_t n) {
  uint32_t present = 0, sum = 0, best = 0, bestc = 0;
  for (int s = 0; s < 256; ++s) {
    const uint32_t cnt = s_hist[s];
    uint32_t f = 0;
    if (cnt) {
      ++present;
      f = (uint32_t)(((uint64_t)cnt * kM) / n);
      if (f == 0) f = 1;
      if (cnt > bestc) { bestc = cnt; best = s; }
    }
    s_freq[s] = (uint16_t)f;
    sum += f;
  }
  if (n == 0 || present <= 1) return (n == 0) ? 1u : 2u;
  if (sum < kM) s_freq[best] = (uint16_t)(s_freq[best] + (kM - sum));
  while (sum > kM) {
    uint32_t bi = 0, bf = 0;
    for (int s = 0; s < 256; ++s) if (s_freq[s] > bf) { bf = s_freq[s]; bi = s; }
    const uint32_t dec = min(sum - kM, bf - 1u);
    s_freq[bi] = (uint16_t)(bf - dec);
    sum -= dec;
  }
  uint32_t cum = 0;
  for (int s = 0; s < 256; ++s) { s_cum[s] = (uint16_t)cum; cum += s_freq[s]; }
  return 0;
}

// Encode the ns <= kSeg symbols at `in` backwards into `sbase` (scratch_per_seg() bytes, 4-byte aligned): the 32
// final states at sbase, the words at the end of the word area.  One warp; ends with __syncwarp so the scratch may
// be read by any lane.  Returns (warp-uniform) the number of words.
__device__ __forceinline__ uint32_t encode_segment(const uint8_t* in, uint32_t ns, const uint16_t* s_freq,
                                                   const uint16_t* s_cum, uint8_t* sbase, int lane) {
  uint16_t* wbuf = (uint16_t*)(sbase + 128);
  uint32_t wp = kSeg;                // capacity in words: <= 1 word per symbol
  uint32_t x = kLow;
  const uint32_t rounds = (ns + 31) >> 5;
  for (uint32_t r = rounds; r-- > 0;) {
    const uint32_t i = (r << 5) + lane;
    const bool active = i < ns;
    uint32_t f = 1, cm = 0;
    bool emit = false;
    if (active) {
      const uint32_t s = in[i];
      f = s_freq[s]; cm = s_cum[s];
      emit = x >= (f << 20);         // x_max = ((L >> 12) << 16) * f
    }
    const unsigned m = __ballot_sync(kFullMask, emit);
    wp -= __popc(m);
    if (emit) {
      wbuf[wp + __popc(m & ((1u << lane) - 1u))] = (uint16_t)(x & 0xffffu);
      x >>= 16;
    }
    if (active) x = ((x / f) << kLog) + (x % f) + cm;
  }
  ((uint32_t*)sbase)[lane] = x;      // final states = decoder's initial states
  __syncwarp();
  return kSeg - wp;
}

// The 16-byte stream header.  One thread.
__device__ __forceinline__ void write_header(uint8_t* out, uint32_t n, uint32_t mode, uint32_t nseg) {
  uint32_t* hw = (uint32_t*)out;
  hw[0] = kMagic; hw[1] = n; hw[2] = mode; hw[3] = (mode == 0) ? nseg : 0u;
}
// The frequency table of a mode-0 stream.
__device__ __forceinline__ void write_freq(uint8_t* out, const uint16_t* s_freq, int tid, int nthreads) {
  for (int i = tid; i < 256; i += nthreads) ((uint16_t*)(out + 16))[i] = s_freq[i];
}
// Segment of `nw` words from the scratch `sbase` to its place `dst` in the stream (seg_bytes(nw) bytes).
__device__ __forceinline__ void copy_segment(uint8_t* dst, const uint8_t* sbase, uint32_t nw, int tid, int nthreads) {
  if (tid < 32) ((uint32_t*)dst)[tid] = ((const uint32_t*)sbase)[tid];
  const uint16_t* src = (const uint16_t*)(sbase + 128) + (kSeg - nw);
  uint16_t* dw = (uint16_t*)(dst + 128);
  for (uint32_t i = tid; i < nw; i += nthreads) dw[i] = src[i];
  if ((nw & 1u) && tid == 0) dw[nw] = 0;   // deterministic pad
}
// The payload of a mode-1 (stored) stream.
__device__ __forceinline__ void copy_stored(uint8_t* out, const uint8_t* in, uint32_t n, int tid, int nthreads) {
  for (uint32_t i = tid; i < n; i += nthreads) out[16 + i] = in[i];
}

}  // namespace detail
}  // namespace ans
}  // namespace device
}  // namespace nvcomp
