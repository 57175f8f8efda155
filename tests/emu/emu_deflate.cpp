// emu_deflate.cpp -- TEST INFRASTRUCTURE: runs the warp-level Deflate chunk encoder of nvcomp_b200/csrc
// (deflate_compress.cuh) inside the host warp emulator.  Built into tests/emu/libemu_lz.so by the Makefile; loaded by
// tests/test_deflate_encode_emu.py and, as the reference bytes for the GPU, by tests/test_deflate_compress_gpu.py.
#include "emu_cuda.h"

#include <sys/mman.h>
#include <unistd.h>

// Warp intrinsics the encoder uses beyond those of emu_cuda.h.  They must be declared before the encoder header.
static inline unsigned __match_any_sync(unsigned, unsigned v) {
  emu::Warp* w = emu::g_warp;
  w->xchg[emu::lane()] = v;
  emu::rendezvous(12, nullptr);
  unsigned m = 0;
  for (int i = 0; i < 32; ++i) m |= ((unsigned)w->xchg[i] == v ? 1u : 0u) << i;
  emu::rendezvous(1012, nullptr);
  return m;
}
// lanes run one at a time between warp intrinsics, so a plain read-modify-write is atomic
static inline unsigned atomicAdd(unsigned* p, unsigned v) {
  const unsigned old = *p;
  *p = old + v;
  return old;
}
static inline unsigned atomicOr(unsigned* p, unsigned v) {
  const unsigned old = *p;
  *p = old | v;
  return old;
}

#include "deflate_compress.cuh"

namespace {

// A buffer that ends (rounded up to its 16-byte granule) exactly at an inaccessible page, with an inaccessible page
// in front: out-of-bounds plain loads / stores fault instead of passing silently.
struct Guarded {
  uint8_t* map = nullptr;
  size_t map_bytes = 0;
  uint8_t* p = nullptr;
  Guarded(size_t n, unsigned misalign) {
    const size_t page = (size_t)sysconf(_SC_PAGESIZE);
    const size_t body = ((n + misalign + 15) / 16 * 16 + page - 1) / page * page + page;
    map_bytes = body + 2 * page;
    map = (uint8_t*)mmap(nullptr, map_bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (map == MAP_FAILED) abort();
    mprotect(map, page, PROT_NONE);
    mprotect(map + page + body, page, PROT_NONE);
    uint8_t* end = map + page + body;
    p = end - (n + misalign + 15) / 16 * 16 + misalign;
    memset(map + page, 0xee, body);
  }
  ~Guarded() { munmap(map, map_bytes); }
};

template <int kAlgo>
void run(emu::Warp& w, const uint8_t* in, uint32_t n, uint8_t* out, uint32_t* produced) {
  emu::run_warp(w, b200::kDeflateWarpSmem<kAlgo>, [&](int lane) {
    const b200::DeflateWarp ws = b200::DeflateWarp::carve<kAlgo>(emu::g_warp->smem);
    const uint32_t r = b200::deflate_compress_chunk<kAlgo>(in, n, out, ws, lane);
    if (lane == 0) *produced = r;
  });
}

// Records the parse: (literal run, distance, length) per sequence, (trailing literals, 0, 0) at the end.
struct TokenRec {
  uint32_t* t;
  uint32_t cap, n;
  void put(uint32_t a, uint32_t b, uint32_t c, int lane) {
    if (lane == 0 && n + 3 <= cap) { t[n] = a; t[n + 1] = b; t[n + 2] = c; }
    n += 3;
  }
  void sequence(const uint8_t*, uint32_t ll, uint32_t off, uint32_t ml, int lane) { put(ll, off, ml, lane); }
  void finish(const uint8_t*, uint32_t ll, int lane) { put(ll, 0, 0, lane); }
};

template <int kAlgo>
void parse(emu::Warp& w, const uint8_t* in, uint32_t n, uint32_t* t, uint32_t cap, uint32_t* words) {
  emu::run_warp(w, b200::kDeflateWarpSmem<kAlgo>, [&](int lane) {
    TokenRec rec{t, cap, 0};
    b200::deflate_parse<kAlgo>(in, n, rec, (uint16_t*)emu::g_warp->smem, lane);
    if (lane == 0) *words = rec.n;
  });
}

}  // namespace

extern "C" {
// The encoder's parse of n bytes with algo 0..2, as (literal run, distance, length) triples into t (cap words; a
// trailing (literals, 0, 0)).  Returns the number of words, or -2 on an emulator fault.
int emu_deflate_parse(int algo, const uint8_t* src, size_t n, uint32_t* t, size_t cap, char* msg, size_t msg_bytes) {
  Guarded gin(n, 0);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  uint32_t words = 0;
  if (algo == 0) parse<0>(w, gin.p, (uint32_t)n, t, (uint32_t)cap, &words);
  else if (algo == 1) parse<1>(w, gin.p, (uint32_t)n, t, (uint32_t)cap, &words);
  else parse<2>(w, gin.p, (uint32_t)n, t, (uint32_t)cap, &words);
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  return (int)words;
}

// Compress n bytes (input at misalignment in_mis) with algo 0..2 into dst, which has room for cap bytes (the maximum
// output size).  Returns the stream length, or -2 on an emulator fault or a write past the stream (msg says why).
int emu_deflate(int algo, const uint8_t* src, size_t n, unsigned in_mis, uint8_t* dst, size_t cap, char* msg,
                size_t msg_bytes) {
  Guarded gin(n, in_mis & 15u), gout(cap, 0);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  emu::add_region(w, gout.p, cap, true);
  uint32_t produced = 0;
  if (algo == 0) run<0>(w, gin.p, (uint32_t)n, gout.p, &produced);
  else if (algo == 1) run<1>(w, gin.p, (uint32_t)n, gout.p, &produced);
  else run<2>(w, gin.p, (uint32_t)n, gout.p, &produced);
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  if (produced > cap) { if (msg) snprintf(msg, msg_bytes, "produced %u > cap %zu", produced, cap); return -2; }
  for (size_t i = produced; i < cap; ++i)
    if (gout.p[i] != 0xee) {
      if (msg) snprintf(msg, msg_bytes, "byte %zu written beyond the stream's %u", i, produced);
      return -2;
    }
  memcpy(dst, gout.p, produced);
  return (int)produced;
}
}
