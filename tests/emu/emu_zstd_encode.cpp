// emu_zstd_encode.cpp -- TEST INFRASTRUCTURE: runs the warp-level Zstandard chunk encoder
// (include/nvcomp/device/detail/zstd_encode.cuh) inside the host warp emulator.  Built into tests/emu/libemu_lz.so by
// the Makefile; loaded by tests/test_zstd_encode_emu.py and, as the reference bytes for the GPU, by
// tests/test_zstd_compress_device_gpu.py.
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

#include "nvcomp/device/detail/zstd_encode.cuh"

namespace {

namespace zd = nvcomp::device::zstd::detail;

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

}  // namespace

extern "C" {
size_t emu_zstd_enc_bound(size_t n) { return zd::zstd_enc_bound((uint32_t)n); }
size_t emu_zstd_enc_smem(void) { return zd::kZstdEncWarpSmem; }

// Compress n <= 64 KB bytes (input at misalignment in_mis, output at out_mis) into dst, which has room for the
// bound.  Returns the frame length, or -2 on an emulator fault or a write past the frame (msg says why).
long emu_zstd_compress(const uint8_t* src, size_t n, unsigned in_mis, unsigned out_mis, uint8_t* dst, char* msg,
                       size_t msg_bytes) {
  const size_t cap = zd::zstd_enc_bound((uint32_t)n);
  Guarded gin(n, in_mis & 15u), gout(cap, out_mis & 15u);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  emu::add_region(w, gout.p, cap, true);
  uint32_t produced = 0;
  emu::run_warp(w, zd::kZstdEncWarpSmem, [&](int lane) {
    const uint32_t r = zd::zstd_compress_chunk(gin.p, (uint32_t)n, gout.p, emu::g_warp->smem, lane);
    if (lane == 0) produced = r;
  });
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  if (produced > cap) { if (msg) snprintf(msg, msg_bytes, "produced %u > cap %zu", produced, cap); return -2; }
  for (size_t i = produced; i < cap; ++i)
    if (gout.p[i] != 0xee) {
      if (msg) snprintf(msg, msg_bytes, "byte %zu written beyond the frame's %u", i, produced);
      return -2;
    }
  memcpy(dst, gout.p, produced);
  return (long)produced;
}
}
