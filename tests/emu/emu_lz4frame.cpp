// emu_lz4frame.cpp -- TEST INFRASTRUCTURE: runs the warp-level LZ4 frame decoder (lz4frame_decode.cuh, with the LZ4
// block bodies and their bulk-copy staging) inside the host warp emulator.  Built into tests/emu/libemu_lz.so by the
// Makefile; loaded by tests/test_lz4frame_emu.py and tests/test_lz4frame_gpu.py.
#include "emu_cuda.h"

#include <sys/mman.h>
#include <unistd.h>

#include "lz_decode.cuh"
#include "nvcomp/device/detail/lz4frame_decode.cuh"

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

}  // namespace

extern "C" {
// count_only: the size query (walk without writing).  reps: decode the chunk reps times in one warp with one region
// and one mbarrier phase, as the batched kernel's chunk loop runs its chunks.  Returns bytes produced, -1 if the
// decoder rejected the chunk, -3 for a checksum mismatch, -2 on an emulator fault (msg says why).  Unless count_only,
// a successful decode must leave the output bytes beyond `produced` untouched.
long emu_lz4frame(int count_only, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, unsigned in_mis,
                  unsigned out_mis, int reps, char* msg, size_t msg_bytes) {
  using namespace nvcomp::device::lz4frame::detail;
  Guarded gin(n, in_mis & 15u), gout(count_only ? 0 : cap, out_mis & 15u);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  if (!count_only) emu::add_region(w, gout.p, cap, true);
  uint32_t produced = 0;
  int result = kLz4fBad;
  emu::run_warp(w, b200::kLzWarpSmem, [&](int lane) {
    uint8_t* ring = emu::g_warp->smem;
    b200::lz_warp_init(b200::smem_addr(ring), lane);
    uint32_t parity = 0;
    for (int r = 0; r < reps; ++r) {
      uint32_t prod = 0;
      int res = kLz4fBad;
      if (n <= 0xffffffffull && cap <= 0xffffffffull)
        res = count_only ? lz4f_chunk<true>(gin.p, (uint32_t)n, nullptr, 0xffffffffu, &prod, ring, parity, lane)
                         : lz4f_chunk<false>(gin.p, (uint32_t)n, gout.p, (uint32_t)cap, &prod, ring, parity, lane);
      if (lane == 0) { result = res; produced = prod; }
    }
  });
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  if (result == kLz4fBad) return -1;
  if (result == kLz4fBadChecksum) return -3;
  if (count_only) return (long)produced;
  if (produced > cap) { if (msg) snprintf(msg, msg_bytes, "produced %u > cap %zu", produced, cap); return -2; }
  for (size_t i = produced; i < cap; ++i)
    if (gout.p[i] != 0xee) {
      if (msg) snprintf(msg, msg_bytes, "byte %zu written beyond produced %u", i, produced);
      return -2;
    }
  memcpy(dst, gout.p, produced);
  return (long)produced;
}
}
