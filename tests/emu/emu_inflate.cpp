// emu_inflate.cpp -- TEST INFRASTRUCTURE: runs the warp-level Deflate / Gzip chunk decoder of nvcomp_b200/csrc
// (inflate_decode.cuh) inside the host warp emulator.  Built into tests/emu/libemu_lz.so by the Makefile; loaded only
// by tests/test_inflate_emu.py.
#include "emu_cuda.h"

#include <sys/mman.h>
#include <unistd.h>

#include "inflate_decode.cuh"

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

struct CrcTables {
  uint32_t table[256], x2n[32];
  CrcTables() {
    for (uint32_t i = 0; i < 256; ++i) table[i] = b200::crc_table_entry(i);
    for (int k = 0; k < 32; ++k) x2n[k] = b200::crc_x2n_entry(k);
  }
};

}  // namespace

extern "C" {
// gzip: 0 = raw Deflate, 1 = Gzip member.  count_only: walk the stream without writing (the size query).
// reps: decode the chunk reps times in one warp (the fixed-code tables are built once and then reused).
// Returns bytes produced, -1 if the decoder rejected the stream, -3 for a Gzip checksum (CRC-32 / ISIZE) mismatch,
// -2 on an emulator fault (msg says why).  Unless count_only, the output bytes beyond `produced` must be untouched.
int emu_inflate(int gzip, int count_only, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, unsigned in_mis,
                unsigned out_mis, int reps, char* msg, size_t msg_bytes) {
  static const CrcTables crc;
  Guarded gin(n, in_mis & 15u), gout(count_only ? 0 : cap, out_mis & 15u);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  if (!count_only) emu::add_region(w, gout.p, cap, true);
  uint32_t produced = 0;
  int result = 0;
  emu::run_warp(w, b200::kInfWarpSmem, [&](int lane) {
    b200::InflateWarp ws{b200::smem_addr(emu::g_warp->smem), false};
    for (int r = 0; r < reps; ++r) {
      uint32_t prod = 0;
      int res;
      if (count_only)
        res = gzip ? b200::inflate_chunk<true, true>(gin.p, (uint32_t)n, nullptr, 0xffffffffu, &prod, ws, crc.table,
                                                      crc.x2n, lane)
                   : b200::inflate_chunk<false, true>(gin.p, (uint32_t)n, nullptr, 0xffffffffu, &prod, ws, crc.table,
                                                       crc.x2n, lane);
      else
        res = gzip ? b200::inflate_chunk<true, false>(gin.p, (uint32_t)n, gout.p, (uint32_t)cap, &prod, ws, crc.table,
                                                       crc.x2n, lane)
                   : b200::inflate_chunk<false, false>(gin.p, (uint32_t)n, gout.p, (uint32_t)cap, &prod, ws,
                                                        crc.table, crc.x2n, lane);
      if (lane == 0) { result = res; produced = prod; }
    }
  });
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  if (result == b200::kInflateBad) return -1;
  if (result == b200::kInflateBadChecksum) return -3;
  if (count_only) return (int)produced;
  if (produced > cap) { if (msg) snprintf(msg, msg_bytes, "produced %u > cap %zu", produced, cap); return -2; }
  for (size_t i = produced; i < cap; ++i)
    if (gout.p[i] != 0xee) {
      if (msg) snprintf(msg, msg_bytes, "byte %zu written beyond produced %u", i, produced);
      return -2;
    }
  memcpy(dst, gout.p, produced);
  return (int)produced;
}
}
