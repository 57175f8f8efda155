// emu_lz.cpp -- TEST INFRASTRUCTURE: runs the warp-level LZ4 / Snappy chunk decoders of
// nvcomp_b200/csrc (lz_decode.cuh, lz4_decode.cuh, snappy_decode.cuh) inside the host warp emulator.
// Built into tests/emu/libemu_lz.so by the Makefile; loaded by tests/test_lz_emu.py,
// tests/test_lz_writer.py and tests/test_lz_oracle_gpu.py.
#include <memory>   // (before emu_cuda.h: its __noinline__ macro clashes with libstdc++ attributes)
#include <vector>

#include "emu_cuda.h"

#include <sys/mman.h>
#include <unistd.h>

#include "lz4_decode.cuh"
#include "snappy_decode.cuh"

// lz_sched.cuh also holds the classification kernel; only its host-callable rules (lz_bucket) are used here, the
// kernel is compiled but never run
#define __launch_bounds__(...)
static const struct { unsigned x; } blockIdx{0}, blockDim{32};
static inline unsigned __match_any_sync(unsigned, int) { emu::fail("__match_any_sync is not emulated"); }
#include "lz_sched.cuh"

namespace {

// A buffer that ends (rounded up to its 16-byte granule) exactly at an inaccessible page, with an
// inaccessible page in front: out-of-bounds plain loads / stores fault instead of passing silently.
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

bool decode_one(int codec, int mode, const uint8_t* in, uint32_t n, uint8_t* out, size_t cap, uint32_t* prod,
                uint8_t* ring, uint32_t& tma_parity, int lane) {
  if (codec == 0)
    return mode == 1 ? b200::lz4_decode_chunk_direct(in, n, out, cap, prod, lane)
                     : b200::lz4_decode_chunk_v2(in, n, out, cap, prod, ring, tma_parity, lane, mode != 2);
  return mode == 1 ? b200::snappy_decode_chunk(in, n, out, cap, prod, lane)
                   : b200::snappy_decode_chunk_v2(in, n, out, cap, prod, ring, tma_parity, lane, mode != 2);
}

int run(int codec, int mode, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, unsigned in_mis,
        unsigned out_mis, char* msg, size_t msg_bytes, unsigned long long* n_sync) {
  Guarded gin(n, in_mis & 15u), gout(cap, out_mis & 15u);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  emu::add_region(w, gout.p, cap, true);
  uint32_t produced = 0;
  bool ok = false;
  emu::run_warp(w, b200::kLzWarpSmem, [&](int lane) {
    uint8_t* ring = emu::g_warp->smem;
    b200::lz_warp_init(b200::smem_addr(ring), lane);
    uint32_t tma_parity = 0;
    uint32_t prod = 0;
    const bool r = decode_one(codec, mode, gin.p, (uint32_t)n, gout.p, cap, &prod, ring, tma_parity, lane);
    if (lane == 0) { ok = r; produced = prod; }
  });
  if (n_sync) *n_sync = w.n_sync;
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  if (!ok) return -1;
  if (produced > cap) { if (msg) snprintf(msg, msg_bytes, "produced %u > cap %zu", produced, cap); return -2; }
  memcpy(dst, gout.p, produced);
  return (int)produced;
}

}  // namespace

extern "C" {
// codec: 0 = LZ4, 1 = Snappy.  mode: 0 = adaptive (as the kernel), 1 = direct loop, 2 = block decoder forced.
// Returns bytes produced, -1 if the decoder rejected the stream, -2 on an emulator fault (msg says why).
int emu_lz_decode(int codec, int mode, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, unsigned in_mis,
                  unsigned out_mis, char* msg, size_t msg_bytes, unsigned long long* n_sync) {
  return run(codec, mode, src, n, dst, cap, in_mis, out_mis, msg, msg_bytes, n_sync);
}

// A sequence of chunks decoded by one warp the way the decode kernels' chunk loop runs them: one ring, one mbarrier
// (initialised once) and one tma_parity carried from chunk to chunk.  Chunk k is src[in_off[k], in_off[k] + n[k]),
// decoded into its own guarded buffer of caps[k] bytes (misaligned by in_mis / out_mis) and copied to
// dst + out_off[k].  produced[k] = bytes produced or -1 (rejected).  Returns 0, or -2 on an emulator fault.
int emu_lz_decode_seq(int codec, int mode, int n_chunks, const uint8_t* src, const size_t* in_off, const size_t* n,
                      uint8_t* dst, const size_t* out_off, const size_t* caps, unsigned in_mis, unsigned out_mis,
                      long long* produced, char* msg, size_t msg_bytes) {
  std::vector<std::unique_ptr<Guarded>> gin, gout;
  for (int k = 0; k < n_chunks; ++k) {
    gin.emplace_back(new Guarded(n[k], in_mis & 15u));
    gout.emplace_back(new Guarded(caps[k], out_mis & 15u));
    if (n[k]) memcpy(gin[k]->p, src + in_off[k], n[k]);
  }
  emu::Warp w;
  std::vector<long long> res(n_chunks, -1);
  emu::run_warp(w, b200::kLzWarpSmem, [&](int lane) {
    uint8_t* ring = emu::g_warp->smem;
    b200::lz_warp_init(b200::smem_addr(ring), lane);
    uint32_t tma_parity = 0;
    for (int k = 0; k < n_chunks; ++k) {
      __syncwarp();
      if (lane == 0) {            // only chunk k's buffers are accessible while it decodes
        emu::g_warp->n_regions = 0;
        emu::add_region(*emu::g_warp, gin[k]->p, n[k], false);
        emu::add_region(*emu::g_warp, gout[k]->p, caps[k], true);
      }
      __syncwarp();
      uint32_t prod = 0;
      const bool r = decode_one(codec, mode, gin[k]->p, (uint32_t)n[k], gout[k]->p, caps[k], &prod, ring, tma_parity,
                                lane);
      if (lane == 0) res[k] = r ? (long long)prod : -1;
    }
  });
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  for (int k = 0; k < n_chunks; ++k) {
    produced[k] = res[k];
    if (res[k] > (long long)caps[k]) {
      if (msg) snprintf(msg, msg_bytes, "chunk %d: produced %lld > cap %zu", k, res[k], caps[k]);
      return -2;
    }
    if (res[k] > 0) memcpy(dst + out_off[k], gout[k]->p, (size_t)res[k]);
  }
  return 0;
}

// Does the dense decoder reject the stream while a staged-block copy is in flight?  Runs lz_decode_loop -- what
// lz_decode_stream runs before its drain -- on a fresh warp and looks at the prefetch state it leaves (then drains it).
// Returns 1: rejected with a copy in flight, 0: rejected with none, 2: accepted, -2: emulator fault.
int emu_lz_fails_in_flight(int codec, const uint8_t* src, size_t n, size_t cap, char* msg, size_t msg_bytes) {
  Guarded gin(n, 0), gout(cap, 0);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  emu::add_region(w, gout.p, cap, true);
  int res = 0;
  emu::run_warp(w, b200::kLzWarpSmem, [&](int lane) {
    uint8_t* ring = emu::g_warp->smem;
    b200::lz_warp_init(b200::smem_addr(ring), lane);
    b200::LzState s;
    s.in = gin.p; s.in_n = (uint32_t)n; s.out = gout.p; s.out_cap = cap;
    s.ip = 0; s.op = 0; s.flushed = 0; s.ring_lo = 0;
    s.align = (uint32_t)((uintptr_t)gout.p & 15u);
    s.ring = b200::smem_addr(ring);
    s.cur = 0; s.pf_ip = b200::kNoPrefetch; s.parity = 0; s.next = b200::kNextUnknown;
    bool ok;
    if (codec == 0) {
      ok = b200::lz_decode_loop<b200::Lz4Decode>(s, lane);
    } else {
      uint64_t ulen = 0;
      if (!b200::snappy_read_preamble(gin.p, (uint32_t)n, s.ip, ulen) || ulen > cap) {
        if (lane == 0) res = 0;
        return;
      }
      s.out_cap = ulen;
      ok = b200::lz_decode_loop<b200::SnappyDecode>(s, lane);
    }
    const bool in_flight = s.pf_ip != b200::kNoPrefetch;
    if (in_flight) b200::lz_stage_wait(s);
    if (lane == 0) res = ok ? 2 : in_flight ? 1 : 0;
  });
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  return res;
}

// lz_bucket of lz_sched.cuh: the cost bucket (0-1 light kernel, 2-5 dense kernel) of a chunk of n compressed bytes
// decoded at capacity cap.
int emu_lz_bucket(unsigned long long cap, unsigned long long n) { return b200::lz_bucket(cap, n); }

// The LZ4 size query (lz4_walk_chunk, what nvcompBatchedLZ4GetDecompressSizeAsync runs per chunk): returns the
// decompressed size, -1 for a malformed block, -2 on an emulator fault.
long long emu_lz4_walk(const uint8_t* src, size_t n, unsigned in_mis, char* msg, size_t msg_bytes) {
  Guarded gin(n, in_mis & 15u);
  if (n) memcpy(gin.p, src, n);
  emu::Warp w;
  emu::add_region(w, gin.p, n, false);
  long long res = -1;
  emu::run_warp(w, 0, [&](int lane) {
    uint32_t prod = 0;
    const bool ok = b200::lz4_walk_chunk(gin.p, (uint32_t)n, &prod, lane);
    if (lane == 0) res = ok ? (long long)prod : -1;
  });
  if (w.failed) {
    if (msg) snprintf(msg, msg_bytes, "%s", w.fail_msg);
    return -2;
  }
  return res;
}
}
