// nvcomp/device/detail/ptx.cuh -- the inline-PTX primitives of the LZ4 / Snappy coder (sm_90a): explicit
// shared-space loads / stores on 32-bit shared-window addresses, streaming global vector accesses, mbarrier and TMA
// bulk-copy wrappers.  The library's batched kernels (nvcomp_b200/csrc/ptx.cuh re-exports these names) and the
// device API (nvcomp/device/lz4.cuh, snappy.cuh) use this one copy.  The LZ headers contain no other asm and include
// this file by its angle-bracket path, so tests/emu can re-run their warp-level logic on the host by shadowing it
// (test infrastructure only; the product is CUDA).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

// 32-bit shared-window address of a pointer into shared memory
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------------------
// Global-memory access helpers.
// ---------------------------------------------------------------------------
// Read-only, streaming (compressed input is read once): bypass L1 allocation.
__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// Streaming store: decompressed output is written once, never re-read by this
// kernel beyond the match window, so do not let it thrash L1.
__device__ __forceinline__ void st_v4(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 ld_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}

// explicit shared-space accesses on 32-bit addresses (the generic-pointer form costs 64-bit address
// arithmetic and generic LD/ST on every byte)
template <int O = 0>
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(v) : "r"(a), "n"(O) : "memory");
  return v;
}
template <int O = 0>
__device__ __forceinline__ void sts_u8(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u8 [%0+%1], %2;" :: "r"(a), "n"(O), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a) : "memory");
  return r;
}
__device__ __forceinline__ void sts_v4(uint32_t a, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u16(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "r"(v) : "memory");
}
template <int O>
__device__ __forceinline__ uint32_t ldg_u8(const uint8_t* p) {
  uint32_t v;
  asm volatile("ld.global.u8 %0, [%1+%2];" : "=r"(v) : "l"(p), "n"(O) : "memory");
  return v;
}
// touch one word of a cache line: the line travels to L1 while the warp goes on (the value is never used, so no
// instruction waits for it)
__device__ __forceinline__ void touch_line(const void* p) {
  asm volatile("{\n\t.reg .u32 t;\n\tld.global.ca.u32 t, [%0];\n\t}" :: "l"(p) : "memory");
}
template <int O>
__device__ __forceinline__ uint32_t ldg_u32(const uint8_t* p) {
  uint32_t v;
  asm volatile("ld.global.u32 %0, [%1+%2];" : "=r"(v) : "l"(p), "n"(O) : "memory");
  return v;
}

// ---------------------------------------------------------------------------
// TMA 1-D bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier helpers: one thread stages a
// 16-byte aligned span of global memory into shared memory asynchronously; consumers wait on
// the mbarrier's phase.  Addresses are 32-bit shared-window addresses.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(mbar), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" :: "r"(mbar), "r"(parity) : "memory");
}
// Invalidate the mbarrier (no thread may wait on it and no copy may complete on it any more): its 8 bytes become
// ordinary shared memory again.  The device API does this before every return, so the caller may reuse its region.
__device__ __forceinline__ void mbar_inval(uint32_t mbar) {
  asm volatile("mbarrier.inval.shared::cta.b64 [%0];" :: "r"(mbar) : "memory");
}
// order this thread's earlier generic-proxy accesses to shared memory before later async-proxy writes
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// smem_dst, gmem_src and bytes must be multiples of 16
__device__ __forceinline__ void tma_bulk_g2s(uint32_t smem_dst, const void* gmem_src, uint32_t bytes, uint32_t mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_dst), "l"(gmem_src), "r"(bytes), "r"(mbar) : "memory");
}

// schedule tracing (lz_sched.cuh, B200_LZ_TRACE builds only): device-wide nanosecond clock and the SM of this thread
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t sm_id() {
  uint32_t s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
