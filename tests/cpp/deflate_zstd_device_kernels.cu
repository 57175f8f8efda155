// deflate_zstd_device_kernels.cu -- test and benchmark kernels over the warp-level Deflate, Gzip and Zstd device APIs
// (nvcomp/device/deflate.cuh, gzip.cuh, zstd.cuh), built into build/tests/libdeflate_zstd_device.so and driven from
// Python (tests/test_deflate_device_gpu.py, tests/test_zstd_device_gpu.py, tools/deflate_zstd_device_bench.py).  Every
// launcher takes device arrays in the batched C API's layout (pointers, sizes), a codec where it matters (0 = Deflate,
// 1 = Gzip, 2 = Zstd), and enqueues on `stream`; it returns the launch's cudaError_t.
//
// The kernels run kWarps warps per CTA, each with its own region of dynamic shared memory of the size its header asks
// for (kDecodeRegion<CODEC>, compress_smem_bytes(algo)); Deflate compression with algo 1 runs kWarps1 warps.  The
// mixed-CTA kernel gives every warp kRegion bytes, the largest of the mixed roles.  A warp takes
// chunks gw, gw + total_warps, ... or, when `ticket` is not null, pulls them from that global counter (zeroed by the
// caller).
//
// This file also includes every other device header, so all eight device APIs are shown to build in one translation
// unit without name clashes.
#include <cuda_runtime.h>

#include "nvcomp/device/ans.cuh"
#include "nvcomp/device/bitcomp.cuh"
#include "nvcomp/device/cascaded.cuh"
#include "nvcomp/device/deflate.cuh"
#include "nvcomp/device/gzip.cuh"
#include "nvcomp/device/lz4.cuh"
#include "nvcomp/device/snappy.cuh"
#include "nvcomp/device/zstd.cuh"

namespace dfd = nvcomp::device::deflate;
namespace gzd = nvcomp::device::gzip;
namespace zsd = nvcomp::device::zstd;

namespace {

constexpr int kWarps = 4;
constexpr int kWarps1 = 3;
constexpr unsigned kMaxCtas = 132 * 16;
constexpr unsigned kFull = 0xffffffffu;

constexpr size_t cmax(size_t a, size_t b) { return a > b ? a : b; }
// one region size for every role but algo-1 compression, so a CTA may mix them
constexpr size_t kRegion = cmax(cmax(dfd::kDecompressSmemBytes, gzd::kDecompressSmemBytes),
                                cmax(zsd::kDecompressSmemBytes,
                                     cmax(dfd::compress_smem_bytes(0), dfd::compress_smem_bytes(2))));
constexpr size_t kRegion1 = dfd::compress_smem_bytes(1);
// algos 0 and 2, and the algos compress_warp rejects
constexpr size_t kRegion02 = dfd::compress_smem_bytes(0);
static_assert(dfd::compress_smem_bytes(2) == kRegion02, "one region for algos 0 and 2");
template <int CODEC>
constexpr size_t kDecodeRegion = CODEC == 0 ? dfd::kDecompressSmemBytes
                                 : CODEC == 1 ? gzd::kDecompressSmemBytes : zsd::kDecompressSmemBytes;
static_assert(kRegion == 16896, "the Zstd region is the largest of the mixed roles");
static_assert(kRegion % dfd::kSmemAlignment == 0 && kRegion1 % dfd::kSmemAlignment == 0, "aligned regions");

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }
__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

template <size_t kBytes = kRegion>
__device__ __forceinline__ uint8_t* warp_smem(int w) {
  extern __shared__ __align__(16) unsigned char smem[];
  return smem + (size_t)w * kBytes;
}

// chunk source of one warp: a static stride, or a global ticket
struct Chunks {
  unsigned long long* ticket;
  size_t next_static;
  __device__ __forceinline__ explicit Chunks(unsigned long long* t) : ticket(t), next_static(global_warp()) {}
  __device__ __forceinline__ size_t next() {
    if (!ticket) { const size_t c = next_static; next_static += total_warps(); return c; }
    unsigned long long t = 0;
    if (lane() == 0) t = atomicAdd(ticket, 1ull);
    return (size_t)__shfl_sync(kFull, t, 0);
  }
};

template <int CODEC>
__device__ __forceinline__ nvcompStatus_t decompress_one(const void* comp, size_t comp_bytes, void* out, size_t cap,
                                                         size_t* actual, void* sm) {
  if (CODEC == 0) return dfd::decompress_warp(comp, comp_bytes, out, cap, actual, sm);
  if (CODEC == 1) return gzd::decompress_warp(comp, comp_bytes, out, cap, actual, sm);
  return zsd::decompress_warp(comp, comp_bytes, out, cap, actual, sm);
}

template <int CODEC>
__device__ __forceinline__ size_t size_one(const void* comp, size_t comp_bytes, void* sm) {
  if (CODEC == 0) return dfd::decompressed_size_warp(comp, comp_bytes, sm);
  if (CODEC == 1) return gzd::decompressed_size_warp(comp, comp_bytes, sm);
  return zsd::decompressed_size_warp(comp, comp_bytes, sm);
}

__device__ __forceinline__ nvcompStatus_t compress_one(const void* in, size_t n, void* out, size_t* comp_bytes,
                                                       int algo, void* sm) {
  nvcompBatchedDeflateOpts_t o;
  o.algo = algo;
  return dfd::compress_warp(in, n, out, comp_bytes, o, sm);
}

// kWarpsPerCta warps with kBytes of shared memory each
template <int kWarpsPerCta, size_t kBytes>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
compress_kernel(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                size_t batch, int algo, unsigned long long* ticket) {
  void* sm = warp_smem<kBytes>(threadIdx.x >> 5);
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    const nvcompStatus_t st = compress_one(in[c], in_bytes[c], out[c], comp_bytes + c, algo, sm);
    if (status && lane() == 0) status[c] = (int)st;
  }
}

template <int CODEC>
__global__ void __launch_bounds__(kWarps * 32)
decompress_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, size_t batch, unsigned long long* ticket) {
  void* sm = warp_smem<kDecodeRegion<CODEC>>(threadIdx.x >> 5);
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    const nvcompStatus_t st = decompress_one<CODEC>(comp[c], comp_bytes[c], out[c], caps[c], actual ? actual + c : nullptr, sm);
    if (status && lane() == 0) status[c] = (int)st;
  }
}

template <int CODEC>
__global__ void __launch_bounds__(kWarps * 32)
size_kernel(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch) {
  void* sm = warp_smem<kDecodeRegion<CODEC>>(threadIdx.x >> 5);
  for (size_t c = global_warp(); c < batch; c += total_warps()) {
    const size_t s = size_one<CODEC>(comp[c], comp_bytes[c], sm);
    if (lane() == 0) sizes[c] = s;
  }
}

// The wrapping u64 sum of the 32-bit little-endian words of n bytes at p (16-byte aligned; a ragged end counts as a
// zero-padded word), by one warp.
__device__ __forceinline__ unsigned long long warp_sum_words(const uint8_t* p, size_t n) {
  const uint4* v = (const uint4*)p;
  const size_t nv = n / 16;
  unsigned long long sum = 0;
#pragma unroll 4
  for (size_t i = lane(); i < nv; i += 32) {
    const uint4 q = v[i];
    sum += (unsigned long long)q.x + q.y + q.z + q.w;
  }
  const size_t t = 16 * nv + 4 * (size_t)lane();
  if (t < n) {
    uint32_t w = 0;
    for (size_t k = 0; k < 4 && t + k < n; ++k) w |= (uint32_t)p[t + k] << (8 * k);
    sum += w;
  }
  for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
  return sum;
}

// decompress_warp, then the same warp sums the chunk it just wrote
template <int CODEC>
__global__ void __launch_bounds__(kWarps * 32)
decompress_sum_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                      unsigned long long* sums, int* status, size_t batch, unsigned long long* ticket) {
  void* sm = warp_smem<kDecodeRegion<CODEC>>(threadIdx.x >> 5);
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    size_t actual = 0;
    const nvcompStatus_t st = decompress_one<CODEC>(comp[c], comp_bytes[c], out[c], caps[c], &actual, sm);
    actual = __shfl_sync(kFull, actual, 0);
    const unsigned long long s = warp_sum_words((const uint8_t*)out[c], actual);
    if (lane() == 0) { sums[c] = s; status[c] = (int)st; }
  }
}

// the unfused path's second kernel: one warp per decoded chunk of sizes[c] bytes
__global__ void __launch_bounds__(kWarps * 32)
sum_kernel(const void* const* data, const size_t* sizes, unsigned long long* sums, size_t batch,
           unsigned long long* ticket) {
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    const unsigned long long s = warp_sum_words((const uint8_t*)data[c], sizes[c]);
    if (lane() == 0) sums[c] = s;
  }
}

// Region reuse.  One CTA of three warps whose regions are packed at the codec's declared kDecompressSmemBytes, so
// warp 1's region has warp 0's right before it and warp 2's right after: a call that touches shared memory outside the
// size its header declares changes a canary.  Warp 1 decodes the chunks in order with one region; after each call it
// overwrites that whole region with 0xA5, reads it back and counts the bytes that differ (mismatch[c]).  Warps 0 and 2
// fill their regions with a canary first and count the canary bytes that changed once warp 1 is done
// (canary_bad[0], [1]).
template <int CODEC>
__global__ void __launch_bounds__(3 * 32)
reuse_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps, size_t* actual,
             int* status, unsigned* mismatch, unsigned* canary_bad, size_t batch) {
  const int w = threadIdx.x >> 5;
  uint8_t* sm = warp_smem<kDecodeRegion<CODEC>>(w);
  if (w != 1) {
    for (size_t i = lane(); i < kDecodeRegion<CODEC>; i += 32) sm[i] = (uint8_t)(0xC3u ^ (i * 7u) ^ (w << 4));
  }
  __syncthreads();
  if (w == 1) {
    for (size_t c = 0; c < batch; ++c) {
      const nvcompStatus_t st = decompress_one<CODEC>(comp[c], comp_bytes[c], out[c], caps[c], actual + c, sm);
      if (lane() == 0) status[c] = (int)st;
      for (size_t i = lane(); i < kDecodeRegion<CODEC>; i += 32) sm[i] = 0xA5;
      __syncwarp();
      unsigned bad = 0;
      for (size_t i = lane(); i < kDecodeRegion<CODEC>; i += 32) bad += sm[i] != 0xA5;
      for (int d = 16; d; d >>= 1) bad += __shfl_xor_sync(kFull, bad, d);
      if (lane() == 0) mismatch[c] = bad;
      __syncwarp();
    }
  }
  __syncthreads();
  if (w != 1) {
    unsigned bad = 0;
    for (size_t i = lane(); i < kDecodeRegion<CODEC>; i += 32) bad += sm[i] != (uint8_t)(0xC3u ^ (i * 7u) ^ (w << 4));
    for (int d = 16; d; d >>= 1) bad += __shfl_xor_sync(kFull, bad, d);
    if (lane() == 0) canary_bad[w / 2] = bad;
  }
}

// Four warps per CTA, one per role: Deflate compress (algo 0 or 2), Deflate decompress, Gzip decompress, Zstd
// decompress, all with kRegion-byte regions.  Each role's warps stride over that role's batch.
struct Role {
  const void* const* src; const size_t* src_bytes; void* const* dst; size_t* dst_bytes; const size_t* caps;
  int* status; size_t batch;
};
__global__ void __launch_bounds__(4 * 32)
mixed_kernel(Role r0, Role r1, Role r2, Role r3, int algo) {
  const int w = threadIdx.x >> 5;
  void* sm = warp_smem(w);
  const Role r = w == 0 ? r0 : w == 1 ? r1 : w == 2 ? r2 : r3;
  for (size_t c = blockIdx.x; c < r.batch; c += gridDim.x) {
    nvcompStatus_t st;
    if (w == 0) st = compress_one(r.src[c], r.src_bytes[c], r.dst[c], r.dst_bytes + c, algo, sm);
    else if (w == 1) st = decompress_one<0>(r.src[c], r.src_bytes[c], r.dst[c], r.caps[c], r.dst_bytes + c, sm);
    else if (w == 2) st = decompress_one<1>(r.src[c], r.src_bytes[c], r.dst[c], r.caps[c], r.dst_bytes + c, sm);
    else st = decompress_one<2>(r.src[c], r.src_bytes[c], r.dst[c], r.caps[c], r.dst_bytes + c, sm);
    if (lane() == 0) r.status[c] = (int)st;
  }
}

template <class K>
cudaError_t prepare(K kernel, size_t smem) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

// CTAs for a batch: one warp per chunk up to kMaxCtas CTAs; with a ticket, as many CTAs as are resident at once
template <class K>
unsigned ctas_for(K kernel, size_t batch, bool ticketed, int warps, size_t smem) {
  const size_t need = (batch + warps - 1) / warps;
  if (ticketed) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, warps * 32, smem);
    const size_t g = (size_t)(sms > 0 ? sms : 1) * (size_t)(per_sm > 0 ? per_sm : 1);
    return (unsigned)(need < g ? (need ? need : 1) : g);
  }
  return (unsigned)(need < kMaxCtas ? (need ? need : 1) : kMaxCtas);
}

template <int kWarpsPerCta = kWarps, size_t kBytes = kRegion, class K, class... A>
int launch(K kernel, size_t batch, unsigned long long* ticket, cudaStream_t stream, A... args) {
  const size_t smem = kWarpsPerCta * kBytes;
  cudaError_t e = prepare(kernel, smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<ctas_for(kernel, batch, ticket != nullptr, kWarpsPerCta, smem), kWarpsPerCta * 32, smem, stream>>>(args...);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

// [deflate kDecompressSmemBytes, compress_smem_bytes(0), (1), (2), (3), (-1), kMaxCompressChunkBytes, kSmemAlignment,
//  gzip kDecompressSmemBytes, kSmemAlignment, zstd kDecompressSmemBytes, kSmemAlignment]
void dz_dev_constants(size_t* out) {
  out[0] = dfd::kDecompressSmemBytes;
  out[1] = dfd::compress_smem_bytes(0); out[2] = dfd::compress_smem_bytes(1);
  out[3] = dfd::compress_smem_bytes(2); out[4] = dfd::compress_smem_bytes(3);
  out[5] = dfd::compress_smem_bytes(-1);
  out[6] = dfd::kMaxCompressChunkBytes; out[7] = dfd::kSmemAlignment;
  out[8] = gzd::kDecompressSmemBytes; out[9] = gzd::kSmemAlignment;
  out[10] = zsd::kDecompressSmemBytes; out[11] = zsd::kSmemAlignment;
}
size_t dz_dev_region_bytes() { return kRegion; }
size_t dz_dev_max_compressed_bytes(size_t n) { return dfd::max_compressed_bytes(n); }

int dz_dev_compress(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                    size_t batch, int algo, unsigned long long* ticket, cudaStream_t stream) {
  if (algo == 1)
    return launch<kWarps1, kRegion1>(compress_kernel<kWarps1, kRegion1>, batch, ticket, stream, in, in_bytes, out,
                                     comp_bytes, status, batch, algo, ticket);
  return launch<kWarps, kRegion02>(compress_kernel<kWarps, kRegion02>, batch, ticket, stream, in, in_bytes, out,
                                   comp_bytes, status, batch, algo, ticket);
}

int dz_dev_decompress(int codec, const void* const* comp, const size_t* comp_bytes, void* const* out,
                      const size_t* caps, size_t* actual, int* status, size_t batch, unsigned long long* ticket,
                      cudaStream_t stream) {
  if (codec == 0)
    return launch<kWarps, kDecodeRegion<0>>(decompress_kernel<0>, batch, ticket, stream, comp, comp_bytes, out, caps, actual, status, batch, ticket);
  if (codec == 1)
    return launch<kWarps, kDecodeRegion<1>>(decompress_kernel<1>, batch, ticket, stream, comp, comp_bytes, out, caps, actual, status, batch, ticket);
  return launch<kWarps, kDecodeRegion<2>>(decompress_kernel<2>, batch, ticket, stream, comp, comp_bytes, out, caps, actual, status, batch, ticket);
}

int dz_dev_decompress_sum(int codec, const void* const* comp, const size_t* comp_bytes, void* const* out,
                          const size_t* caps, unsigned long long* sums, int* status, size_t batch,
                          unsigned long long* ticket, cudaStream_t stream) {
  if (codec == 0)
    return launch<kWarps, kDecodeRegion<0>>(decompress_sum_kernel<0>, batch, ticket, stream, comp, comp_bytes, out, caps, sums, status, batch, ticket);
  if (codec == 1)
    return launch<kWarps, kDecodeRegion<1>>(decompress_sum_kernel<1>, batch, ticket, stream, comp, comp_bytes, out, caps, sums, status, batch, ticket);
  return launch<kWarps, kDecodeRegion<2>>(decompress_sum_kernel<2>, batch, ticket, stream, comp, comp_bytes, out, caps, sums, status, batch, ticket);
}

int dz_dev_sum(const void* const* data, const size_t* sizes, unsigned long long* sums, size_t batch,
               unsigned long long* ticket, cudaStream_t stream) {
  const unsigned ctas = ctas_for(sum_kernel, batch, ticket != nullptr, kWarps, 0);
  sum_kernel<<<ctas, kWarps * 32, 0, stream>>>(data, sizes, sums, batch, ticket);
  return (int)cudaGetLastError();
}

int dz_dev_decompressed_size(int codec, const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch,
                             cudaStream_t stream) {
  if (batch == 0) return 0;
  if (codec == 0) return launch<kWarps, kDecodeRegion<0>>(size_kernel<0>, batch, nullptr, stream, comp, comp_bytes, sizes, batch);
  if (codec == 1) return launch<kWarps, kDecodeRegion<1>>(size_kernel<1>, batch, nullptr, stream, comp, comp_bytes, sizes, batch);
  return launch<kWarps, kDecodeRegion<2>>(size_kernel<2>, batch, nullptr, stream, comp, comp_bytes, sizes, batch);
}

int dz_dev_reuse(int codec, const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                 size_t* actual, int* status, unsigned* mismatch, unsigned* canary_bad, size_t batch,
                 cudaStream_t stream) {
  cudaError_t e;
  if (codec == 0) {
    const size_t smem = 3 * kDecodeRegion<0>;
    if ((e = prepare(reuse_kernel<0>, smem)) != cudaSuccess) return (int)e;
    reuse_kernel<0><<<1, 3 * 32, smem, stream>>>(comp, comp_bytes, out, caps, actual, status, mismatch, canary_bad, batch);
  } else if (codec == 1) {
    const size_t smem = 3 * kDecodeRegion<1>;
    if ((e = prepare(reuse_kernel<1>, smem)) != cudaSuccess) return (int)e;
    reuse_kernel<1><<<1, 3 * 32, smem, stream>>>(comp, comp_bytes, out, caps, actual, status, mismatch, canary_bad, batch);
  } else {
    const size_t smem = 3 * kDecodeRegion<2>;
    if ((e = prepare(reuse_kernel<2>, smem)) != cudaSuccess) return (int)e;
    reuse_kernel<2><<<1, 3 * 32, smem, stream>>>(comp, comp_bytes, out, caps, actual, status, mismatch, canary_bad, batch);
  }
  return (int)cudaGetLastError();
}

// roles: 0 Deflate compress (algo), 1 Deflate decompress, 2 Gzip decompress, 3 Zstd decompress.  For the compress role
// dst_bytes receives the compressed sizes, for decompress roles the actual sizes (caps are the capacities).
int dz_dev_mixed(const void* const* src0, const size_t* sb0, void* const* dst0, size_t* db0, int* st0, size_t n0,
                 const void* const* src1, const size_t* sb1, void* const* dst1, const size_t* caps1, size_t* db1,
                 int* st1, size_t n1, const void* const* src2, const size_t* sb2, void* const* dst2,
                 const size_t* caps2, size_t* db2, int* st2, size_t n2, const void* const* src3, const size_t* sb3,
                 void* const* dst3, const size_t* caps3, size_t* db3, int* st3, size_t n3, int algo,
                 cudaStream_t stream) {
  const Role r0{src0, sb0, dst0, db0, nullptr, st0, n0}, r1{src1, sb1, dst1, db1, caps1, st1, n1};
  const Role r2{src2, sb2, dst2, db2, caps2, st2, n2}, r3{src3, sb3, dst3, db3, caps3, st3, n3};
  size_t most = n0 > n1 ? n0 : n1;
  most = most > n2 ? most : n2;
  most = most > n3 ? most : n3;
  const size_t smem = 4 * kRegion;
  cudaError_t e = prepare(mixed_kernel, smem);
  if (e != cudaSuccess) return (int)e;
  const unsigned ctas = (unsigned)(most < kMaxCtas ? (most ? most : 1) : kMaxCtas);
  mixed_kernel<<<ctas, 4 * 32, smem, stream>>>(r0, r1, r2, r3, algo);
  return (int)cudaGetLastError();
}

}  // extern "C"
