// zstd_compress_device_kernels.cu -- test and benchmark kernels over zstd::compress_warp (nvcomp/device/zstd.cuh),
// built into build/tests/libzstd_compress_device.so and driven from Python (tests/test_zstd_compress_device_gpu.py,
// tools/zstd_compress_device_bench.py).  Every launcher takes device arrays in the batched C API's layout (pointers,
// sizes) and enqueues on `stream`; it returns the launch's cudaError_t.
//
// Every warp owns a region of dynamic shared memory: kCompressSmemBytes for the compress kernel, kRegion (the largest
// of the roles) for the mixed and region-reuse kernels.  A compressing warp takes chunks gw, gw + total_warps, ... or,
// when `ticket` is not null, pulls them from that global counter (zeroed by the caller).
#include <cuda_runtime.h>

#include "nvcomp/device/deflate.cuh"
#include "nvcomp/device/zstd.cuh"

namespace dfd = nvcomp::device::deflate;
namespace zsd = nvcomp::device::zstd;

// One role of the mixed-CTA kernel (extern "C": zc_dev_mixed takes an array of them).
struct Role {
  const void* const* src;
  const size_t* src_bytes;
  void* const* dst;
  size_t* dst_bytes;   // compressed sizes (compress) or capacities (decode)
  size_t* actual;
  int* status;
  size_t n;
};

namespace {

constexpr int kWarps = 4;
constexpr unsigned kMaxCtas = 132 * 16;
constexpr unsigned kFull = 0xffffffffu;

constexpr size_t cmax(size_t a, size_t b) { return a > b ? a : b; }
constexpr size_t kRegion = cmax(zsd::kCompressSmemBytes, cmax(zsd::kDecompressSmemBytes, dfd::kDecompressSmemBytes));
static_assert(kRegion == zsd::kCompressSmemBytes, "the compress region is the largest role");
static_assert(kRegion % zsd::kSmemAlignment == 0, "aligned regions");

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }
__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

__device__ __forceinline__ uint8_t* warp_smem(int w) {
  extern __shared__ __align__(16) unsigned char smem[];
  return smem + (size_t)w * kRegion;
}

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

__device__ __forceinline__ nvcompStatus_t zstd_compress(const void* in, size_t n, void* out, size_t* comp_bytes,
                                                        int algo, void* sm) {
  nvcompBatchedZstdOpts_t o;
  o.algo = algo;
  return zsd::compress_warp(in, n, out, comp_bytes, o, sm);
}

__global__ void __launch_bounds__(kWarps * 32)
compress_kernel(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                size_t batch, int algo, unsigned long long* ticket) {
  void* sm = warp_smem(threadIdx.x >> 5);
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    const nvcompStatus_t st = zstd_compress(in[c], in_bytes[c], out[c], comp_bytes ? comp_bytes + c : nullptr, algo,
                                            sm);
    if (status && lane() == 0) status[c] = (int)st;
  }
}

// Four warps per CTA with four roles: warps 0 and 2 compress Zstd (chunk sets A and D), warp 1 decodes Zstd chunks
// (B), warp 3 decodes Deflate chunks (C).  CTA b takes chunk b, b + gridDim.x, ... of each set.
__global__ void __launch_bounds__(kWarps * 32) mixed_kernel(Role a, Role b, Role c, Role d) {
  const int w = threadIdx.x >> 5;
  void* sm = warp_smem(w);
  const Role r = w == 0 ? a : w == 1 ? b : w == 2 ? d : c;
  for (size_t i = blockIdx.x; i < r.n; i += gridDim.x) {
    nvcompStatus_t st;
    if (w == 0 || w == 2) st = zstd_compress(r.src[i], r.src_bytes[i], r.dst[i], r.dst_bytes + i, 0, sm);
    else if (w == 1) st = zsd::decompress_warp(r.src[i], r.src_bytes[i], r.dst[i], r.dst_bytes[i], r.actual + i, sm);
    else st = dfd::decompress_warp(r.src[i], r.src_bytes[i], r.dst[i], r.dst_bytes[i], r.actual + i, sm);
    if (lane() == 0) r.status[i] = (int)st;
  }
}

// One region per warp, not cleared between calls: compress chunk i into comp[i], then decode comp[i] into dec[i]
// in the same region, then the next chunk.
__global__ void __launch_bounds__(kWarps * 32)
reuse_kernel(const void* const* in, const size_t* in_bytes, void* const* comp, size_t* comp_bytes, void* const* dec,
             const size_t* dec_caps, size_t* dec_actual, int* cstatus, int* dstatus, size_t batch) {
  void* sm = warp_smem(threadIdx.x >> 5);
  for (size_t i = global_warp(); i < batch; i += total_warps()) {
    const nvcompStatus_t cs = zstd_compress(in[i], in_bytes[i], comp[i], comp_bytes + i, 0, sm);
    size_t cb = 0;
    if (lane() == 0) cb = comp_bytes[i];
    cb = __shfl_sync(kFull, cb, 0);
    const nvcompStatus_t ds = zsd::decompress_warp(comp[i], cb, dec[i], dec_caps[i], dec_actual + i, sm);
    if (lane() == 0) { cstatus[i] = (int)cs; dstatus[i] = (int)ds; }
  }
}

template <class K>
unsigned ctas_for(K kernel, size_t batch, bool ticketed) {
  const size_t need = (batch + kWarps - 1) / kWarps;
  if (ticketed) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kWarps * 32, kWarps * kRegion);
    const size_t g = (size_t)(sms > 0 ? sms : 1) * (size_t)(per_sm > 0 ? per_sm : 1);
    return (unsigned)(need < g ? (need ? need : 1) : g);
  }
  return (unsigned)(need < kMaxCtas ? (need ? need : 1) : kMaxCtas);
}

template <class K>
cudaError_t prepare(K kernel) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWarps * kRegion));
}

}  // namespace

extern "C" {

// [kCompressSmemBytes, kMaxCompressChunkBytes, kSmemAlignment, kDecompressSmemBytes]
void zc_dev_constants(size_t* out) {
  out[0] = zsd::kCompressSmemBytes;
  out[1] = zsd::kMaxCompressChunkBytes;
  out[2] = zsd::kSmemAlignment;
  out[3] = zsd::kDecompressSmemBytes;
}
size_t zc_dev_max_compressed_bytes(size_t n) { return zsd::max_compressed_bytes(n); }

int zc_dev_compress(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                    size_t batch, int algo, unsigned long long* ticket, cudaStream_t stream) {
  cudaError_t e = prepare(compress_kernel);
  if (e != cudaSuccess) return (int)e;
  const unsigned ctas = ctas_for(compress_kernel, batch, ticket != nullptr);
  compress_kernel<<<ctas, kWarps * 32, kWarps * kRegion, stream>>>(in, in_bytes, out, comp_bytes, status, batch, algo,
                                                                   ticket);
  return (int)cudaGetLastError();
}

int zc_dev_mixed(const Role* roles, unsigned ctas, cudaStream_t stream) {
  cudaError_t e = prepare(mixed_kernel);
  if (e != cudaSuccess) return (int)e;
  mixed_kernel<<<ctas, kWarps * 32, kWarps * kRegion, stream>>>(roles[0], roles[1], roles[2], roles[3]);
  return (int)cudaGetLastError();
}

int zc_dev_reuse(const void* const* in, const size_t* in_bytes, void* const* comp, size_t* comp_bytes,
                 void* const* dec, const size_t* dec_caps, size_t* dec_actual, int* cstatus, int* dstatus,
                 size_t batch, cudaStream_t stream) {
  cudaError_t e = prepare(reuse_kernel);
  if (e != cudaSuccess) return (int)e;
  reuse_kernel<<<ctas_for(reuse_kernel, batch, false), kWarps * 32, kWarps * kRegion, stream>>>(
      in, in_bytes, comp, comp_bytes, dec, dec_caps, dec_actual, cstatus, dstatus, batch);
  return (int)cudaGetLastError();
}

}  // extern "C"
