// lz_device_kernels.cu -- test and benchmark kernels over the warp-level LZ4 and Snappy device APIs
// (nvcomp/device/lz4.cuh, nvcomp/device/snappy.cuh), built into build/tests/liblz_device.so and driven from Python
// (tests/test_lz_device_gpu.py, tools/lz_device_bench.py).  Every launcher takes device arrays in the batched C API's
// layout (pointers, sizes), a codec (0 = LZ4, 1 = Snappy), and enqueues on `stream`; it returns the launch's
// cudaError_t.
//
// The kernels run kWarps warps per CTA, each with its own region of dynamic shared memory.  A warp takes chunks
// gw, gw + total_warps, ... or, when `ticket` is not null, pulls them from that global counter (zeroed by the caller).
#include <cuda_runtime.h>

#include "nvcomp/device/lz4.cuh"
#include "nvcomp/device/snappy.cuh"

namespace lz4d = nvcomp::device::lz4;
namespace snd = nvcomp::device::snappy;

namespace {

constexpr int kWarps = 4;
constexpr unsigned kMaxCtas = 132 * 16;
constexpr unsigned kFull = 0xffffffffu;
// one region size for every role, so a CTA may mix them
constexpr size_t kRegion = lz4d::kCompressSmemBytes > lz4d::kDecompressSmemBytes ? lz4d::kCompressSmemBytes
                                                                                 : lz4d::kDecompressSmemBytes;
static_assert(lz4d::kDecompressSmemBytes == snd::kDecompressSmemBytes, "one decode region for both codecs");
static_assert(lz4d::kCompressSmemBytes == snd::kCompressSmemBytes, "one hash table for both codecs");
static_assert(kRegion % lz4d::kSmemAlignment == 0, "aligned regions");

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }
__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

__device__ __forceinline__ uint8_t* warp_smem(int w) {
  extern __shared__ __align__(16) unsigned char smem[];
  return smem + (size_t)w * kRegion;
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
__device__ __forceinline__ nvcompStatus_t compress_one(const void* in, size_t n, void* out, size_t* comp_bytes,
                                                       int data_type, void* sm) {
  if (CODEC == 0) {
    nvcompBatchedLZ4Opts_t o;
    o.data_type = (nvcompType_t)data_type;
    return lz4d::compress_warp(in, n, out, comp_bytes, o, sm);
  }
  return snd::compress_warp(in, n, out, comp_bytes, sm);
}

template <int CODEC>
__device__ __forceinline__ nvcompStatus_t decompress_one(const void* comp, size_t comp_bytes, void* out, size_t cap,
                                                         size_t* actual, void* sm) {
  if (CODEC == 0) return lz4d::decompress_warp(comp, comp_bytes, out, cap, actual, sm);
  return snd::decompress_warp(comp, comp_bytes, out, cap, actual, sm);
}

template <int CODEC>
__global__ void __launch_bounds__(kWarps * 32)
compress_kernel(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                size_t batch, int data_type, unsigned long long* ticket) {
  void* sm = warp_smem(threadIdx.x >> 5);
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    const nvcompStatus_t st = compress_one<CODEC>(in[c], in_bytes[c], out[c], comp_bytes + c, data_type, sm);
    if (status && lane() == 0) status[c] = (int)st;
  }
}

template <int CODEC>
__global__ void __launch_bounds__(kWarps * 32)
decompress_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, size_t batch, unsigned long long* ticket) {
  void* sm = warp_smem(threadIdx.x >> 5);
  Chunks q(ticket);
  for (size_t c = q.next(); c < batch; c = q.next()) {
    const nvcompStatus_t st = decompress_one<CODEC>(comp[c], comp_bytes[c], out[c], caps[c], actual ? actual + c : nullptr, sm);
    if (status && lane() == 0) status[c] = (int)st;
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
  void* sm = warp_smem(threadIdx.x >> 5);
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

template <int CODEC>
__global__ void __launch_bounds__(kWarps * 32)
size_kernel(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch) {
  if (CODEC == 0) {
    for (size_t c = global_warp(); c < batch; c += total_warps()) {
      const size_t s = lz4d::decompressed_size_warp(comp[c], comp_bytes[c]);
      if (lane() == 0) sizes[c] = s;
    }
  } else {
    const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per chunk
    if (c < batch) sizes[c] = snd::decompressed_size(comp[c], comp_bytes[c]);
  }
}

// Region hygiene.  One CTA of three warps: warp 1 decodes the chunks in order with one region; after each call it
// overwrites that whole region with a pattern derived from the chunk index, reads it back and counts the bytes that
// differ (mismatch[c]).  Warps 0 and 2 fill their regions with a canary first and count the canary bytes that changed
// once warp 1 is done (canary_bad[0], [1]).
template <int CODEC>
__global__ void __launch_bounds__(3 * 32)
hygiene_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
               size_t* actual, int* status, unsigned* mismatch, unsigned* canary_bad, size_t batch) {
  const int w = threadIdx.x >> 5;
  uint8_t* sm = warp_smem(w);
  if (w != 1) {
    for (size_t i = lane(); i < kRegion; i += 32) sm[i] = (uint8_t)(0xC3u ^ (i * 7u) ^ (w << 4));
  }
  __syncthreads();
  if (w == 1) {
    for (size_t c = 0; c < batch; ++c) {
      const nvcompStatus_t st = decompress_one<CODEC>(comp[c], comp_bytes[c], out[c], caps[c], actual + c, sm);
      if (lane() == 0) status[c] = (int)st;
      const uint8_t pat = (uint8_t)(0x5Au + 13u * (unsigned)c);
      for (size_t i = lane(); i < kRegion; i += 32) sm[i] = (uint8_t)(pat ^ i);
      __syncwarp();
      unsigned bad = 0;
      for (size_t i = lane(); i < kRegion; i += 32) bad += sm[i] != (uint8_t)(pat ^ i);
      for (int d = 16; d; d >>= 1) bad += __shfl_xor_sync(kFull, bad, d);
      if (lane() == 0) mismatch[c] = bad;
      __syncwarp();
    }
  }
  __syncthreads();
  if (w != 1) {
    unsigned bad = 0;
    for (size_t i = lane(); i < kRegion; i += 32) bad += sm[i] != (uint8_t)(0xC3u ^ (i * 7u) ^ (w << 4));
    for (int d = 16; d; d >>= 1) bad += __shfl_xor_sync(kFull, bad, d);
    if (lane() == 0) canary_bad[w / 2] = bad;
  }
}

// Four warps per CTA, one per role: LZ4 compress, Snappy compress, LZ4 decompress, Snappy decompress.  Each role's
// warps stride over that role's batch.
struct Role {
  const void* const* src; const size_t* src_bytes; void* const* dst; size_t* dst_bytes; const size_t* caps;
  int* status; size_t batch;
};
__global__ void __launch_bounds__(4 * 32)
mixed_kernel(Role r0, Role r1, Role r2, Role r3, int data_type) {
  const int w = threadIdx.x >> 5;
  void* sm = warp_smem(w);
  const Role r = w == 0 ? r0 : w == 1 ? r1 : w == 2 ? r2 : r3;
  for (size_t c = blockIdx.x; c < r.batch; c += gridDim.x) {
    nvcompStatus_t st;
    if (w == 0) st = compress_one<0>(r.src[c], r.src_bytes[c], r.dst[c], r.dst_bytes + c, data_type, sm);
    else if (w == 1) st = compress_one<1>(r.src[c], r.src_bytes[c], r.dst[c], r.dst_bytes + c, 0, sm);
    else if (w == 2) st = decompress_one<0>(r.src[c], r.src_bytes[c], r.dst[c], r.caps[c], r.dst_bytes + c, sm);
    else st = decompress_one<1>(r.src[c], r.src_bytes[c], r.dst[c], r.caps[c], r.dst_bytes + c, sm);
    if (lane() == 0) r.status[c] = (int)st;
  }
}

template <class K>
cudaError_t prepare(K kernel, size_t smem) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

// CTAs for a batch: one warp per chunk up to kMaxCtas CTAs; with a ticket, as many CTAs as are resident at once
template <class K>
unsigned ctas_for(K kernel, size_t batch, bool ticketed, size_t smem) {
  if (ticketed) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kWarps * 32, smem);
    const size_t g = (size_t)(sms > 0 ? sms : 1) * (size_t)(per_sm > 0 ? per_sm : 1);
    const size_t need = (batch + kWarps - 1) / kWarps;
    return (unsigned)(need < g ? (need ? need : 1) : g);
  }
  const size_t need = (batch + kWarps - 1) / kWarps;
  return (unsigned)(need < kMaxCtas ? (need ? need : 1) : kMaxCtas);
}

template <class K, class... A>
int launch(K kernel, size_t batch, unsigned long long* ticket, cudaStream_t stream, A... args) {
  const size_t smem = kWarps * kRegion;
  cudaError_t e = prepare(kernel, smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<ctas_for(kernel, batch, ticket != nullptr, smem), kWarps * 32, smem, stream>>>(args...);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

// [kMaxChunkBytes, kSmemAlignment, kDecompressSmemBytes, kCompressSmemBytes] of the codec
void lz_dev_constants(int codec, size_t* out) {
  if (codec == 0) {
    out[0] = lz4d::kMaxChunkBytes; out[1] = lz4d::kSmemAlignment;
    out[2] = lz4d::kDecompressSmemBytes; out[3] = lz4d::kCompressSmemBytes;
  } else {
    out[0] = snd::kMaxChunkBytes; out[1] = snd::kSmemAlignment;
    out[2] = snd::kDecompressSmemBytes; out[3] = snd::kCompressSmemBytes;
  }
}
size_t lz_dev_region_bytes() { return kRegion; }
size_t lz_dev_max_compressed_bytes(int codec, size_t n) {
  return codec == 0 ? lz4d::max_compressed_bytes(n) : snd::max_compressed_bytes(n);
}

int lz_dev_compress(int codec, const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes,
                    int* status, size_t batch, int data_type, unsigned long long* ticket, cudaStream_t stream) {
  if (codec == 0)
    return launch(compress_kernel<0>, batch, ticket, stream, in, in_bytes, out, comp_bytes, status, batch, data_type, ticket);
  return launch(compress_kernel<1>, batch, ticket, stream, in, in_bytes, out, comp_bytes, status, batch, data_type, ticket);
}

int lz_dev_decompress(int codec, const void* const* comp, const size_t* comp_bytes, void* const* out,
                      const size_t* caps, size_t* actual, int* status, size_t batch, unsigned long long* ticket,
                      cudaStream_t stream) {
  if (codec == 0)
    return launch(decompress_kernel<0>, batch, ticket, stream, comp, comp_bytes, out, caps, actual, status, batch, ticket);
  return launch(decompress_kernel<1>, batch, ticket, stream, comp, comp_bytes, out, caps, actual, status, batch, ticket);
}

int lz_dev_decompress_sum(int codec, const void* const* comp, const size_t* comp_bytes, void* const* out,
                          const size_t* caps, unsigned long long* sums, int* status, size_t batch,
                          unsigned long long* ticket, cudaStream_t stream) {
  if (codec == 0)
    return launch(decompress_sum_kernel<0>, batch, ticket, stream, comp, comp_bytes, out, caps, sums, status, batch, ticket);
  return launch(decompress_sum_kernel<1>, batch, ticket, stream, comp, comp_bytes, out, caps, sums, status, batch, ticket);
}

int lz_dev_sum(const void* const* data, const size_t* sizes, unsigned long long* sums, size_t batch,
               unsigned long long* ticket, cudaStream_t stream) {
  const unsigned ctas = ctas_for(sum_kernel, batch, ticket != nullptr, 0);
  sum_kernel<<<ctas, kWarps * 32, 0, stream>>>(data, sizes, sums, batch, ticket);
  return (int)cudaGetLastError();
}

int lz_dev_decompressed_size(int codec, const void* const* comp, const size_t* comp_bytes, size_t* sizes,
                             size_t batch, cudaStream_t stream) {
  if (batch == 0) return 0;
  if (codec == 0) {
    const size_t ctas = (batch + kWarps - 1) / kWarps;
    size_kernel<0><<<(unsigned)(ctas < kMaxCtas ? ctas : kMaxCtas), kWarps * 32, 0, stream>>>(comp, comp_bytes, sizes, batch);
  } else {
    size_kernel<1><<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp, comp_bytes, sizes, batch);
  }
  return (int)cudaGetLastError();
}

int lz_dev_hygiene(int codec, const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                   size_t* actual, int* status, unsigned* mismatch, unsigned* canary_bad, size_t batch,
                   cudaStream_t stream) {
  const size_t smem = 3 * kRegion;
  if (codec == 0) {
    cudaError_t e = prepare(hygiene_kernel<0>, smem);
    if (e != cudaSuccess) return (int)e;
    hygiene_kernel<0><<<1, 3 * 32, smem, stream>>>(comp, comp_bytes, out, caps, actual, status, mismatch, canary_bad, batch);
  } else {
    cudaError_t e = prepare(hygiene_kernel<1>, smem);
    if (e != cudaSuccess) return (int)e;
    hygiene_kernel<1><<<1, 3 * 32, smem, stream>>>(comp, comp_bytes, out, caps, actual, status, mismatch, canary_bad, batch);
  }
  return (int)cudaGetLastError();
}

// roles: 0 LZ4 compress (data_type), 1 Snappy compress, 2 LZ4 decompress, 3 Snappy decompress.  For compress roles
// dst_bytes receives the compressed sizes, for decompress roles the actual sizes (caps are the capacities).
int lz_dev_mixed(const void* const* src0, const size_t* sb0, void* const* dst0, size_t* db0, int* st0, size_t n0,
                 const void* const* src1, const size_t* sb1, void* const* dst1, size_t* db1, int* st1, size_t n1,
                 const void* const* src2, const size_t* sb2, void* const* dst2, const size_t* caps2, size_t* db2,
                 int* st2, size_t n2, const void* const* src3, const size_t* sb3, void* const* dst3,
                 const size_t* caps3, size_t* db3, int* st3, size_t n3, int data_type, cudaStream_t stream) {
  const Role r0{src0, sb0, dst0, db0, nullptr, st0, n0}, r1{src1, sb1, dst1, db1, nullptr, st1, n1};
  const Role r2{src2, sb2, dst2, db2, caps2, st2, n2}, r3{src3, sb3, dst3, db3, caps3, st3, n3};
  size_t most = n0 > n1 ? n0 : n1;
  most = most > n2 ? most : n2;
  most = most > n3 ? most : n3;
  const size_t smem = 4 * kRegion;
  cudaError_t e = prepare(mixed_kernel, smem);
  if (e != cudaSuccess) return (int)e;
  const unsigned ctas = (unsigned)(most < kMaxCtas ? (most ? most : 1) : kMaxCtas);
  mixed_kernel<<<ctas, 4 * 32, smem, stream>>>(r0, r1, r2, r3, data_type);
  return (int)cudaGetLastError();
}

}  // extern "C"
