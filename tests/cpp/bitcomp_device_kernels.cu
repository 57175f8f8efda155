// bitcomp_device_kernels.cu -- test and benchmark kernels over the warp-level Bitcomp device API
// (nvcomp/device/bitcomp.cuh), built into build/tests/libbitcomp_device.so and driven from Python
// (tests/test_bitcomp_device_gpu.py, tools/bitcomp_device_bench.py).  Every launcher takes device arrays in the batched
// C API's layout (pointers, sizes) and enqueues on `stream`; it returns the launch's cudaError_t.
//
// The kernels are persistent: kWarps warps per CTA, each warp takes chunks gw, gw + total_warps, ...
#include <cuda_runtime.h>

#include <type_traits>

#include "nvcomp/device/bitcomp.cuh"

namespace dev = nvcomp::device::bitcomp;

namespace {

constexpr int kWarps = 4;
constexpr unsigned kMaxCtas = 132 * 16;
constexpr unsigned kFull = 0xffffffffu;

unsigned ctas_for(size_t batch) {
  const size_t need = (batch + kWarps - 1) / kWarps;
  return (unsigned)(need < kMaxCtas ? (need ? need : 1) : kMaxCtas);
}

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }
__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

__device__ __forceinline__ void* warp_smem() {
  __shared__ __align__(dev::kSmemAlignment) unsigned char smem[kWarps * dev::kCompressSmemBytes];
  return smem + (threadIdx.x >> 5) * dev::kCompressSmemBytes;
}

__device__ __forceinline__ void compress_one(const void* const* in, const size_t* in_bytes, void* const* out,
                                             size_t* comp_bytes, int* status, nvcompBatchedBitcompFormatOpts opts,
                                             size_t c) {
  const nvcompStatus_t st = dev::compress_warp(in[c], in_bytes[c], out[c], comp_bytes + c, opts, warp_smem());
  if (lane() == 0) status[c] = (int)st;
}

__device__ __forceinline__ void decompress_one(const void* const* comp, const size_t* comp_bytes, void* const* out,
                                               const size_t* caps, size_t* actual, int* status, size_t c) {
  const nvcompStatus_t st = dev::decompress_warp(comp[c], comp_bytes[c], out[c], caps[c], actual + c);
  if (lane() == 0) status[c] = (int)st;
}

__device__ __forceinline__ uint64_t mix64(uint64_t x) {   // splitmix64 finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

template <class T> __device__ __forceinline__ uint64_t widen(T v) {
  // signed types sign-extend, unsigned ones zero-extend
  return (uint64_t)(typename std::conditional<std::is_signed<T>::value, int64_t, uint64_t>::type)v;
}

// Visit one chunk with for_each_block<T>: the wrapping u64 sum of its elements; an order-sensitive hash
// h = (h ^ D_b) * FNV_prime over the blocks b in visit order, where D_b is the wrapping sum over the block's valid
// elements i of mix64(widen(v_i) ^ (i * golden)); and the number of visits.
template <class T>
__device__ __forceinline__ void visit_one(const void* const* comp, const size_t* comp_bytes, unsigned long long* sums,
                                          unsigned long long* hashes, unsigned long long* visits, int* status,
                                          size_t c) {
  uint64_t sum = 0, hash = 0, nvis = 0;
  const nvcompStatus_t st = dev::for_each_block<T>(comp[c], comp_bytes[c],
      [&](const T (&v)[4], uint32_t first, uint32_t valid) {
        uint64_t dsum = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
          if (k < valid) {
            const uint64_t x = widen(v[k]);
            sum += x;
            dsum += mix64(x ^ ((uint64_t)(first + k) * 0x9e3779b97f4a7c15ull));
          }
        }
        for (int d = 16; d; d >>= 1) dsum += __shfl_xor_sync(kFull, dsum, d);
        hash = (hash ^ dsum) * 0x100000001b3ull;
        ++nvis;
      });
  for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
  if (lane() == 0) { sums[c] = sum; hashes[c] = hash; visits[c] = nvis; status[c] = (int)st; }
}

__global__ void __launch_bounds__(kWarps * 32)
compress_kernel(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                size_t batch, nvcompBatchedBitcompFormatOpts opts) {
  for (size_t c = global_warp(); c < batch; c += total_warps()) compress_one(in, in_bytes, out, comp_bytes, status, opts, c);
}

__global__ void __launch_bounds__(kWarps * 32)
decompress_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, size_t batch) {
  for (size_t c = global_warp(); c < batch; c += total_warps()) decompress_one(comp, comp_bytes, out, caps, actual, status, c);
}

template <class T>
__global__ void __launch_bounds__(kWarps * 32)
visit_kernel(const void* const* comp, const size_t* comp_bytes, unsigned long long* sums, unsigned long long* hashes,
             unsigned long long* visits, int* status, size_t batch) {
  for (size_t c = global_warp(); c < batch; c += total_warps()) visit_one<T>(comp, comp_bytes, sums, hashes, visits, status, c);
}

// Warps 3k compress chunks of one batch, warps 3k + 1 decompress chunks of another and warps 3k + 2 visit a third
// (as int64), side by side in the same CTAs.
__global__ void __launch_bounds__(kWarps * 32)
mixed_kernel(const void* const* in, const size_t* in_bytes, void* const* cout, size_t* cbytes, int* cstatus,
             size_t cbatch, nvcompBatchedBitcompFormatOpts opts, const void* const* comp, const size_t* comp_bytes,
             void* const* dout, const size_t* caps, size_t* actual, int* dstatus, size_t dbatch,
             const void* const* vcomp, const size_t* vcomp_bytes, unsigned long long* sums,
             unsigned long long* hashes, unsigned long long* visits, int* vstatus, size_t vbatch) {
  const size_t role = global_warp() % 3, gw = global_warp() / 3, stride = total_warps() / 3;
  if (gw >= stride) return;                       // the last warps of an uneven split sit out
  if (role == 0) {
    for (size_t c = gw; c < cbatch; c += stride) compress_one(in, in_bytes, cout, cbytes, cstatus, opts, c);
  } else if (role == 1) {
    for (size_t c = gw; c < dbatch; c += stride) decompress_one(comp, comp_bytes, dout, caps, actual, dstatus, c);
  } else {
    for (size_t c = gw; c < vbatch; c += stride) visit_one<int64_t>(vcomp, vcomp_bytes, sums, hashes, visits, vstatus, c);
  }
}

// The fused path of the benchmark: the wrapping int64 sum of every chunk, decoded in registers.
__global__ void __launch_bounds__(kWarps * 32)
fused_sum_kernel(const void* const* comp, const size_t* comp_bytes, long long* sums, int* status, size_t batch) {
  for (size_t c = global_warp(); c < batch; c += total_warps()) {
    uint64_t sum = 0;
    const nvcompStatus_t st = dev::for_each_block<int64_t>(comp[c], comp_bytes[c],
        [&](const int64_t (&v)[4], uint32_t, uint32_t valid) {
#pragma unroll
          for (uint32_t k = 0; k < 4; ++k) sum += k < valid ? (uint64_t)v[k] : 0ull;
        });
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
    if (lane() == 0) { sums[c] = (long long)sum; status[c] = (int)st; }
  }
}

// The unfused path's second kernel: the wrapping int64 sum of every decoded chunk of sizes[c] bytes (a multiple of 8,
// 16-byte aligned), 16-byte loads.
__global__ void __launch_bounds__(kWarps * 32)
sum_i64_kernel(const void* const* data, const size_t* sizes, long long* sums, size_t batch) {
  for (size_t c = global_warp(); c < batch; c += total_warps()) {
    const longlong2* p = (const longlong2*)data[c];
    const size_t nv = sizes[c] / 16;
    uint64_t sum = 0;
#pragma unroll 4
    for (size_t i = lane(); i < nv; i += 32) {
      const longlong2 q = __ldcs(p + i);
      sum += (uint64_t)q.x + (uint64_t)q.y;
    }
    if ((sizes[c] & 15) && lane() == 0) sum += (uint64_t)((const long long*)data[c])[2 * nv];
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
    if (lane() == 0) sums[c] = (long long)sum;
  }
}

__global__ void size_kernel(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < batch) sizes[c] = dev::decompressed_size(comp[c], comp_bytes[c]);
}

nvcompBatchedBitcompFormatOpts opts_of(int algo, int type) {
  nvcompBatchedBitcompFormatOpts o;
  o.algorithm_type = algo;
  o.data_type = (nvcompType_t)type;
  return o;
}

}  // namespace

extern "C" {

size_t bitcomp_dev_max_compressed_bytes(size_t n, int algo, int type) {
  return dev::max_compressed_bytes(n, opts_of(algo, type));
}
size_t bitcomp_dev_max_chunk_bytes() { return dev::kMaxChunkBytes; }
size_t bitcomp_dev_compress_smem_bytes() { return dev::kCompressSmemBytes; }
size_t bitcomp_dev_smem_alignment() { return dev::kSmemAlignment; }

int bitcomp_dev_compress(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes,
                         int* status, size_t batch, int algo, int type, cudaStream_t stream) {
  compress_kernel<<<ctas_for(batch), kWarps * 32, 0, stream>>>(in, in_bytes, out, comp_bytes, status, batch,
                                                                opts_of(algo, type));
  return (int)cudaGetLastError();
}

int bitcomp_dev_decompress(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                           size_t* actual, int* status, size_t batch, cudaStream_t stream) {
  decompress_kernel<<<ctas_for(batch), kWarps * 32, 0, stream>>>(comp, comp_bytes, out, caps, actual, status, batch);
  return (int)cudaGetLastError();
}

// elem: the visited element type as an nvcompType_t (CHAR .. ULONGLONG).
int bitcomp_dev_visit(const void* const* comp, const size_t* comp_bytes, unsigned long long* sums,
                      unsigned long long* hashes, unsigned long long* visits, int* status, size_t batch, int elem,
                      cudaStream_t stream) {
  const unsigned g = ctas_for(batch);
  switch (elem) {
    case NVCOMP_TYPE_CHAR: visit_kernel<int8_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_UCHAR: visit_kernel<uint8_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_SHORT: visit_kernel<int16_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_USHORT: visit_kernel<uint16_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_INT: visit_kernel<int32_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_UINT: visit_kernel<uint32_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_LONGLONG: visit_kernel<int64_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    case NVCOMP_TYPE_ULONGLONG: visit_kernel<uint64_t><<<g, kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch); break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}

int bitcomp_dev_mixed(const void* const* in, const size_t* in_bytes, void* const* cout, size_t* cbytes, int* cstatus,
                      size_t cbatch, int algo, int type, const void* const* comp, const size_t* comp_bytes,
                      void* const* dout, const size_t* caps, size_t* actual, int* dstatus, size_t dbatch,
                      const void* const* vcomp, const size_t* vcomp_bytes, unsigned long long* sums,
                      unsigned long long* hashes, unsigned long long* visits, int* vstatus, size_t vbatch,
                      cudaStream_t stream) {
  size_t most = cbatch > dbatch ? cbatch : dbatch;
  most = most > vbatch ? most : vbatch;
  mixed_kernel<<<ctas_for(3 * most), kWarps * 32, 0, stream>>>(
      in, in_bytes, cout, cbytes, cstatus, cbatch, opts_of(algo, type), comp, comp_bytes, dout, caps, actual, dstatus,
      dbatch, vcomp, vcomp_bytes, sums, hashes, visits, vstatus, vbatch);
  return (int)cudaGetLastError();
}

int bitcomp_dev_fused_sum(const void* const* comp, const size_t* comp_bytes, long long* sums, int* status,
                          size_t batch, cudaStream_t stream) {
  fused_sum_kernel<<<ctas_for(batch), kWarps * 32, 0, stream>>>(comp, comp_bytes, sums, status, batch);
  return (int)cudaGetLastError();
}

int bitcomp_dev_sum_i64(const void* const* data, const size_t* sizes, long long* sums, size_t batch,
                        cudaStream_t stream) {
  sum_i64_kernel<<<ctas_for(batch), kWarps * 32, 0, stream>>>(data, sizes, sums, batch);
  return (int)cudaGetLastError();
}

int bitcomp_dev_decompressed_size(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch,
                                  cudaStream_t stream) {
  if (batch == 0) return 0;
  size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp, comp_bytes, sizes, batch);
  return (int)cudaGetLastError();
}

}  // extern "C"
