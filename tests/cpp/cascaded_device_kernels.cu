// cascaded_device_kernels.cu -- test and benchmark kernels over the warp-level Cascaded device API
// (nvcomp/device/cascaded.cuh), built into build/tests/libcascaded_device.so and driven from Python
// (tests/test_cascaded_device_gpu.py, tools/cascaded_device_bench.py).  Every launcher takes device arrays in the
// batched C API's layout (pointers, sizes) and enqueues on `stream`; it returns the launch's cudaError_t.
//
// The kernels are persistent: each warp takes chunks gw, gw + total_warps, ...  Every warp owns `region` bytes of
// dynamic shared memory (a multiple of kSmemAlignment), and a CTA holds as many warps (<= kWarps) as fit in the
// opt-in limit, so a region of kMaxDecompressSmemBytes runs 3 warps per CTA.
#include <cuda_runtime.h>

#include <type_traits>

#include "nvcomp/device/cascaded.cuh"

namespace dev = nvcomp::device::cascaded;

namespace {

constexpr int kWarps = 4;
constexpr unsigned kMaxCtas = 132 * 16;
constexpr unsigned kFull = 0xffffffffu;
constexpr size_t kSmemOptIn = 227 * 1024;

struct Launch { unsigned ctas, threads; size_t smem; };

// CTAs of min(kWarps, what fits) warps of `region` bytes each, enough for one warp per chunk (up to kMaxCtas).
// threads = 0 when one warp does not fit.
Launch launch_for(size_t batch, size_t region, int max_warps = kWarps) {
  const size_t fit = region ? kSmemOptIn / region : (size_t)max_warps;
  const int w = (int)(fit < (size_t)max_warps ? fit : (size_t)max_warps);
  if (w < 1) return {0, 0, 0};
  const size_t need = (batch + w - 1) / w;
  return {(unsigned)(need < kMaxCtas ? (need ? need : 1) : kMaxCtas), (unsigned)(32 * w), (size_t)w * region};
}

template <class K>
cudaError_t prepare(K kernel) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOptIn);
}

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }
__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

__device__ __forceinline__ void* warp_smem(size_t region) {
  extern __shared__ __align__(dev::kSmemAlignment) unsigned char smem[];
  return smem + (threadIdx.x >> 5) * region;
}

__device__ __forceinline__ void compress_one(const void* const* in, const size_t* in_bytes, void* const* out,
                                             size_t* comp_bytes, int* status, nvcompBatchedCascadedOpts_t opts,
                                             void* sm, size_t c) {
  const nvcompStatus_t st = dev::compress_warp(in[c], in_bytes[c], out[c], comp_bytes + c, opts, sm);
  if (lane() == 0) status[c] = (int)st;
}

__device__ __forceinline__ void decompress_one(const void* const* comp, const size_t* comp_bytes, void* const* out,
                                               const size_t* caps, size_t* actual, int* status, void* sm,
                                               size_t region, size_t c) {
  const nvcompStatus_t st = dev::decompress_warp(comp[c], comp_bytes[c], out[c], caps[c], actual + c, sm, region);
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
                                          void* sm, size_t region, size_t c) {
  uint64_t sum = 0, hash = 0, nvis = 0;
  const nvcompStatus_t st = dev::for_each_block<T>(comp[c], comp_bytes[c], sm, region,
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
                size_t batch, nvcompBatchedCascadedOpts_t opts, size_t region) {
  for (size_t c = global_warp(); c < batch; c += total_warps())
    compress_one(in, in_bytes, out, comp_bytes, status, opts, warp_smem(region), c);
}

__global__ void __launch_bounds__(kWarps * 32)
decompress_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, size_t batch, size_t region) {
  for (size_t c = global_warp(); c < batch; c += total_warps())
    decompress_one(comp, comp_bytes, out, caps, actual, status, warp_smem(region), region, c);
}

template <class T>
__global__ void __launch_bounds__(kWarps * 32)
visit_kernel(const void* const* comp, const size_t* comp_bytes, unsigned long long* sums, unsigned long long* hashes,
             unsigned long long* visits, int* status, size_t batch, size_t region) {
  for (size_t c = global_warp(); c < batch; c += total_warps())
    visit_one<T>(comp, comp_bytes, sums, hashes, visits, status, warp_smem(region), region, c);
}

// Warp 0 of every CTA compresses chunks of one batch, warp 1 decompresses chunks of another and warp 2 visits a third
// (as int64), side by side in the same CTA.
__global__ void __launch_bounds__(kWarps * 32)
mixed_kernel(const void* const* in, const size_t* in_bytes, void* const* cout, size_t* cbytes, int* cstatus,
             size_t cbatch, nvcompBatchedCascadedOpts_t opts, const void* const* comp, const size_t* comp_bytes,
             void* const* dout, const size_t* caps, size_t* actual, int* dstatus, size_t dbatch,
             const void* const* vcomp, const size_t* vcomp_bytes, unsigned long long* sums,
             unsigned long long* hashes, unsigned long long* visits, int* vstatus, size_t vbatch, size_t region) {
  const size_t role = threadIdx.x >> 5, gw = blockIdx.x, stride = gridDim.x;   // (three warps per CTA)
  void* sm = warp_smem(region);
  if (role == 0) {
    for (size_t c = gw; c < cbatch; c += stride) compress_one(in, in_bytes, cout, cbytes, cstatus, opts, sm, c);
  } else if (role == 1) {
    for (size_t c = gw; c < dbatch; c += stride)
      decompress_one(comp, comp_bytes, dout, caps, actual, dstatus, sm, region, c);
  } else {
    for (size_t c = gw; c < vbatch; c += stride)
      visit_one<int64_t>(vcomp, vcomp_bytes, sums, hashes, visits, vstatus, sm, region, c);
  }
}

// The fused path of the benchmark: the wrapping int64 sum of every chunk, decoded in registers.
__global__ void __launch_bounds__(kWarps * 32)
fused_sum_kernel(const void* const* comp, const size_t* comp_bytes, long long* sums, int* status, size_t batch,
                 size_t region) {
  void* sm = warp_smem(region);
  for (size_t c = global_warp(); c < batch; c += total_warps()) {
    uint64_t sum = 0;
    const nvcompStatus_t st = dev::for_each_block<int64_t>(comp[c], comp_bytes[c], sm, region,
        [&](const int64_t (&v)[4], uint32_t, uint32_t valid) {
#pragma unroll
          for (uint32_t k = 0; k < 4; ++k) sum += k < valid ? (uint64_t)v[k] : 0ull;
        });
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
    if (lane() == 0) { sums[c] = (long long)sum; status[c] = (int)st; }
  }
}

// for_each_block's first pass alone (the partition walk that unpacks only the run-length streams), on 8-byte
// streams: 1 when the chunk would be visited.  It reaches into the API's detail namespace (header_smem_bytes,
// walk_chunk), so it follows for_each_block's first steps by hand; test_cascaded_device_gpu.py holds its verdicts to
// for_each_block's, so a change in detail that breaks it fails there.
__global__ void __launch_bounds__(kWarps * 32)
check_kernel(const void* const* comp, const size_t* comp_bytes, int* ok, size_t batch, size_t region) {
  namespace d = dev::detail;
  uint8_t* sm = (uint8_t*)warp_smem(region);
  for (size_t c = global_warp(); c < batch; c += total_warps()) {
    const uint8_t* in = (const uint8_t*)comp[c];
    d::CascHeader h;
    bool good = d::casc_read_header(in, comp_bytes[c], h) && d::casc_type_size(h.type) == 8 &&
                d::header_smem_bytes(h) <= region;
    good = good && d::walk_chunk<8, d::kCascCheck>(in, comp_bytes[c], h, nullptr, sm, d::CascNoVisit(), lane());
    if (lane() == 0) ok[c] = good ? 1 : 0;
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

template <class T>
int launch_visit(const void* const* comp, const size_t* comp_bytes, unsigned long long* sums,
                 unsigned long long* hashes, unsigned long long* visits, int* status, size_t batch, size_t region,
                 cudaStream_t stream) {
  const Launch l = launch_for(batch, region);
  if (!l.threads) return (int)cudaErrorInvalidValue;
  cudaError_t e = prepare(visit_kernel<T>);
  if (e != cudaSuccess) return (int)e;
  visit_kernel<T><<<l.ctas, l.threads, l.smem, stream>>>(comp, comp_bytes, sums, hashes, visits, status, batch, region);
  return (int)cudaGetLastError();
}

nvcompBatchedCascadedOpts_t opts_of(size_t chunk_size, int type, int rle, int delta, int bp) {
  nvcompBatchedCascadedOpts_t o;
  o.chunk_size = chunk_size;
  o.type = (nvcompType_t)type;
  o.num_RLEs = rle;
  o.num_deltas = delta;
  o.use_bp = bp;
  return o;
}

}  // namespace

extern "C" {

size_t cascaded_dev_max_compressed_bytes(size_t n, size_t chunk_size, int type, int rle, int delta, int bp) {
  return dev::max_compressed_bytes(n, opts_of(chunk_size, type, rle, delta, bp));
}
size_t cascaded_dev_compress_smem_bytes(size_t chunk_size, int type, int rle, int delta, int bp) {
  return dev::compress_smem_bytes(opts_of(chunk_size, type, rle, delta, bp));
}
size_t cascaded_dev_decompress_smem_bytes(size_t chunk_size, int type, int rle, int delta, int bp) {
  return dev::decompress_smem_bytes(opts_of(chunk_size, type, rle, delta, bp));
}
size_t cascaded_dev_max_decompress_smem_bytes() { return dev::kMaxDecompressSmemBytes; }
size_t cascaded_dev_max_chunk_bytes() { return dev::kMaxChunkBytes; }
size_t cascaded_dev_smem_alignment() { return dev::kSmemAlignment; }

// The compress launcher sizes each warp's region with compress_smem_bytes(opts) (one warp's worth of 16 bytes for
// options it rejects, so the kernel still reports their status).
int cascaded_dev_compress(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes,
                          int* status, size_t batch, size_t chunk_size, int type, int rle, int delta, int bp,
                          cudaStream_t stream) {
  const nvcompBatchedCascadedOpts_t o = opts_of(chunk_size, type, rle, delta, bp);
  size_t region = dev::compress_smem_bytes(o);
  if (region == 0) region = dev::kSmemAlignment;
  const Launch l = launch_for(batch, region);
  cudaError_t e = prepare(compress_kernel);
  if (e != cudaSuccess) return (int)e;
  compress_kernel<<<l.ctas, l.threads, l.smem, stream>>>(in, in_bytes, out, comp_bytes, status, batch, o, region);
  return (int)cudaGetLastError();
}

// region: each warp's decode workspace in bytes (a multiple of kSmemAlignment).
int cascaded_dev_decompress(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                            size_t* actual, int* status, size_t batch, size_t region, cudaStream_t stream) {
  const Launch l = launch_for(batch, region);
  if (!l.threads) return (int)cudaErrorInvalidValue;
  cudaError_t e = prepare(decompress_kernel);
  if (e != cudaSuccess) return (int)e;
  decompress_kernel<<<l.ctas, l.threads, l.smem, stream>>>(comp, comp_bytes, out, caps, actual, status, batch, region);
  return (int)cudaGetLastError();
}

// elem: the visited element type as an nvcompType_t (CHAR .. ULONGLONG).
int cascaded_dev_visit(const void* const* comp, const size_t* comp_bytes, unsigned long long* sums,
                       unsigned long long* hashes, unsigned long long* visits, int* status, size_t batch, int elem,
                       size_t region, cudaStream_t stream) {
  switch (elem) {
    case NVCOMP_TYPE_CHAR: return launch_visit<int8_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_UCHAR: return launch_visit<uint8_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_SHORT: return launch_visit<int16_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_USHORT: return launch_visit<uint16_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_INT: return launch_visit<int32_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_UINT: return launch_visit<uint32_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_LONGLONG: return launch_visit<int64_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    case NVCOMP_TYPE_ULONGLONG: return launch_visit<uint64_t>(comp, comp_bytes, sums, hashes, visits, status, batch, region, stream);
    default: return (int)cudaErrorInvalidValue;
  }
}

// Three warps per CTA (one of each role), each with max(compress_smem_bytes(opts), dregion) bytes.
int cascaded_dev_mixed(const void* const* in, const size_t* in_bytes, void* const* cout, size_t* cbytes, int* cstatus,
                       size_t cbatch, size_t chunk_size, int type, int rle, int delta, int bp,
                       const void* const* comp, const size_t* comp_bytes, void* const* dout, const size_t* caps,
                       size_t* actual, int* dstatus, size_t dbatch, const void* const* vcomp,
                       const size_t* vcomp_bytes, unsigned long long* sums, unsigned long long* hashes,
                       unsigned long long* visits, int* vstatus, size_t vbatch, size_t dregion, cudaStream_t stream) {
  const nvcompBatchedCascadedOpts_t o = opts_of(chunk_size, type, rle, delta, bp);
  size_t region = dev::compress_smem_bytes(o);
  region = region > dregion ? region : dregion;
  size_t most = cbatch > dbatch ? cbatch : dbatch;
  most = most > vbatch ? most : vbatch;
  if (3 * region > kSmemOptIn) return (int)cudaErrorInvalidValue;
  cudaError_t e = prepare(mixed_kernel);
  if (e != cudaSuccess) return (int)e;
  const unsigned ctas = (unsigned)(most < kMaxCtas ? (most ? most : 1) : kMaxCtas);
  mixed_kernel<<<ctas, 3 * 32, 3 * region, stream>>>(
      in, in_bytes, cout, cbytes, cstatus, cbatch, o, comp, comp_bytes, dout, caps, actual, dstatus, dbatch, vcomp,
      vcomp_bytes, sums, hashes, visits, vstatus, vbatch, region);
  return (int)cudaGetLastError();
}

int cascaded_dev_fused_sum(const void* const* comp, const size_t* comp_bytes, long long* sums, int* status,
                           size_t batch, size_t region, cudaStream_t stream) {
  const Launch l = launch_for(batch, region);
  if (!l.threads) return (int)cudaErrorInvalidValue;
  cudaError_t e = prepare(fused_sum_kernel);
  if (e != cudaSuccess) return (int)e;
  fused_sum_kernel<<<l.ctas, l.threads, l.smem, stream>>>(comp, comp_bytes, sums, status, batch, region);
  return (int)cudaGetLastError();
}

int cascaded_dev_check(const void* const* comp, const size_t* comp_bytes, int* ok, size_t batch, size_t region,
                       cudaStream_t stream) {
  const Launch l = launch_for(batch, region);
  if (!l.threads) return (int)cudaErrorInvalidValue;
  cudaError_t e = prepare(check_kernel);
  if (e != cudaSuccess) return (int)e;
  check_kernel<<<l.ctas, l.threads, l.smem, stream>>>(comp, comp_bytes, ok, batch, region);
  return (int)cudaGetLastError();
}

int cascaded_dev_sum_i64(const void* const* data, const size_t* sizes, long long* sums, size_t batch,
                         cudaStream_t stream) {
  const Launch l = launch_for(batch, 0);
  sum_i64_kernel<<<l.ctas, l.threads, 0, stream>>>(data, sizes, sums, batch);
  return (int)cudaGetLastError();
}

int cascaded_dev_decompressed_size(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch,
                                   cudaStream_t stream) {
  if (batch == 0) return 0;
  size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp, comp_bytes, sizes, batch);
  return (int)cudaGetLastError();
}

}  // extern "C"
