// ans_device_kernels.cu -- test and benchmark kernels over the warp-level ANS device API (nvcomp/device/ans.cuh),
// built into build/tests/libans_device.so and driven from Python (tests/test_ans_device_gpu.py,
// tools/ans_device_bench.py).  Every launcher takes device arrays in the batched C API's layout (pointers, sizes)
// and enqueues on `stream`; it returns the launch's cudaError_t.
//
// The kernels are persistent: kWarps warps per CTA, each warp takes chunks gw, gw + total_warps, ...  A warp that
// compresses uses tmp + gw * compress_tmp_bytes().
#include <cuda_runtime.h>

#include "nvcomp/device/ans.cuh"

namespace dev = nvcomp::device::ans;

namespace {

constexpr int kWarps = 4;
constexpr unsigned kMaxCtas = 132 * 4;
constexpr size_t kSmemPerWarp = dev::kDecompressSmemBytes;   // >= kCompressSmemBytes; every warp may do either
static_assert(dev::kCompressSmemBytes <= kSmemPerWarp, "one region serves both directions");
static_assert(kSmemPerWarp % dev::kSmemAlignment == 0, "regions stay aligned");

unsigned ctas_for(size_t batch) {
  const size_t need = (batch + kWarps - 1) / kWarps;
  return (unsigned)(need < kMaxCtas ? (need ? need : 1) : kMaxCtas);
}

__device__ __forceinline__ void* warp_smem() {
  extern __shared__ __align__(1024) unsigned char smem[];
  return smem + (threadIdx.x >> 5) * kSmemPerWarp;
}

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }

__device__ __forceinline__ void decompress_one(const void* const* comp, const size_t* comp_bytes, void* const* out,
                                               const size_t* caps, size_t* actual, int* status, size_t c) {
  const nvcompStatus_t st = dev::decompress_warp(comp[c], comp_bytes[c], out[c], caps[c], actual + c, warp_smem());
  if ((threadIdx.x & 31) == 0) status[c] = (int)st;
}

__device__ __forceinline__ void compress_one(const void* const* in, const size_t* in_bytes, void* const* out,
                                             size_t* comp_bytes, int* status, uint8_t* tmp, size_t c) {
  const nvcompStatus_t st = dev::compress_warp(in[c], in_bytes[c], out[c], comp_bytes + c, warp_smem(), tmp);
  if ((threadIdx.x & 31) == 0) status[c] = (int)st;
}

__global__ void __launch_bounds__(kWarps * 32)
decompress_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, size_t batch) {
  for (size_t c = global_warp(); c < batch; c += total_warps()) decompress_one(comp, comp_bytes, out, caps, actual, status, c);
}

__global__ void __launch_bounds__(kWarps * 32)
compress_kernel(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                size_t batch, uint8_t* tmp) {
  uint8_t* my_tmp = tmp + global_warp() * dev::compress_tmp_bytes();
  for (size_t c = global_warp(); c < batch; c += total_warps()) compress_one(in, in_bytes, out, comp_bytes, status, my_tmp, c);
}

// Even warps compress chunks of one batch while the odd warps of the same CTAs decompress another.
__global__ void __launch_bounds__(kWarps * 32)
mixed_kernel(const void* const* in, const size_t* in_bytes, void* const* cout, size_t* cbytes, int* cstatus,
             size_t cbatch, uint8_t* tmp, const void* const* comp, const size_t* comp_bytes, void* const* dout,
             const size_t* caps, size_t* actual, int* dstatus, size_t dbatch) {
  const size_t gw = global_warp() >> 1, stride = total_warps() >> 1;
  if ((global_warp() & 1) == 0) {
    uint8_t* my_tmp = tmp + gw * dev::compress_tmp_bytes();
    for (size_t c = gw; c < cbatch; c += stride) compress_one(in, in_bytes, cout, cbytes, cstatus, my_tmp, c);
  } else {
    for (size_t c = gw; c < dbatch; c += stride) decompress_one(comp, comp_bytes, dout, caps, actual, dstatus, c);
  }
}

// Decode a chunk and reduce it in the same kernel: the byte sum and the 256-bin histogram of the decoded bytes.
// The warp's decode shared memory is free after the decode and holds the histogram.
__global__ void __launch_bounds__(kWarps * 32)
fused_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
             size_t* actual, int* status, unsigned long long* sums, unsigned* hists, size_t batch) {
  const int lane = threadIdx.x & 31;
  unsigned* s_hist = (unsigned*)warp_smem();
  for (size_t c = global_warp(); c < batch; c += total_warps()) {
    size_t got = 0;
    const nvcompStatus_t st = dev::decompress_warp(comp[c], comp_bytes[c], out[c], caps[c], &got, warp_smem());
    got = __shfl_sync(0xffffffffu, got, 0);         // written by lane 0
    __syncwarp();                                   // the decoded bytes and the free smem are visible to all lanes
    for (int i = lane; i < 256; i += 32) s_hist[i] = 0;
    __syncwarp();
    const uint8_t* o = (const uint8_t*)out[c];
    unsigned long long sum = 0;
    for (size_t i = lane; i < got; i += 32) {
      const uint8_t b = o[i];
      sum += b;
      atomicAdd(&s_hist[b], 1u);
    }
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    __syncwarp();
    for (int i = lane; i < 256; i += 32) hists[c * 256 + i] = s_hist[i];
    if (lane == 0) { actual[c] = got; status[c] = (int)st; sums[c] = sum; }
    __syncwarp();                                   // s_hist is the next decode's smem
  }
}

__global__ void size_kernel(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < batch) sizes[c] = dev::decompressed_size(comp[c], comp_bytes[c]);
}

cudaError_t set_smem(const void* fn) {
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWarps * kSmemPerWarp));
}

}  // namespace

extern "C" {

size_t ans_dev_max_compressed_bytes(size_t n) { return dev::max_compressed_bytes(n); }
size_t ans_dev_max_chunk_bytes() { return dev::kMaxChunkBytes; }
size_t ans_dev_decompress_smem_bytes() { return dev::kDecompressSmemBytes; }
size_t ans_dev_compress_smem_bytes() { return dev::kCompressSmemBytes; }
size_t ans_dev_smem_alignment() { return dev::kSmemAlignment; }

// Global scratch the compress (and mixed) launchers need for `batch` chunks.
size_t ans_dev_compress_temp_bytes(size_t batch) {
  return (size_t)ctas_for(batch) * kWarps * dev::compress_tmp_bytes();
}

int ans_dev_decompress(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                       size_t* actual, int* status, size_t batch, cudaStream_t stream) {
  cudaError_t e = set_smem((const void*)decompress_kernel);
  if (e != cudaSuccess) return (int)e;
  decompress_kernel<<<ctas_for(batch), kWarps * 32, kWarps * kSmemPerWarp, stream>>>(
      comp, comp_bytes, out, caps, actual, status, batch);
  return (int)cudaGetLastError();
}

int ans_dev_compress(const void* const* in, const size_t* in_bytes, void* const* out, size_t* comp_bytes, int* status,
                     size_t batch, void* tmp, cudaStream_t stream) {
  cudaError_t e = set_smem((const void*)compress_kernel);
  if (e != cudaSuccess) return (int)e;
  compress_kernel<<<ctas_for(batch), kWarps * 32, kWarps * kSmemPerWarp, stream>>>(
      in, in_bytes, out, comp_bytes, status, batch, (uint8_t*)tmp);
  return (int)cudaGetLastError();
}

// tmp: ans_dev_compress_temp_bytes(max(cbatch, dbatch)) bytes.
int ans_dev_mixed(const void* const* in, const size_t* in_bytes, void* const* cout, size_t* cbytes, int* cstatus,
                  size_t cbatch, void* tmp, const void* const* comp, const size_t* comp_bytes, void* const* dout,
                  const size_t* caps, size_t* actual, int* dstatus, size_t dbatch, cudaStream_t stream) {
  cudaError_t e = set_smem((const void*)mixed_kernel);
  if (e != cudaSuccess) return (int)e;
  mixed_kernel<<<ctas_for(cbatch > dbatch ? cbatch : dbatch), kWarps * 32, kWarps * kSmemPerWarp, stream>>>(
      in, in_bytes, cout, cbytes, cstatus, cbatch, (uint8_t*)tmp, comp, comp_bytes, dout, caps, actual, dstatus,
      dbatch);
  return (int)cudaGetLastError();
}

int ans_dev_fused(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, unsigned long long* sums, unsigned* hists, size_t batch,
                  cudaStream_t stream) {
  cudaError_t e = set_smem((const void*)fused_kernel);
  if (e != cudaSuccess) return (int)e;
  fused_kernel<<<ctas_for(batch), kWarps * 32, kWarps * kSmemPerWarp, stream>>>(
      comp, comp_bytes, out, caps, actual, status, sums, hists, batch);
  return (int)cudaGetLastError();
}

int ans_dev_decompressed_size(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t batch,
                              cudaStream_t stream) {
  if (batch == 0) return 0;
  size_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, stream>>>(comp, comp_bytes, sizes, batch);
  return (int)cudaGetLastError();
}

}  // extern "C"
