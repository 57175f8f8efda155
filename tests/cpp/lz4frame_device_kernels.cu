// lz4frame_device_kernels.cu -- test and benchmark kernels over the warp-level LZ4 frame device API
// (nvcomp/device/lz4frame.cuh), built into build/tests/liblz4frame_device.so (and, with -rdc=true and a second
// translation unit that includes the same headers, build/tests/liblz4frame_device_rdc.so) and driven from Python
// (tests/test_lz4frame_device_gpu.py).  Every launcher takes device arrays in the batched C API's layout (pointers,
// sizes) and enqueues on `stream`; it returns the launch's cudaError_t.
//
// The kernels run kWarps warps per CTA, each with its own region of dynamic shared memory; warp gw takes chunks gw,
// gw + total_warps, ...
#include <cuda_runtime.h>

#include "nvcomp/device/lz4.cuh"
#include "nvcomp/device/lz4frame.cuh"

#ifndef LZ4F_LINK_ONLY

namespace lz4d = nvcomp::device::lz4;
namespace lz4fd = nvcomp::device::lz4frame;

namespace {

constexpr int kWarps = 4;
constexpr unsigned kMaxCtas = 132 * 16;
constexpr size_t kRegion = lz4fd::kDecompressSmemBytes;
static_assert(lz4fd::kDecompressSmemBytes == lz4d::kDecompressSmemBytes, "one decode region for both formats");
static_assert(kRegion % lz4fd::kSmemAlignment == 0, "aligned regions");

__device__ __forceinline__ size_t global_warp() { return ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ size_t total_warps() { return ((size_t)gridDim.x * blockDim.x) >> 5; }
__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

__device__ __forceinline__ uint8_t* warp_smem() {
  extern __shared__ __align__(16) unsigned char smem[];
  return smem + (size_t)(threadIdx.x >> 5) * kRegion;
}

// scribble: fill the warp's region with garbage after every call (the region holds nothing between calls)
__global__ void __launch_bounds__(kWarps * 32)
decompress_kernel(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                  size_t* actual, int* status, size_t n, int scribble) {
  uint8_t* sm = warp_smem();
  for (size_t c = global_warp(); c < n; c += total_warps()) {
    const nvcompStatus_t st = lz4fd::decompress_warp(comp[c], comp_bytes[c], out[c], caps[c], actual ? actual + c : nullptr, sm);
    if (lane() == 0 && status) status[c] = (int)st;
    if (scribble) {
      for (size_t i = (size_t)lane() * 4; i < kRegion; i += 128) *(uint32_t*)(sm + i) = 0xdeadbeefu ^ (uint32_t)(c + i);
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(kWarps * 32)
size_kernel(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t n) {
  for (size_t c = global_warp(); c < n; c += total_warps()) {
    const size_t s = lz4fd::decompressed_size_warp(comp[c], comp_bytes[c]);
    if (lane() == 0) sizes[c] = s;
  }
}

// even warps of a CTA decode LZ4 frames, odd warps raw LZ4 blocks (lz4::decompress_warp), at the same time
struct Batch {
  const void* const* comp;
  const size_t* comp_bytes;
  void* const* out;
  const size_t* caps;
  size_t* actual;
  int* status;
  size_t n;
};

__global__ void __launch_bounds__(kWarps * 32) mixed_kernel(Batch frames, Batch blocks) {
  uint8_t* sm = warp_smem();
  const bool frame_warp = ((threadIdx.x >> 5) & 1) == 0;
  const Batch& b = frame_warp ? frames : blocks;
  const size_t half = total_warps() / 2, me = global_warp() / 2;
  for (size_t c = me; c < b.n; c += half) {
    nvcompStatus_t st;
    if (frame_warp) st = lz4fd::decompress_warp(b.comp[c], b.comp_bytes[c], b.out[c], b.caps[c], b.actual + c, sm);
    else st = lz4d::decompress_warp(b.comp[c], b.comp_bytes[c], b.out[c], b.caps[c], b.actual + c, sm);
    if (lane() == 0) b.status[c] = (int)st;
  }
}

template <class K>
cudaError_t prepare(K kernel) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWarps * kRegion));
}

unsigned grid_for(size_t n) {
  const size_t ctas = (n + kWarps - 1) / kWarps;
  return (unsigned)(ctas < 1 ? 1 : ctas > kMaxCtas ? kMaxCtas : ctas);
}

}  // namespace

extern "C" {

size_t lz4f_dev_region_bytes() { return kRegion; }

int lz4f_dev_decompress(const void* const* comp, const size_t* comp_bytes, void* const* out, const size_t* caps,
                        size_t* actual, int* status, size_t n, int scribble, cudaStream_t stream) {
  cudaError_t e = prepare(decompress_kernel);
  if (e != cudaSuccess || n == 0) return (int)e;
  decompress_kernel<<<grid_for(n), kWarps * 32, kWarps * kRegion, stream>>>(comp, comp_bytes, out, caps, actual,
                                                                            status, n, scribble);
  return (int)cudaGetLastError();
}

int lz4f_dev_decompressed_size(const void* const* comp, const size_t* comp_bytes, size_t* sizes, size_t n,
                               cudaStream_t stream) {
  if (n == 0) return 0;
  size_kernel<<<grid_for(n), kWarps * 32, 0, stream>>>(comp, comp_bytes, sizes, n);
  return (int)cudaGetLastError();
}

int lz4f_dev_mixed(const void* const* fc, const size_t* fcb, void* const* fo, const size_t* fcap, size_t* fact,
                   int* fst, size_t fn, const void* const* bc, const size_t* bcb, void* const* bo, const size_t* bcap,
                   size_t* bact, int* bst, size_t bn, cudaStream_t stream) {
  cudaError_t e = prepare(mixed_kernel);
  if (e != cudaSuccess) return (int)e;
  const size_t n = fn > bn ? fn : bn;
  mixed_kernel<<<grid_for(2 * n), kWarps * 32, kWarps * kRegion, stream>>>(Batch{fc, fcb, fo, fcap, fact, fst, fn},
                                                                           Batch{bc, bcb, bo, bcap, bact, bst, bn});
  return (int)cudaGetLastError();
}

}  // extern "C"

#else

// second translation unit of the -rdc=true build: the same headers, one more kernel over them
__global__ void lz4f_link_probe(const void* comp, size_t n, size_t* size) {
  const size_t s = nvcomp::device::lz4frame::decompressed_size_warp(comp, n);
  if ((threadIdx.x & 31) == 0) *size = s;
}

#endif
