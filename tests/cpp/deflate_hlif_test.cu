// deflate_hlif_test.cu -- GPU test of DeflateManager and create_manager on a Deflate container.  Built by the Makefile
// into build/tests/deflate_hlif_test, run by tests/test_deflate_compress_gpu.py.  Exit code 0 = all checks passed.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "nvcomp.hpp"
#include "nvcomp/nvcompManagerFactory.hpp"

using namespace nvcomp;

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(2); } } while (0)
#define REQUIRE(c) do { if (!(c)) { printf("FAILED: %s (line %d)\n", #c, __LINE__); exit(1); } } while (0)

static std::vector<uint8_t> make_data(size_t n, int kind, uint32_t seed) {
  std::mt19937 rng(seed);
  std::vector<uint8_t> v(n);
  if (kind == 0) { for (auto& b : v) b = (uint8_t)(rng() & 3); }                 // low entropy
  else if (kind == 1) {                                                          // int32 run-length
    size_t i = 0;
    while (i < n) { uint32_t val = rng(); size_t run = 4 * (1 + rng() % 256);
      for (size_t k = 0; k < run && i < n; ++k, ++i) v[i] = (uint8_t)(val >> (8 * (i & 3))); }
  } else { for (auto& b : v) b = (uint8_t)rng(); }                               // incompressible
  return v;
}

// compress with mgr, decompress with mgr itself or with the manager create_manager builds from the buffer
static void roundtrip(nvcompManagerBase& mgr, const std::vector<uint8_t>& host, cudaStream_t stream, bool via_factory,
                      ChecksumPolicy policy) {
  const size_t n = host.size();
  uint8_t* d_in; CK(cudaMalloc(&d_in, n ? n : 1));
  CK(cudaMemcpy(d_in, host.data(), n, cudaMemcpyHostToDevice));
  CompressionConfig cc = mgr.configure_compression(n);
  uint8_t* d_comp; CK(cudaMalloc(&d_comp, cc.max_compressed_buffer_size));
  mgr.compress(d_in, d_comp, cc);
  CK(cudaStreamSynchronize(stream));
  REQUIRE(*cc.get_status() == nvcompSuccess);
  const size_t csize = mgr.get_compressed_output_size(d_comp);
  REQUIRE(csize > 0 && csize <= cc.max_compressed_buffer_size);
  std::shared_ptr<nvcompManagerBase> other;
  nvcompManagerBase* dm = &mgr;
  if (via_factory) {
    other = create_manager(d_comp, stream, 0, policy);
    REQUIRE(dynamic_cast<DeflateManager*>(other.get()) != nullptr);
    dm = other.get();
  }
  DecompressionConfig dc = dm->configure_decompression(d_comp);
  REQUIRE(dc.decomp_data_size == n);
  uint8_t* d_out; CK(cudaMalloc(&d_out, n ? n : 1));
  CK(cudaMemset(d_out, 0xA5, n ? n : 1));
  dm->decompress(d_out, d_comp, dc);
  CK(cudaStreamSynchronize(stream));
  REQUIRE(*dc.get_status() == nvcompSuccess);
  std::vector<uint8_t> back(n);
  CK(cudaMemcpy(back.data(), d_out, n, cudaMemcpyDeviceToHost));
  REQUIRE(back == host);
  CK(cudaFree(d_in)); CK(cudaFree(d_comp)); CK(cudaFree(d_out));
}

int main() {
  cudaStream_t stream; CK(cudaStreamCreate(&stream));
  const ChecksumPolicy policies[] = {NoComputeNoVerify, ComputeAndNoVerify, NoComputeAndVerifyIfPresent,
                                     ComputeAndVerifyIfPresent, ComputeAndVerify};
  const size_t sizes[] = {0, 1, 65535, 65536, 65537, 1000000};
  int cases = 0;
  for (int algo = 0; algo < 3; ++algo)
    for (ChecksumPolicy pol : policies)
      for (size_t n : sizes)
        for (int kind = 0; kind < 3; ++kind) {
          DeflateManager mgr{1 << 16, nvcompBatchedDeflateOpts_t{algo}, stream, 0, pol};
          roundtrip(mgr, make_data(n, kind, 31 * algo + kind), stream, /*via_factory=*/(kind + (int)n) % 2 == 0, pol);
          ++cases;
        }
  // an algo outside 0..2, or a chunk over 64 KB, is refused at construction
  for (int bad : {-1, 3}) {
    bool threw = false;
    try { DeflateManager m{1 << 16, nvcompBatchedDeflateOpts_t{bad}, stream}; }
    catch (const NVCompException& e) { threw = e.get_error() == nvcompErrorInvalidValue; }
    REQUIRE(threw);
  }
  {
    bool threw = false;
    try { DeflateManager m{(1 << 16) + 1, nvcompBatchedDeflateDefaultOpts, stream}; }
    catch (const NVCompException& e) { threw = e.get_error() == nvcompErrorChunkSizeTooLarge; }
    REQUIRE(threw);
  }
  printf("deflate_hlif_test ok: %d round trips + option checks\n", cases);
  return 0;
}
