// hlif.cu -- high-level interface (nvcomp::*Manager, create_manager) over the low-level batched API.
//
// Replaces the closed HLIF of nvCOMP 3.0.3 (include/nvcomp/nvcompManager.hpp cites the call sites).
// Since 3.0.0 the reference HLIF "dispatches to LLIF" (CHANGELOG.md:17); this one does the same:
//   compress  : chunk-pointer setup kernel -> nvcompBatched<Fmt>CompressAsync into scratch ->
//               scan of chunk sizes + header/table write -> gather kernel compacting the chunks
//   decompress: scan of the size table -> pointer setup -> nvcompBatched<Fmt>DecompressAsync ->
//               status reduction into pinned host memory (DecompressionConfig::get_status()).
// Container (8-byte aligned):
//   HlifHeader (72 B) | u64 chunk_bytes[num_chunks] | chunks (each 8-byte aligned)
// Checksums (optional, ChecksumPolicy; reference doc/highlevel_cpp_quickstart.md:59, policies at
// examples/high_level_quickstart_example.cpp:244-322): CRC-32 (crc32.cu) of the whole uncompressed buffer and
// of the whole compressed payload -- size table and every chunk, i.e. all bytes after the header.
#include <cuda_runtime.h>

#include <cstddef>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "common.cuh"
#include "crc32.cuh"
#include "nvcomp/nvcompManagerFactory.hpp"

namespace nvcomp {
namespace detail {

constexpr uint32_t kHlifMagic = 0x3242564eu;   // "NVB2"
enum FormatId : uint32_t { kFmtLZ4 = 1, kFmtSnappy = 2, kFmtCascaded = 3, kFmtBitcomp = 4, kFmtANS = 5,
                        kFmtDeflate = 6 };

struct HlifHeader {
  uint32_t magic;
  uint32_t format;
  uint8_t opts[24];
  uint64_t uncompressed_bytes;
  uint64_t chunk_bytes;
  uint32_t num_chunks;
  uint32_t flags;            // bit0: checksums present
  uint64_t total_bytes;      // header + table + chunks; written by the device
  uint32_t checksum_uncomp;
  uint32_t checksum_comp;
};
static_assert(sizeof(HlifHeader) == 72, "header layout");
constexpr size_t kHeaderBytes = 72;

struct StatusHolder {
  nvcompStatus_t* host = nullptr;     // pinned
  StatusHolder() { if (cudaMallocHost(&host, sizeof(nvcompStatus_t)) != cudaSuccess) host = nullptr; else *host = nvcompSuccess; }
  ~StatusHolder() { if (host) cudaFreeHost(host); }
};

// Type-erased binding of one format's LLIF entry points with its options captured.
struct FormatBinding {
  uint32_t format = 0;
  uint8_t opts[24] = {0};
  // chunk sizes must be a multiple of this, so that every chunk pointer the manager derives (input, output, container)
  // keeps the alignment the low-level decoder requires: the typed codecs reject chunk pointers that are not 8-byte
  // aligned and outputs not aligned to the element size
  size_t chunk_multiple = 1;
  nvcompStatus_t (*comp_temp)(const FormatBinding&, size_t, size_t, size_t*) = nullptr;
  nvcompStatus_t (*comp_max)(const FormatBinding&, size_t, size_t*) = nullptr;
  nvcompStatus_t (*comp)(const FormatBinding&, const void* const*, const size_t*, size_t, size_t, void*, size_t,
                         void* const*, size_t*, cudaStream_t) = nullptr;
  nvcompStatus_t (*decomp_temp)(size_t, size_t, size_t*) = nullptr;
  nvcompStatus_t (*decomp)(const void* const*, const size_t*, const size_t*, size_t*, size_t, void* const, size_t,
                           void* const*, nvcompStatus_t*, cudaStream_t) = nullptr;
};

template <class Opts>
static Opts opts_of(const FormatBinding& b) { Opts o; std::memcpy(&o, b.opts, sizeof(Opts)); return o; }

#define B200_BIND(FMT, OPTS, ID, MULTIPLE)                                                                   \
  static FormatBinding bind_##FMT(const OPTS& o) {                                                           \
    static_assert(sizeof(OPTS) <= 24, "opts blob");                                                         \
    FormatBinding b;                                                                                         \
    b.format = ID; b.chunk_multiple = MULTIPLE;                                                              \
    std::memcpy(b.opts, &o, sizeof(OPTS));                                                                   \
    b.comp_temp = [](const FormatBinding& f, size_t n, size_t m, size_t* t) {                                \
      return nvcompBatched##FMT##CompressGetTempSize(n, m, opts_of<OPTS>(f), t); };                          \
    b.comp_max = [](const FormatBinding& f, size_t m, size_t* t) {                                           \
      return nvcompBatched##FMT##CompressGetMaxOutputChunkSize(m, opts_of<OPTS>(f), t); };                   \
    b.comp = [](const FormatBinding& f, const void* const* ip, const size_t* ib, size_t m, size_t n, void* tp, \
                size_t tb, void* const* op, size_t* ob, cudaStream_t s) {                                    \
      return nvcompBatched##FMT##CompressAsync(ip, ib, m, n, tp, tb, op, ob, opts_of<OPTS>(f), s); };        \
    b.decomp_temp = nvcompBatched##FMT##DecompressGetTempSize;                                               \
    b.decomp = nvcompBatched##FMT##DecompressAsync;                                                          \
    return b;                                                                                                \
  }

B200_BIND(LZ4, nvcompBatchedLZ4Opts_t, kFmtLZ4, 1)
B200_BIND(Snappy, nvcompBatchedSnappyOpts_t, kFmtSnappy, 1)
B200_BIND(Cascaded, nvcompBatchedCascadedOpts_t, kFmtCascaded, nvcompCascadedRequiredAlignment)
B200_BIND(Bitcomp, nvcompBatchedBitcompFormatOpts, kFmtBitcomp, nvcompBitcompRequiredAlignment)
B200_BIND(ANS, nvcompBatchedANSOpts_t, kFmtANS, 1)
B200_BIND(Deflate, nvcompBatchedDeflateOpts_t, kFmtDeflate, 1)

static void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw NVCompException(nvcompErrorCudaError, std::string(what) + ": " + cudaGetErrorString(e));
}
static void check(nvcompStatus_t s, const char* what) {
  if (s != nvcompSuccess) throw NVCompException(s, what);
}

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------
__global__ void hlif_setup_compress(const uint8_t* in, size_t n, size_t chunk, size_t num_chunks, uint8_t* scratch_out,
                                    size_t max_out, const void** in_ptrs, size_t* in_bytes, void** out_ptrs) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num_chunks) return;
  in_ptrs[i] = in + i * chunk;
  in_bytes[i] = (i + 1 < num_chunks) ? chunk : n - i * chunk;
  out_ptrs[i] = scratch_out + i * max_out;
}

// single-CTA exclusive scan of 8-byte aligned chunk sizes -> offsets; writes header + size table
__global__ void __launch_bounds__(1024)
hlif_layout(const size_t* comp_bytes, size_t num_chunks, HlifHeader hdr, uint8_t* comp_buffer, size_t* offsets) {
  __shared__ unsigned long long s_warp[32];
  __shared__ unsigned long long s_carry;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  unsigned long long* table = (unsigned long long*)(comp_buffer + kHeaderBytes);
  const size_t payload0 = kHeaderBytes + 8 * num_chunks;
  for (size_t base = 0; base < num_chunks; base += blockDim.x) {
    const size_t i = base + threadIdx.x;
    const unsigned long long sz = (i < num_chunks) ? (unsigned long long)comp_bytes[i] : 0ull;
    const unsigned long long al = (sz + 7ull) & ~7ull;
    unsigned long long incl = al;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long o = __shfl_up_sync(b200::kFull, incl, d);
      if (lane >= d) incl += o;
    }
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    unsigned long long wbase = 0;
    for (int k = 0; k < w; ++k) wbase += s_warp[k];
    const unsigned long long excl = s_carry + wbase + incl - al;
    if (i < num_chunks) { offsets[i] = payload0 + excl; table[i] = sz; }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = excl + al;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    hdr.total_bytes = payload0 + s_carry;
    *(HlifHeader*)comp_buffer = hdr;
  }
}

// one CTA per chunk: copy the compressed chunk from scratch to its final place
__global__ void hlif_gather(const void* const* scratch_ptrs, const size_t* comp_bytes, const size_t* offsets,
                            uint8_t* comp_buffer) {
  const size_t c = blockIdx.x;
  const uint8_t* src = (const uint8_t*)scratch_ptrs[c];
  uint8_t* dst = comp_buffer + offsets[c];
  const size_t n = comp_bytes[c];
  const size_t nv = n >> 3;     // both 8-byte aligned
  const unsigned long long* s8 = (const unsigned long long*)src;
  unsigned long long* d8 = (unsigned long long*)dst;
  for (size_t i = threadIdx.x; i < nv; i += blockDim.x) d8[i] = s8[i];
  for (size_t i = (nv << 3) + threadIdx.x; i < ((n + 7) & ~(size_t)7); i += blockDim.x) dst[i] = (i < n) ? src[i] : 0;
}

// decompress setup: scan size table -> chunk pointers, output pointers, capacities
__global__ void __launch_bounds__(1024)
hlif_setup_decompress(const uint8_t* comp_buffer, size_t num_chunks, size_t chunk, size_t total_uncomp, uint8_t* out,
                      const void** comp_ptrs, size_t* comp_bytes, void** out_ptrs, size_t* out_caps) {
  __shared__ unsigned long long s_warp[32];
  __shared__ unsigned long long s_carry;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const unsigned long long* table = (const unsigned long long*)(comp_buffer + kHeaderBytes);
  const size_t payload0 = kHeaderBytes + 8 * num_chunks;
  for (size_t base = 0; base < num_chunks; base += blockDim.x) {
    const size_t i = base + threadIdx.x;
    const unsigned long long sz = (i < num_chunks) ? table[i] : 0ull;
    const unsigned long long al = (sz + 7ull) & ~7ull;
    unsigned long long incl = al;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long o = __shfl_up_sync(b200::kFull, incl, d);
      if (lane >= d) incl += o;
    }
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();
    unsigned long long wbase = 0;
    for (int k = 0; k < w; ++k) wbase += s_warp[k];
    const unsigned long long excl = s_carry + wbase + incl - al;
    if (i < num_chunks) {
      comp_ptrs[i] = comp_buffer + payload0 + excl;
      comp_bytes[i] = sz;
      out_ptrs[i] = out + i * chunk;
      out_caps[i] = (i + 1 < num_chunks) ? chunk : total_uncomp - i * chunk;
    }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = excl + al;
    __syncthreads();
  }
}

__global__ void hlif_store_checksums(uint8_t* comp_buffer, const uint32_t* sums) {
  HlifHeader* h = (HlifHeader*)comp_buffer;
  h->checksum_uncomp = sums[0];
  h->checksum_comp = sums[1];
}

__global__ void hlif_set_status(nvcompStatus_t* host_status, nvcompStatus_t v) { *host_status = v; }

// ------------------------------------------------------------------------------------------
struct ManagerImpl {
  FormatBinding fmt;
  size_t chunk;
  cudaStream_t stream;
  int device;
  ChecksumPolicy policy;
  uint8_t* scratch = nullptr;
  size_t scratch_bytes = 0;
  bool own_scratch = true;
  size_t required_scratch = 0;

  ManagerImpl(const FormatBinding& f, size_t chunk_size, cudaStream_t s, int dev, ChecksumPolicy p)
      : fmt(f), chunk(chunk_size), stream(s), device(dev), policy(p) {
    if (chunk_size == 0) throw NVCompException(nvcompErrorInvalidValue, "chunk size must be positive");
    if (chunk_size % fmt.chunk_multiple != 0)
      throw NVCompException(nvcompErrorInvalidValue, "chunk size must be a multiple of the format's required alignment");
    size_t probe = 0;
    check(fmt.comp_max(fmt, chunk, &probe), "invalid format options / chunk size");
  }
  ~ManagerImpl() { if (own_scratch && scratch) cudaFree(scratch); }

  bool computes() const { return policy == ComputeAndNoVerify || policy == ComputeAndVerifyIfPresent || policy == ComputeAndVerify; }
  bool verifies() const { return policy == NoComputeAndVerifyIfPresent || policy == ComputeAndVerifyIfPresent || policy == ComputeAndVerify; }

  struct Layout { size_t ptrs, sizes, outptrs, caps, actual, offsets, statuses, sums, crc, temp, temp_bytes, slab, total; };

  static size_t al(size_t x) { return (x + 255) & ~(size_t)255; }

  // crc_bytes: the longest buffer a checksum pass hashes with this layout (0 when no checksums are computed)
  Layout compress_layout(size_t n_chunks, size_t crc_bytes) const {
    Layout L{};
    size_t max_out = 0, temp = 0;
    check(fmt.comp_max(fmt, chunk, &max_out), "CompressGetMaxOutputChunkSize");
    check(fmt.comp_temp(fmt, n_chunks, chunk, &temp), "CompressGetTempSize");
    max_out = (max_out + 15) & ~(size_t)15;
    size_t off = 0;
    L.ptrs = off; off += al(8 * n_chunks);
    L.sizes = off; off += al(8 * n_chunks);
    L.outptrs = off; off += al(8 * n_chunks);
    L.caps = off; off += al(8 * n_chunks);       // compressed sizes
    L.offsets = off; off += al(8 * n_chunks);
    L.sums = off; off += 256;
    L.crc = off; off += al(4 * b200::crc_scratch_words(crc_bytes));
    L.temp = off; L.temp_bytes = temp; off += al(temp);
    L.slab = off; off += al(max_out * n_chunks);
    L.total = off;
    return L;
  }
  Layout decompress_layout(size_t n_chunks, size_t chunk_bytes, size_t crc_bytes) const {
    Layout L{};
    size_t temp = 0;
    check(fmt.decomp_temp(n_chunks, chunk_bytes, &temp), "DecompressGetTempSize");
    size_t off = 0;
    L.ptrs = off; off += al(8 * n_chunks);
    L.sizes = off; off += al(8 * n_chunks);
    L.outptrs = off; off += al(8 * n_chunks);
    L.caps = off; off += al(8 * n_chunks);
    L.actual = off; off += al(8 * n_chunks);
    L.statuses = off; off += al(4 * n_chunks);
    L.sums = off; off += 256;
    L.crc = off; off += al(4 * b200::crc_scratch_words(crc_bytes));
    L.temp = off; L.temp_bytes = temp; off += al(temp);
    L.total = off;
    return L;
  }

  void ensure_scratch(size_t bytes) {
    if (bytes > required_scratch) required_scratch = bytes;
    if (bytes <= scratch_bytes) return;
    if (!own_scratch) throw NVCompException(nvcompErrorInvalidValue, "user scratch buffer too small");
    check(cudaStreamSynchronize(stream), "sync before scratch growth");
    if (scratch) cudaFree(scratch);
    check(cudaMalloc(&scratch, bytes), "scratch allocation");
    scratch_bytes = bytes;
  }

  size_t n_chunks_of(size_t bytes) const { return bytes == 0 ? 0 : (bytes + chunk - 1) / chunk; }
  // longest span one checksum pass hashes for an (uncompressed, compressed-bound) pair under this policy
  size_t crc_span(size_t uncomp, size_t comp_bound) const {
    if (!computes() && !verifies()) return 0;
    return uncomp > comp_bound ? uncomp : comp_bound;
  }

  CompressionConfig configure_compression(size_t n) {
    CompressionConfig c;
    c.uncompressed_buffer_size = n;
    c.num_chunks = n_chunks_of(n);
    size_t max_out = 0;
    check(fmt.comp_max(fmt, chunk, &max_out), "CompressGetMaxOutputChunkSize");
    c.max_compressed_buffer_size = kHeaderBytes + 8 * c.num_chunks + c.num_chunks * ((max_out + 7) & ~(size_t)7) + 8;
    c.status = std::make_shared<StatusHolder>();
    const Layout L = compress_layout(c.num_chunks ? c.num_chunks : 1, crc_span(n, c.max_compressed_buffer_size));
    if (L.total > required_scratch) required_scratch = L.total;
    return c;
  }

  void compress(const uint8_t* in, uint8_t* out, const CompressionConfig& cfg) {
    check(cudaSetDevice(device), "cudaSetDevice");
    if (((uintptr_t)out & 7) != 0) throw NVCompException(nvcompErrorAlignment, "compressed buffer must be 8-byte aligned");
    const size_t n = cfg.uncompressed_buffer_size, nc = cfg.num_chunks;
    const Layout L = compress_layout(nc ? nc : 1, crc_span(n, cfg.max_compressed_buffer_size));
    ensure_scratch(L.total);
    HlifHeader h{};
    h.magic = kHlifMagic; h.format = fmt.format; std::memcpy(h.opts, fmt.opts, 24);
    h.uncompressed_bytes = n; h.chunk_bytes = chunk; h.num_chunks = (uint32_t)nc; h.flags = computes() ? 1u : 0u;
    size_t max_out = 0;
    check(fmt.comp_max(fmt, chunk, &max_out), "CompressGetMaxOutputChunkSize");
    max_out = (max_out + 15) & ~(size_t)15;
    const void** ptrs = (const void**)(scratch + L.ptrs);
    size_t* sizes = (size_t*)(scratch + L.sizes);
    void** outptrs = (void**)(scratch + L.outptrs);
    size_t* csizes = (size_t*)(scratch + L.caps);
    size_t* offsets = (size_t*)(scratch + L.offsets);
    uint32_t* sums = (uint32_t*)(scratch + L.sums);
    if (nc) {
      hlif_setup_compress<<<(unsigned)((nc + 255) / 256), 256, 0, stream>>>(in, n, chunk, nc, scratch + L.slab, max_out,
                                                                          ptrs, sizes, outptrs);
      check(fmt.comp(fmt, ptrs, sizes, chunk, nc, scratch + L.temp, L.temp_bytes, outptrs, csizes, stream), "CompressAsync");
    }
    hlif_layout<<<1, 1024, 0, stream>>>(csizes, nc, h, out, offsets);
    if (nc) hlif_gather<<<(unsigned)nc, 256, 0, stream>>>(outptrs, csizes, offsets, out);
    if (computes()) {
      uint32_t* crc_scratch = (uint32_t*)(scratch + L.crc);
      check(b200::crc32_buffer_async(in, n, nullptr, 0, n, crc_scratch, sums, stream), "uncompressed checksum");
      // the compressed payload (size table + every chunk) ends at header.total_bytes, which only the device knows:
      // the pass is sized for the bound and reads the length from the header just written (stays asynchronous)
      const unsigned long long* total_dev = (const unsigned long long*)(out + offsetof(HlifHeader, total_bytes));
      check(b200::crc32_buffer_async(out + kHeaderBytes, 0, total_dev, kHeaderBytes,
                                     cfg.max_compressed_buffer_size - kHeaderBytes, crc_scratch, sums + 1, stream),
            "compressed checksum");
      hlif_store_checksums<<<1, 1, 0, stream>>>(out, sums);
    }
    if (cfg.status && cfg.status->host) hlif_set_status<<<1, 1, 0, stream>>>(cfg.status->host, nvcompSuccess);
    check(cudaGetLastError(), "compress launch");
  }

  HlifHeader read_header(const uint8_t* comp) {
    HlifHeader h;
    check(cudaMemcpyAsync(&h, comp, sizeof(HlifHeader), cudaMemcpyDeviceToHost, stream), "header read");
    check(cudaStreamSynchronize(stream), "header sync");
    if (h.magic != kHlifMagic) throw NVCompException(nvcompErrorInvalidValue, "not a compressed buffer of this library");
    return h;
  }

  DecompressionConfig configure_decompression(const uint8_t* comp) {
    const HlifHeader h = read_header(comp);
    if (h.format != fmt.format) throw NVCompException(nvcompErrorInvalidValue, "buffer was compressed with another format");
    if (policy == ComputeAndVerify && !(h.flags & 1u))
      throw NVCompException(nvcompErrorCannotVerifyChecksums, "checksums requested but absent from the buffer");
    // the header is untrusted input: every field the pointer setup uses is checked against the others
    size_t probe = 0;
    if (h.chunk_bytes == 0 || h.chunk_bytes % fmt.chunk_multiple != 0 ||
        fmt.comp_max(fmt, (size_t)h.chunk_bytes, &probe) != nvcompSuccess)
      throw NVCompException(nvcompErrorInvalidValue, "corrupt header: chunk size");
    const uint64_t want_chunks = h.uncompressed_bytes == 0 ? 0 : (h.uncompressed_bytes + h.chunk_bytes - 1) / h.chunk_bytes;
    if ((uint64_t)h.num_chunks != want_chunks || h.total_bytes < kHeaderBytes + 8ull * h.num_chunks)
      throw NVCompException(nvcompErrorInvalidValue, "corrupt header: chunk count");
    check_size_table(comp, h);
    DecompressionConfig d;
    d.decomp_data_size = h.uncompressed_bytes;
    d.num_chunks = h.num_chunks;
    d.chunk_bytes = (size_t)h.chunk_bytes;
    d.comp_bytes_bound = (size_t)h.total_bytes;
    d.status = std::make_shared<StatusHolder>();
    const Layout L = decompress_layout(d.num_chunks ? d.num_chunks : 1, d.chunk_bytes,
                                       crc_span(d.decomp_data_size, d.comp_bytes_bound));
    if (L.total > required_scratch) required_scratch = L.total;
    return d;
  }

  // The size table is untrusted as well: every chunk pointer and the compressed-payload checksum pass are derived
  // from it, so every chunk must fit the format's bound and the chunks must end exactly at total_bytes.  The bound is
  // the one of the options stored in the header, which the chunks were written with: for Cascaded and Bitcomp it
  // depends on them, and this manager's own options only matter for compression (the decoders read the streams).
  void check_size_table(const uint8_t* comp, const HlifHeader& h) {
    FormatBinding stored = fmt;
    std::memcpy(stored.opts, h.opts, sizeof(stored.opts));
    size_t max_out = 0;
    if (stored.comp_max(stored, (size_t)h.chunk_bytes, &max_out) != nvcompSuccess)
      throw NVCompException(nvcompErrorInvalidValue, "corrupt header: format options");
    std::vector<uint64_t> sizes;
    try {
      sizes.resize(h.num_chunks);
    } catch (const std::bad_alloc&) {
      throw NVCompException(nvcompErrorInternal, "no host memory for the size table");
    }
    if (h.num_chunks) {
      check(cudaMemcpyAsync(sizes.data(), comp + kHeaderBytes, 8 * sizes.size(), cudaMemcpyDeviceToHost, stream),
            "size table read");
      check(cudaStreamSynchronize(stream), "size table sync");
    }
    uint64_t total = kHeaderBytes + 8ull * h.num_chunks;     // no overflow: num_chunks < 2^32, each size <= max_out
    for (const uint64_t s : sizes) {
      if (s > max_out) throw NVCompException(nvcompErrorInvalidValue, "corrupt size table: chunk above the format's bound");
      total += (s + 7) & ~7ull;
    }
    if (total != h.total_bytes)
      throw NVCompException(nvcompErrorInvalidValue, "corrupt size table: chunks do not end at total_bytes");
  }

  DecompressionConfig configure_decompression(const CompressionConfig& c) {
    DecompressionConfig d;
    d.decomp_data_size = c.uncompressed_buffer_size;
    d.num_chunks = (uint32_t)c.num_chunks;
    d.chunk_bytes = chunk;
    d.comp_bytes_bound = c.max_compressed_buffer_size;
    d.status = std::make_shared<StatusHolder>();
    return d;
  }

  void decompress(uint8_t* out, const uint8_t* comp, const DecompressionConfig& cfg) {
    check(cudaSetDevice(device), "cudaSetDevice");
    const size_t nc = cfg.num_chunks;
    const Layout L = decompress_layout(nc ? nc : 1, cfg.chunk_bytes, crc_span(cfg.decomp_data_size, cfg.comp_bytes_bound));
    ensure_scratch(L.total);
    const void** ptrs = (const void**)(scratch + L.ptrs);
    size_t* sizes = (size_t*)(scratch + L.sizes);
    void** outptrs = (void**)(scratch + L.outptrs);
    size_t* caps = (size_t*)(scratch + L.caps);
    size_t* actual = (size_t*)(scratch + L.actual);
    nvcompStatus_t* statuses = (nvcompStatus_t*)(scratch + L.statuses);
    uint32_t* sums = (uint32_t*)(scratch + L.sums);
    if (nc) {
      hlif_setup_decompress<<<1, 1024, 0, stream>>>(comp, nc, cfg.chunk_bytes, cfg.decomp_data_size, out, ptrs, sizes, outptrs, caps);
      check(fmt.decomp(ptrs, sizes, caps, actual, nc, scratch + L.temp, L.temp_bytes, outptrs, statuses, stream),
            "DecompressAsync");
    }
    int verify = 0;
    if (verifies()) {
      // verification is decided on the device from the header flag (no host sync here)
      uint32_t* crc_scratch = (uint32_t*)(scratch + L.crc);
      check(b200::crc32_buffer_async(out, cfg.decomp_data_size, nullptr, 0, cfg.decomp_data_size, crc_scratch, sums, stream),
            "uncompressed checksum");
      const unsigned long long* total_dev = (const unsigned long long*)(comp + offsetof(HlifHeader, total_bytes));
      const size_t bound = cfg.comp_bytes_bound > kHeaderBytes ? cfg.comp_bytes_bound - kHeaderBytes : 0;
      check(b200::crc32_buffer_async(comp + kHeaderBytes, 0, total_dev, kHeaderBytes, bound, crc_scratch, sums + 1, stream),
            "compressed checksum");
      verify = 1;
    }
    if (cfg.status && cfg.status->host)
      hlif_reduce_status_launch(statuses, actual, caps, nc, comp, sums, verify, cfg.status->host);
    check(cudaGetLastError(), "decompress launch");
  }

  void hlif_reduce_status_launch(const nvcompStatus_t* statuses, const size_t* actual, const size_t* caps, size_t nc,
                                 const uint8_t* comp, const uint32_t* sums, int verify, nvcompStatus_t* host);

  size_t get_compressed_output_size(const uint8_t* comp) { return read_header(comp).total_bytes; }
};

// a chunk fails unless it decodes to exactly its slot (a valid stream may decode to fewer bytes than the capacity);
// verification only applies when the buffer carries checksums (flag read on the device)
__global__ void hlif_reduce_status_flagged(const nvcompStatus_t* statuses, const size_t* actual, const size_t* caps,
                                           size_t num_chunks, const uint8_t* comp_buffer, const uint32_t* sums,
                                           int verify, nvcompStatus_t* host_status) {
  __shared__ int s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  for (size_t i = threadIdx.x; i < num_chunks; i += blockDim.x)
    if (statuses[i] != nvcompSuccess || actual[i] != caps[i]) s_bad = 1;
  __syncthreads();
  if (threadIdx.x == 0) {
    nvcompStatus_t st = s_bad ? nvcompErrorCannotDecompress : nvcompSuccess;
    const HlifHeader* h = (const HlifHeader*)comp_buffer;
    if (st == nvcompSuccess && verify && (h->flags & 1u)) {
      if (h->checksum_uncomp != sums[0] || h->checksum_comp != sums[1]) st = nvcompErrorBadChecksum;
    }
    *host_status = st;
  }
}

void ManagerImpl::hlif_reduce_status_launch(const nvcompStatus_t* statuses, const size_t* actual, const size_t* caps,
                                            size_t nc, const uint8_t* comp, const uint32_t* sums, int verify,
                                            nvcompStatus_t* host) {
  hlif_reduce_status_flagged<<<1, 256, 0, stream>>>(statuses, actual, caps, nc, comp, sums, verify, host);
}

}  // namespace detail

// ------------------------------------------------------------------------------------------
nvcompStatus_t* CompressionConfig::get_status() const { return status ? status->host : nullptr; }
nvcompStatus_t* DecompressionConfig::get_status() const { return status ? status->host : nullptr; }

PimplManager::PimplManager() = default;
PimplManager::~PimplManager() = default;
CompressionConfig PimplManager::configure_compression(const size_t n) { return impl->configure_compression(n); }
void PimplManager::compress(const uint8_t* in, uint8_t* out, const CompressionConfig& c) { impl->compress(in, out, c); }
DecompressionConfig PimplManager::configure_decompression(const uint8_t* comp) { return impl->configure_decompression(comp); }
DecompressionConfig PimplManager::configure_decompression(const CompressionConfig& c) { return impl->configure_decompression(c); }
void PimplManager::decompress(uint8_t* out, const uint8_t* comp, const DecompressionConfig& c) { impl->decompress(out, comp, c); }
size_t PimplManager::get_compressed_output_size(uint8_t* comp) { return impl->get_compressed_output_size(comp); }
size_t PimplManager::get_required_scratch_buffer_size() { return impl->required_scratch; }
void PimplManager::set_scratch_buffer(uint8_t* p) {
  if (impl->own_scratch && impl->scratch) cudaFree(impl->scratch);
  impl->scratch = p; impl->own_scratch = false; impl->scratch_bytes = impl->required_scratch;
}

#define B200_MANAGER(FMT, OPTS)                                                                                   \
  FMT##Manager::FMT##Manager(size_t chunk, const OPTS& o, cudaStream_t s, const int dev, ChecksumPolicy p) {      \
    impl.reset(new detail::ManagerImpl(detail::bind_##FMT(o), chunk, s, dev, p));                                 \
  }                                                                                                               \
  FMT##Manager::~FMT##Manager() = default;

B200_MANAGER(LZ4, nvcompBatchedLZ4Opts_t)
B200_MANAGER(Snappy, nvcompBatchedSnappyOpts_t)
B200_MANAGER(Cascaded, nvcompBatchedCascadedOpts_t)
B200_MANAGER(Bitcomp, nvcompBatchedBitcompFormatOpts)
B200_MANAGER(ANS, nvcompBatchedANSOpts_t)
B200_MANAGER(Deflate, nvcompBatchedDeflateOpts_t)

#define B200_UNSUPPORTED_MANAGER(FMT)                                                                             \
  FMT##Manager::FMT##Manager(size_t, const nvcompBatched##FMT##Opts_t&, cudaStream_t, const int, ChecksumPolicy) { \
    throw NVCompException(nvcompErrorNotSupported, #FMT " is out of scope for this library");                      \
  }                                                                                                               \
  FMT##Manager::~FMT##Manager() = default;

B200_UNSUPPORTED_MANAGER(Gdeflate)
B200_UNSUPPORTED_MANAGER(Zstd)

std::shared_ptr<nvcompManagerBase> create_manager(const uint8_t* comp_buffer, cudaStream_t stream, const int device_id,
                                                  ChecksumPolicy policy) {
  detail::HlifHeader h;
  detail::check(cudaSetDevice(device_id), "cudaSetDevice");
  detail::check(cudaMemcpyAsync(&h, comp_buffer, sizeof(h), cudaMemcpyDeviceToHost, stream), "header read");
  detail::check(cudaStreamSynchronize(stream), "header sync");
  if (h.magic != detail::kHlifMagic) throw NVCompException(nvcompErrorInvalidValue, "not a compressed buffer of this library");
  switch (h.format) {
    case detail::kFmtLZ4: { nvcompBatchedLZ4Opts_t o; std::memcpy(&o, h.opts, sizeof(o));
      return std::make_shared<LZ4Manager>(h.chunk_bytes, o, stream, device_id, policy); }
    case detail::kFmtSnappy: { nvcompBatchedSnappyOpts_t o; std::memcpy(&o, h.opts, sizeof(o));
      return std::make_shared<SnappyManager>(h.chunk_bytes, o, stream, device_id, policy); }
    case detail::kFmtCascaded: { nvcompBatchedCascadedOpts_t o; std::memcpy(&o, h.opts, sizeof(o));
      return std::make_shared<CascadedManager>(h.chunk_bytes, o, stream, device_id, policy); }
    case detail::kFmtBitcomp: { nvcompBatchedBitcompFormatOpts o; std::memcpy(&o, h.opts, sizeof(o));
      return std::make_shared<BitcompManager>(h.chunk_bytes, o, stream, device_id, policy); }
    case detail::kFmtANS: { nvcompBatchedANSOpts_t o; std::memcpy(&o, h.opts, sizeof(o));
      return std::make_shared<ANSManager>(h.chunk_bytes, o, stream, device_id, policy); }
    case detail::kFmtDeflate: { nvcompBatchedDeflateOpts_t o; std::memcpy(&o, h.opts, sizeof(o));
      return std::make_shared<DeflateManager>(h.chunk_bytes, o, stream, device_id, policy); }
    default: throw NVCompException(nvcompErrorInvalidValue, "unknown format id in compressed buffer");
  }
}

}  // namespace nvcomp

// ------------------------------------------------------------------------------------------
// Out-of-scope formats: LLIF symbols that report nvcompErrorNotSupported (see include/nvcomp/gdeflate.h).  Deflate
// and Gzip live in deflate.cu; Zstd decompression lives in zstd.cu, Zstd compression is not provided.
// ------------------------------------------------------------------------------------------
#define B200_UNSUPPORTED_COMPRESS(FMT)                                                                           \
  extern "C" {                                                                                                   \
  nvcompStatus_t nvcompBatched##FMT##CompressGetTempSize(size_t, size_t, nvcompBatched##FMT##Opts_t, size_t*) {   \
    return nvcompErrorNotSupported; }                                                                            \
  nvcompStatus_t nvcompBatched##FMT##CompressGetMaxOutputChunkSize(size_t, nvcompBatched##FMT##Opts_t, size_t*) { \
    return nvcompErrorNotSupported; }                                                                            \
  nvcompStatus_t nvcompBatched##FMT##CompressAsync(const void* const*, const size_t*, size_t, size_t, void*, size_t, \
      void* const*, size_t*, nvcompBatched##FMT##Opts_t, cudaStream_t) { return nvcompErrorNotSupported; }        \
  }
#define B200_UNSUPPORTED_LLIF(FMT)                                                                               \
  B200_UNSUPPORTED_COMPRESS(FMT)                                                                                 \
  extern "C" {                                                                                                   \
  nvcompStatus_t nvcompBatched##FMT##DecompressGetTempSize(size_t, size_t, size_t*) { return nvcompErrorNotSupported; } \
  nvcompStatus_t nvcompBatched##FMT##GetDecompressSizeAsync(const void* const*, const size_t*, size_t*, size_t,    \
      cudaStream_t) { return nvcompErrorNotSupported; }                                                          \
  nvcompStatus_t nvcompBatched##FMT##DecompressAsync(const void* const*, const size_t*, const size_t*, size_t*, size_t, \
      void* const, size_t, void* const*, nvcompStatus_t*, cudaStream_t) { return nvcompErrorNotSupported; }        \
  }

B200_UNSUPPORTED_LLIF(Gdeflate)
B200_UNSUPPORTED_COMPRESS(Zstd)
