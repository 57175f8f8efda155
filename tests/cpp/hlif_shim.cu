// hlif_shim.cu -- extern "C" dispatch onto the C++ high-level interface (nvcomp::*Manager, create_manager), so that
// tests/test_hlif_oracle_gpu.py can drive the managers with ctypes on torch-owned device memory.  Built by `make` into
// build/tests/libhlif_shim.so.  Every entry point returns an nvcompStatus_t: the error of an NVCompException, or
// nvcompErrorInternal for any other exception; nothing throws across the C boundary.  Managers and configs are heap
// objects owned by the caller through opaque handles.
#include <cstring>
#include <memory>

#include "nvcomp.hpp"
#include "nvcomp/nvcompManagerFactory.hpp"

using namespace nvcomp;

using Mgr = std::shared_ptr<nvcompManagerBase>;

template <class F>
static int guard(F&& f) {
  try {
    f();
    return nvcompSuccess;
  } catch (const NVCompException& e) {
    return e.get_error();
  } catch (...) {
    return nvcompErrorInternal;
  }
}

template <class Opts>
static Opts opts_from(const void* blob) {
  Opts o;
  std::memcpy(&o, blob, sizeof(Opts));
  return o;
}

extern "C" {

// format ids as stored in the container header: LZ4 1, Snappy 2, Cascaded 3, Bitcomp 4, ANS 5, Deflate 6
int hlif_shim_create(unsigned format, const void* opts24, size_t chunk, int policy, void* stream, int device,
                     void** out) {
  return guard([&] {
    const cudaStream_t s = (cudaStream_t)stream;
    const ChecksumPolicy p = (ChecksumPolicy)policy;
    Mgr m;
    switch (format) {
      case 1: m = std::make_shared<LZ4Manager>(chunk, opts_from<nvcompBatchedLZ4Opts_t>(opts24), s, device, p); break;
      case 2: m = std::make_shared<SnappyManager>(chunk, opts_from<nvcompBatchedSnappyOpts_t>(opts24), s, device, p); break;
      case 3: m = std::make_shared<CascadedManager>(chunk, opts_from<nvcompBatchedCascadedOpts_t>(opts24), s, device, p); break;
      case 4: m = std::make_shared<BitcompManager>(chunk, opts_from<nvcompBatchedBitcompFormatOpts>(opts24), s, device, p); break;
      case 5: m = std::make_shared<ANSManager>(chunk, opts_from<nvcompBatchedANSOpts_t>(opts24), s, device, p); break;
      case 6: m = std::make_shared<DeflateManager>(chunk, opts_from<nvcompBatchedDeflateOpts_t>(opts24), s, device, p); break;
      default: throw NVCompException(nvcompErrorInvalidValue, "unknown format id");
    }
    *out = new Mgr(std::move(m));
  });
}

int hlif_shim_create_from(const void* comp, void* stream, int device, int policy, void** out) {
  return guard([&] {
    *out = new Mgr(create_manager((const uint8_t*)comp, (cudaStream_t)stream, device, (ChecksumPolicy)policy));
  });
}

void hlif_shim_destroy(void* mgr) { delete (Mgr*)mgr; }

int hlif_shim_configure_compression(void* mgr, size_t n, void** cfg, size_t* max_comp, size_t* num_chunks) {
  return guard([&] {
    auto* c = new CompressionConfig((*(Mgr*)mgr)->configure_compression(n));
    *cfg = c;
    *max_comp = c->max_compressed_buffer_size;
    *num_chunks = c->num_chunks;
  });
}

void hlif_shim_free_compression_config(void* cfg) { delete (CompressionConfig*)cfg; }

int hlif_shim_compress(void* mgr, const void* in, void* out, void* cfg) {
  return guard([&] { (*(Mgr*)mgr)->compress((const uint8_t*)in, (uint8_t*)out, *(CompressionConfig*)cfg); });
}

// the status of the last call issued with the config; the caller synchronizes the stream first
int hlif_shim_compression_status(void* cfg) { return *((CompressionConfig*)cfg)->get_status(); }

static void describe(const DecompressionConfig& d, size_t* decomp_size, size_t* num_chunks) {
  *decomp_size = d.decomp_data_size;
  *num_chunks = d.num_chunks;
}

int hlif_shim_configure_decompression(void* mgr, const void* comp, void** cfg, size_t* decomp_size, size_t* num_chunks) {
  return guard([&] {
    auto* d = new DecompressionConfig((*(Mgr*)mgr)->configure_decompression((const uint8_t*)comp));
    *cfg = d;
    describe(*d, decomp_size, num_chunks);
  });
}

int hlif_shim_configure_decompression_cc(void* mgr, void* ccfg, void** cfg, size_t* decomp_size, size_t* num_chunks) {
  return guard([&] {
    auto* d = new DecompressionConfig((*(Mgr*)mgr)->configure_decompression(*(CompressionConfig*)ccfg));
    *cfg = d;
    describe(*d, decomp_size, num_chunks);
  });
}

void hlif_shim_free_decompression_config(void* cfg) { delete (DecompressionConfig*)cfg; }

int hlif_shim_decompress(void* mgr, void* out, const void* comp, void* cfg) {
  return guard([&] { (*(Mgr*)mgr)->decompress((uint8_t*)out, (const uint8_t*)comp, *(DecompressionConfig*)cfg); });
}

int hlif_shim_decompression_status(void* cfg) { return *((DecompressionConfig*)cfg)->get_status(); }

int hlif_shim_compressed_output_size(void* mgr, void* comp, size_t* out) {
  return guard([&] { *out = (*(Mgr*)mgr)->get_compressed_output_size((uint8_t*)comp); });
}

int hlif_shim_required_scratch(void* mgr, size_t* out) {
  return guard([&] { *out = (*(Mgr*)mgr)->get_required_scratch_buffer_size(); });
}

int hlif_shim_set_scratch(void* mgr, void* scratch) {
  return guard([&] { (*(Mgr*)mgr)->set_scratch_buffer((uint8_t*)scratch); });
}

}  // extern "C"
