/*
 * nvcomp/nvcompManager.hpp -- high-level interface (HLIF): one contiguous device buffer in,
 * one self-describing compressed buffer out.  Surface pinned by the reference call sites:
 *   configure_compression / compress / configure_decompression / decompress /
 *   get_compressed_output_size            (doc/highlevel_cpp_quickstart.md:84-149,
 *                                          benchmarks/benchmark_hlif.hpp:68-137)
 *   CompressionConfig::max_compressed_buffer_size, DecompressionConfig::decomp_data_size,
 *   DecompressionConfig::get_status()     (examples/high_level_quickstart_example.cpp:79,92,313)
 *   ChecksumPolicy enumerators            (examples/high_level_quickstart_example.cpp:256-281)
 *   configs stored in std::vector         (benchmarks/benchmark_allgather.cpp:311-328)
 * Since 3.0.0 the HLIF dispatches to the low-level batched API (CHANGELOG.md:17); so does
 * this one: chunk the buffer, call nvcompBatched<Fmt>{Compress,Decompress}Async, compact
 * the chunks behind a header + size table (nvcomp_b200/csrc/hlif.cu).
 */
#ifndef NVCOMP_MANAGER_HPP
#define NVCOMP_MANAGER_HPP

#include "../nvcomp.hpp"

#include <cstddef>
#include <cstdint>
#include <memory>

namespace nvcomp
{

enum ChecksumPolicy
{
  /* no checksums computed on compression, none verified on decompression */
  NoComputeNoVerify = 0,
  /* computed and stored on compression, not verified on decompression */
  ComputeAndNoVerify = 1,
  /* not computed on compression, verified on decompression if the buffer carries them */
  NoComputeAndVerifyIfPresent = 2,
  /* computed on compression, verified on decompression if present */
  ComputeAndVerifyIfPresent = 3,
  /* computed on compression, verified on decompression; configure_decompression throws if absent */
  ComputeAndVerify = 4
};

namespace detail { struct StatusHolder; struct ManagerImpl; struct FormatBinding; }

struct CompressionConfig
{
  size_t uncompressed_buffer_size;
  size_t max_compressed_buffer_size;
  size_t num_chunks;
  /* pinned host status of the last compress() issued with this config; valid after a stream sync */
  nvcompStatus_t* get_status() const;
  std::shared_ptr<detail::StatusHolder> status;
};

struct DecompressionConfig
{
  size_t decomp_data_size;
  uint32_t num_chunks;
  /* uncompressed bytes per chunk of the buffer this config describes (from its header, validated) */
  size_t chunk_bytes;
  /* upper bound of the compressed buffer's size (header total, or the compression config's bound): sizes the
   * checksum pass over the compressed payload */
  size_t comp_bytes_bound;
  /* pinned host status of the last decompress() issued with this config; valid after a stream sync.
   * nvcompSuccess: every chunk decoded to exactly its slot of the output (and, when verified, both checksums match);
   * nvcompErrorCannotDecompress: some chunk failed to decode or decoded to fewer or more bytes than its slot;
   * nvcompErrorBadChecksum: every chunk decoded but a stored checksum disagrees */
  nvcompStatus_t* get_status() const;
  std::shared_ptr<detail::StatusHolder> status;
};

struct nvcompManagerBase
{
  virtual CompressionConfig configure_compression(const size_t decomp_buffer_size) = 0;
  virtual void compress(const uint8_t* decomp_buffer, uint8_t* comp_buffer, const CompressionConfig& comp_config) = 0;
  /* reads the header of comp_buffer: synchronises the stream */
  virtual DecompressionConfig configure_decompression(const uint8_t* comp_buffer) = 0;
  virtual DecompressionConfig configure_decompression(const CompressionConfig& comp_config) = 0;
  virtual void decompress(uint8_t* decomp_buffer, const uint8_t* comp_buffer, const DecompressionConfig& decomp_config) = 0;
  /* total bytes of the compressed buffer (header + table + chunks): synchronises the stream */
  virtual size_t get_compressed_output_size(uint8_t* comp_buffer) = 0;
  /* scratch the manager needs for the largest configure_* issued so far */
  virtual size_t get_required_scratch_buffer_size() = 0;
  /* let the caller own the scratch (otherwise the manager allocates and grows its own) */
  virtual void set_scratch_buffer(uint8_t* new_scratch_buffer) = 0;
  virtual ~nvcompManagerBase() = default;
};

/* Common implementation: every format manager forwards to detail::ManagerImpl. */
struct PimplManager : nvcompManagerBase
{
  PimplManager();
  ~PimplManager() override;
  PimplManager(const PimplManager&) = delete;
  PimplManager& operator=(const PimplManager&) = delete;

  CompressionConfig configure_compression(const size_t decomp_buffer_size) override;
  void compress(const uint8_t* decomp_buffer, uint8_t* comp_buffer, const CompressionConfig& comp_config) override;
  DecompressionConfig configure_decompression(const uint8_t* comp_buffer) override;
  DecompressionConfig configure_decompression(const CompressionConfig& comp_config) override;
  void decompress(uint8_t* decomp_buffer, const uint8_t* comp_buffer, const DecompressionConfig& decomp_config) override;
  size_t get_compressed_output_size(uint8_t* comp_buffer) override;
  size_t get_required_scratch_buffer_size() override;
  void set_scratch_buffer(uint8_t* new_scratch_buffer) override;

protected:
  std::unique_ptr<detail::ManagerImpl> impl;
};

} // namespace nvcomp

#endif
