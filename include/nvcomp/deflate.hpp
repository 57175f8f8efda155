/*
 * nvcomp/deflate.hpp -- DeflateManager: the high-level interface over the batched Deflate codec (deflate.h).  An
 * algo outside 0..2 throws NVCompException(nvcompErrorInvalidValue).
 */
#ifndef NVCOMP_DEFLATE_HPP
#define NVCOMP_DEFLATE_HPP

#include "nvcompManager.hpp"
#include "deflate.h"

namespace nvcomp
{

struct DeflateManager : PimplManager
{
  DeflateManager(
      size_t uncomp_chunk_size,
      const nvcompBatchedDeflateOpts_t& format_opts,
      cudaStream_t user_stream = 0,
      const int device_id = 0,
      ChecksumPolicy checksum_policy = NoComputeNoVerify);
  ~DeflateManager() override;
};

} // namespace nvcomp

#endif
