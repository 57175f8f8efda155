// nvcomp/device/detail/lz_region.cuh -- one LZ4 / Snappy chunk decoded in a caller's per-warp shared-memory region:
// the routing and the mbarrier lifecycle that nvcomp/device/lz4.cuh and snappy.cuh share.
#pragma once

#include "nvcomp/shared_types.h"
#include "nvcomp/device/detail/lz_decode.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

// Decode one chunk with the body the batched call runs for it: light(&produced) -- the direct loop -- when
// lz_chunk_is_light(capacity, comp_bytes), the batched classifier's rule, else dense(&produced, ring, parity) -- the
// block-parallel decoder.  The batched dense kernel initializes its warps' mbarriers once and carries the phase from
// chunk to chunk; here the caller owns the region between calls, and PTX makes mbarrier.init on a live mbarrier, or
// reusing the memory of a valid one, undefined.  So lane 0 initializes the region's mbarrier on entry (parity 0), and
// after the decode -- which leaves no bulk copy in flight on any return: lz_decode_stream waits for a prefetched block,
// the direct loop issues none -- a __syncwarp puts every lane past its last wait before lane 0 invalidates the
// barrier.  The closing __syncwarp hands the region back to the caller.
template <class Light, class Dense>
__device__ __forceinline__ nvcompStatus_t lz_decompress_in_region(size_t comp_bytes, size_t capacity, size_t* actual,
                                                                  void* smem, const Light& light, const Dense& dense) {
  const int lane = lane_id();
  uint8_t* ring = (uint8_t*)smem;
  const uint32_t ra = smem_addr(ring);
  lz_warp_init(ra, lane);
  uint32_t parity = 0;
  uint32_t produced = 0;
  bool ok = comp_bytes <= 0xffffffffull;
  if (ok) ok = lz_chunk_is_light((uint64_t)capacity, (uint64_t)comp_bytes) ? light(&produced)
                                                                           : dense(&produced, ring, parity);
  __syncwarp();
  if (lane == 0) {
    mbar_inval(ra + kSmemMbar);
    if (actual) *actual = ok ? (size_t)produced : 0;
  }
  __syncwarp();
  return ok ? nvcompSuccess : nvcompErrorCannotDecompress;
}

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
