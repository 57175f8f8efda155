// xxhash64.cuh -- XXH64 (seed 0) of a span of global memory by one warp, the Zstandard content checksum.  It lives in
// nvcomp/device/detail/xxhash64.cuh, shared with the device API of nvcomp/device/zstd.cuh; this file re-exports its
// names into namespace b200.
#pragma once

#include "common.cuh"
#include "nvcomp/device/detail/xxhash64.cuh"

namespace b200 {

using nvcomp::device::zstd::detail::kXxP1;
using nvcomp::device::zstd::detail::kXxP2;
using nvcomp::device::zstd::detail::kXxP3;
using nvcomp::device::zstd::detail::kXxP4;
using nvcomp::device::zstd::detail::kXxP5;
using nvcomp::device::zstd::detail::xx_rotl;
using nvcomp::device::zstd::detail::xx_round;
using nvcomp::device::zstd::detail::xx_merge;
using nvcomp::device::zstd::detail::xx_le32;
using nvcomp::device::zstd::detail::xx_le64;
using nvcomp::device::zstd::detail::xxh64_warp;

}  // namespace b200
