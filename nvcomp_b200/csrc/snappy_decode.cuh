// snappy_decode.cuh -- Snappy raw-format decode for one chunk owned by one warp.  It lives in
// nvcomp/device/detail/snappy_decode.cuh, shared with the device API of nvcomp/device/snappy.cuh; this file re-exports
// its names into namespace b200.  Kernels and the C ABI are in snappy.cu.
#pragma once

#include "common.cuh"
#include "lz_decode.cuh"
#include "nvcomp/device/detail/snappy_decode.cuh"

namespace b200 {

using nvcomp::device::lz::detail::snappy_read_preamble;
using nvcomp::device::lz::detail::kRlWindow;
using nvcomp::device::lz::detail::kRlNone;
using nvcomp::device::lz::detail::rl_nibbles;
using nvcomp::device::lz::detail::rl_const_mask;
using nvcomp::device::lz::detail::RlMap;
using nvcomp::device::lz::detail::rl_perm;
using nvcomp::device::lz::detail::rl_window;
using nvcomp::device::lz::detail::rl_lookup;
using nvcomp::device::lz::detail::rl_reload;
using nvcomp::device::lz::detail::snappy_decode_chunk;
using nvcomp::device::lz::detail::SnappyDecode;
using nvcomp::device::lz::detail::snappy_decode_chunk_v2;

}  // namespace b200
