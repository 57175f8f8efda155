// lz4_decode.cuh -- LZ4 block-format decode for one chunk owned by one warp.  It lives in
// nvcomp/device/detail/lz4_decode.cuh, shared with the device API of nvcomp/device/lz4.cuh; this file re-exports its
// names into namespace b200.  Kernels and the C ABI are in lz4.cu.
#pragma once

#include "common.cuh"
#include "lz_decode.cuh"
#include "nvcomp/device/detail/lz4_decode.cuh"

namespace b200 {

using nvcomp::device::lz::detail::lz4_read_ext;
using nvcomp::device::lz::detail::lz4_walk_chunk;
using nvcomp::device::lz::detail::lz4_decode_chunk_direct;
using nvcomp::device::lz::detail::Lz4Decode;
using nvcomp::device::lz::detail::lz4_decode_chunk_v2;

}  // namespace b200
