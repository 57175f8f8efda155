// lz77_compress.cuh -- warp-per-chunk LZ77 matcher shared by the LZ4, Snappy and Deflate batched compressors.  It lives
// in nvcomp/device/detail/lz77_compress.cuh, shared with the device API of nvcomp/device/lz4.cuh and snappy.cuh; this
// file re-exports its names into namespace b200.
#pragma once

#include "common.cuh"
#include "nvcomp/device/detail/lz77_compress.cuh"

namespace b200 {

using nvcomp::device::lz::detail::kHashLog;
using nvcomp::device::lz::detail::kHashEntries;
using nvcomp::device::lz::detail::kHashBytesPerWarp;
using nvcomp::device::lz::detail::hash4;
using nvcomp::device::lz::detail::LzParams;
using nvcomp::device::lz::detail::det_insert;
using nvcomp::device::lz::detail::lz_extend;
using nvcomp::device::lz::detail::lz77_compress_chunk;

}  // namespace b200
