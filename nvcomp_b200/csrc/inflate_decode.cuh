// inflate_decode.cuh -- Deflate (RFC 1951) and Gzip (RFC 1952) decode of one chunk by one warp.  It lives in
// nvcomp/device/detail/inflate_decode.cuh, shared with the device API of nvcomp/device/deflate.cuh and gzip.cuh; this
// file re-exports its names into namespace b200.
#pragma once

#include "common.cuh"
#include "crc32.cuh"
#include "nvcomp/device/detail/inflate_decode.cuh"

namespace b200 {

using nvcomp::device::deflate::detail::InflateResult;
using nvcomp::device::deflate::detail::kInflateOk;
using nvcomp::device::deflate::detail::kInflateBad;
using nvcomp::device::deflate::detail::kInflateBadChecksum;
using nvcomp::device::deflate::detail::kInfLitRoot;
using nvcomp::device::deflate::detail::kInfDistRoot;
using nvcomp::device::deflate::detail::kInfClenRoot;
using nvcomp::device::deflate::detail::kInfLitEntries;
using nvcomp::device::deflate::detail::kInfDistEntries;
using nvcomp::device::deflate::detail::kInfClenEntries;
using nvcomp::device::deflate::detail::kInfFixLitEntries;
using nvcomp::device::deflate::detail::kInfFixDistEntries;
using nvcomp::device::deflate::detail::kInfLitOff;
using nvcomp::device::deflate::detail::kInfDistOff;
using nvcomp::device::deflate::detail::kInfFixLitOff;
using nvcomp::device::deflate::detail::kInfFixDistOff;
using nvcomp::device::deflate::detail::kInfClenOff;
using nvcomp::device::deflate::detail::kInfRankOff;
using nvcomp::device::deflate::detail::kInfLensOff;
using nvcomp::device::deflate::detail::kInfWarpSmem;
using nvcomp::device::deflate::detail::InflateWarp;
using nvcomp::device::deflate::detail::InfBits;
using nvcomp::device::deflate::detail::inf_scan_excl;
using nvcomp::device::deflate::detail::inf_brev;
using nvcomp::device::deflate::detail::inflate_build_table;
using nvcomp::device::deflate::detail::inf_lookup;
using nvcomp::device::deflate::detail::inf_clen_order;
using nvcomp::device::deflate::detail::inflate_build_fixed;
using nvcomp::device::deflate::detail::inflate_read_dynamic;
using nvcomp::device::deflate::detail::inflate_huffman_block;
using nvcomp::device::deflate::detail::inflate_stream;
using nvcomp::device::deflate::detail::inf_skip_zstring;
using nvcomp::device::deflate::detail::inf_le32;
using nvcomp::device::deflate::detail::inflate_chunk;

}  // namespace b200
