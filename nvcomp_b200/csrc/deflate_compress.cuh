// deflate_compress.cuh -- warp-per-chunk Deflate (RFC 1951) encoder behind nvcompBatchedDeflateCompressAsync.  It
// lives in nvcomp/device/detail/deflate_compress.cuh, shared with the device API of nvcomp/device/deflate.cuh; this
// file re-exports its names into namespace b200.
#pragma once

#include "common.cuh"
#include "lz77_compress.cuh"
#include "nvcomp/device/detail/deflate_compress.cuh"

namespace b200 {

using nvcomp::device::deflate::detail::kDeflateLitSyms;
using nvcomp::device::deflate::detail::kDeflateDistSyms;
using nvcomp::device::deflate::detail::kDeflateClenSyms;
using nvcomp::device::deflate::detail::kDeflateDistBase;
using nvcomp::device::deflate::detail::kDeflateClenBase;
using nvcomp::device::deflate::detail::kDeflateSymWords;
using nvcomp::device::deflate::detail::kDeflateStageWords;
using nvcomp::device::deflate::detail::kDeflateFlushBits;
using nvcomp::device::deflate::detail::kDeflateMaxChunk;
using nvcomp::device::deflate::detail::kStoredMax;
using nvcomp::device::deflate::detail::kPmFlagWords;
using nvcomp::device::deflate::detail::kPmWords;
using nvcomp::device::deflate::detail::DeflateAlgo;
using nvcomp::device::deflate::detail::kDeflateWarpSmem;
using nvcomp::device::deflate::detail::DeflateWarp;
using nvcomp::device::deflate::detail::deflate_len_code;
using nvcomp::device::deflate::detail::deflate_dist_code;
using nvcomp::device::deflate::detail::deflate_len_extra;
using nvcomp::device::deflate::detail::deflate_dist_extra;
using nvcomp::device::deflate::detail::deflate_fixed_lit_len;
using nvcomp::device::deflate::detail::DeflateHist;
using nvcomp::device::deflate::detail::DeflateBits;
using nvcomp::device::deflate::detail::pm_lengths;
using nvcomp::device::deflate::detail::canonical_codes;
using nvcomp::device::deflate::detail::rle_lengths;
using nvcomp::device::deflate::detail::deflate_parse;
using nvcomp::device::deflate::detail::deflate_compress_chunk;

}  // namespace b200
