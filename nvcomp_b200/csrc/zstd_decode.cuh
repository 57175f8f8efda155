// zstd_decode.cuh -- Zstandard (RFC 8878) decode of one chunk by one warp.  It lives in
// nvcomp/device/detail/zstd_decode.cuh, shared with the device API of nvcomp/device/zstd.cuh; this file re-exports its
// names into namespace b200.
#pragma once

#include "common.cuh"
#include "xxhash64.cuh"
#include "nvcomp/device/detail/zstd_decode.cuh"

namespace b200 {

using nvcomp::device::zstd::detail::ZstdResult;
using nvcomp::device::zstd::detail::kZstdOk;
using nvcomp::device::zstd::detail::kZstdBad;
using nvcomp::device::zstd::detail::kZstdBadChecksum;
using nvcomp::device::zstd::detail::kZsBlockMax;
using nvcomp::device::zstd::detail::kZsHufMaxLog;
using nvcomp::device::zstd::detail::kZsHufOff;
using nvcomp::device::zstd::detail::kZsLLOff;
using nvcomp::device::zstd::detail::kZsOFOff;
using nvcomp::device::zstd::detail::kZsMLOff;
using nvcomp::device::zstd::detail::kZsWtOff;
using nvcomp::device::zstd::detail::kZsNormOff;
using nvcomp::device::zstd::detail::kZsWeightOff;
using nvcomp::device::zstd::detail::kZsSymOff;
using nvcomp::device::zstd::detail::kZsSeqOff;
using nvcomp::device::zstd::detail::kZsNextOff;
using nvcomp::device::zstd::detail::kZsWarpSmem;
using nvcomp::device::zstd::detail::kZsPreLLOff;
using nvcomp::device::zstd::detail::kZsPreOFOff;
using nvcomp::device::zstd::detail::kZsPreMLOff;
using nvcomp::device::zstd::detail::kZsLLInfoOff;
using nvcomp::device::zstd::detail::kZsMLInfoOff;
using nvcomp::device::zstd::detail::kZsPreSmem;
using nvcomp::device::zstd::detail::ZstdWarp;
using nvcomp::device::zstd::detail::zs_highbit;
using nvcomp::device::zstd::detail::zs_le16;
using nvcomp::device::zstd::detail::zs_le24;
using nvcomp::device::zstd::detail::zs_le32;
using nvcomp::device::zstd::detail::zs_ld64;
using nvcomp::device::zstd::detail::ZsReload;
using nvcomp::device::zstd::detail::kZsUnfinished;
using nvcomp::device::zstd::detail::kZsEndOfBuffer;
using nvcomp::device::zstd::detail::kZsCompleted;
using nvcomp::device::zstd::detail::kZsOverflow;
using nvcomp::device::zstd::detail::ZBits;
using nvcomp::device::zstd::detail::zs_scan_excl;
using nvcomp::device::zstd::detail::zs_read_ncount;
using nvcomp::device::zstd::detail::zs_build_fse;
using nvcomp::device::zstd::detail::zs_ll_info;
using nvcomp::device::zstd::detail::zs_ml_info;
using nvcomp::device::zstd::detail::zstd_build_predefined;
using nvcomp::device::zstd::detail::zs_fse_symbol;
using nvcomp::device::zstd::detail::zs_fse_weights;
using nvcomp::device::zstd::detail::zs_read_huffman;
using nvcomp::device::zstd::detail::zs_huffman_literals;
using nvcomp::device::zstd::detail::ZsFrame;
using nvcomp::device::zstd::detail::kZsLL;
using nvcomp::device::zstd::detail::kZsOF;
using nvcomp::device::zstd::detail::kZsML;
using nvcomp::device::zstd::detail::zs_seq_table;
using nvcomp::device::zstd::detail::ZsSeq;
using nvcomp::device::zstd::detail::zs_seq_init;
using nvcomp::device::zstd::detail::zs_seq_decode;
using nvcomp::device::zstd::detail::zs_fill;
using nvcomp::device::zstd::detail::zs_move_fwd;
using nvcomp::device::zstd::detail::zs_compressed_block;
using nvcomp::device::zstd::detail::zstd_chunk;

}  // namespace b200
