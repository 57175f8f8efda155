// lz_decode.cuh -- the block-parallel LZ77 (LZ4 / Snappy) chunk decoder.  It lives in
// nvcomp/device/detail/lz_decode.cuh, shared with the device API of nvcomp/device/lz4.cuh and snappy.cuh; this file
// re-exports its names into namespace b200.
#pragma once

#include "common.cuh"
#include "nvcomp/device/detail/lz_decode.cuh"

namespace b200 {

using nvcomp::device::lz::detail::kRingBytes;
using nvcomp::device::lz::detail::kRingMask;
using nvcomp::device::lz::detail::kFlushBlock;
using nvcomp::device::lz::detail::kRingReach;
using nvcomp::device::lz::detail::LzState;
using nvcomp::device::lz::detail::kNoPrefetch;
using nvcomp::device::lz::detail::kNextUnknown;
using nvcomp::device::lz::detail::kNextSerial;
using nvcomp::device::lz::detail::kNextBlock;
using nvcomp::device::lz::detail::ring_idx;
using nvcomp::device::lz::detail::ring_ld;
using nvcomp::device::lz::detail::ring_st;
using nvcomp::device::lz::detail::lz_flush;
using nvcomp::device::lz::detail::lz_flush_blocks;
using nvcomp::device::lz::detail::kTokStop;
using nvcomp::device::lz::detail::kTokExt;
using nvcomp::device::lz::detail::kMaxTokOut;
using nvcomp::device::lz::detail::lds_u32_any;
using nvcomp::device::lz::detail::lane_private;
using nvcomp::device::lz::detail::byte_mask;
using nvcomp::device::lz::detail::Lz4Policy;
using nvcomp::device::lz::detail::SnappyPolicy;
using nvcomp::device::lz::detail::kSegBytes;
using nvcomp::device::lz::detail::kBlkBytes;
using nvcomp::device::lz::detail::kBlkPad;
using nvcomp::device::lz::detail::kBlkStage;
using nvcomp::device::lz::detail::kMaxStepOut;
using nvcomp::device::lz::detail::kSmemIn;
using nvcomp::device::lz::detail::kSmemRec;
using nvcomp::device::lz::detail::kSmemMbar;
using nvcomp::device::lz::detail::kLzWarpSmem;
using nvcomp::device::lz::detail::lz_warp_init;
using nvcomp::device::lz::detail::lz_stage_wait;
using nvcomp::device::lz::detail::lz_stage_issue;
using nvcomp::device::lz::detail::lz_prefetch_block;
using nvcomp::device::lz::detail::lz_serial_lookahead;
using nvcomp::device::lz::detail::lz_block;
using nvcomp::device::lz::detail::kMediumMax;
using nvcomp::device::lz::detail::ring_put_literals;
using nvcomp::device::lz::detail::ring_match;
using nvcomp::device::lz::detail::ring_from_of;
using nvcomp::device::lz::detail::lz_out_byte;
using nvcomp::device::lz::detail::lz_emit_literals;
using nvcomp::device::lz::detail::lz_emit_match;
using nvcomp::device::lz::detail::lz_decode_loop;
using nvcomp::device::lz::detail::lz_decode_stream;

}  // namespace b200
