// ptx.cuh -- the library's inline-PTX primitives (sm_90a).  They live in nvcomp/device/detail/ptx.cuh, shared with
// the device API of nvcomp/device/lz4.cuh and snappy.cuh; this file re-exports them into namespace b200.  The codec
// headers contain no asm, so tests/emu can re-run their warp-level logic on the host by shadowing this file and that
// one (test infrastructure only; the product is CUDA).
#pragma once

#include <nvcomp/device/detail/ptx.cuh>

namespace b200 {

using nvcomp::device::lz::detail::smem_addr;
using nvcomp::device::lz::detail::ld_nc_v4;
using nvcomp::device::lz::detail::st_v4;
using nvcomp::device::lz::detail::ld_v4;
using nvcomp::device::lz::detail::lds_u8;
using nvcomp::device::lz::detail::sts_u8;
using nvcomp::device::lz::detail::lds_v4;
using nvcomp::device::lz::detail::sts_v4;
using nvcomp::device::lz::detail::lds_u32;
using nvcomp::device::lz::detail::sts_u32;
using nvcomp::device::lz::detail::lds_u16;
using nvcomp::device::lz::detail::sts_u16;
using nvcomp::device::lz::detail::ldg_u8;
using nvcomp::device::lz::detail::touch_line;
using nvcomp::device::lz::detail::ldg_u32;
using nvcomp::device::lz::detail::mbar_init;
using nvcomp::device::lz::detail::mbar_expect_tx;
using nvcomp::device::lz::detail::mbar_wait;
using nvcomp::device::lz::detail::fence_proxy_async_smem;
using nvcomp::device::lz::detail::tma_bulk_g2s;
using nvcomp::device::lz::detail::globaltimer_ns;
using nvcomp::device::lz::detail::sm_id;

}  // namespace b200
