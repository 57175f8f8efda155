// tests/emu/nvcomp/device/detail/ptx.cuh -- TEST INFRASTRUCTURE: shadows include/nvcomp/device/detail/ptx.cuh in
// the host emulator build.  The LZ headers under include/nvcomp/device/detail include the PTX by this angle-bracket
// path and tests/emu is first on the emulator's include path, so they get the host stand-ins of tests/emu/ptx.cuh
// (bounds-checked shared and global accesses, the emulated mbarrier and bulk copy) under the names they call.
#pragma once

#include "../../../ptx.cuh"

namespace nvcomp {
namespace device {
namespace lz {
namespace detail {

using b200::smem_addr;
using b200::ld_nc_v4;
using b200::st_v4;
using b200::ld_v4;
using b200::lds_u8;
using b200::sts_u8;
using b200::lds_v4;
using b200::sts_v4;
using b200::lds_u32;
using b200::sts_u32;
using b200::lds_u16;
using b200::sts_u16;
using b200::ldg_u8;
using b200::touch_line;
using b200::ldg_u32;
using b200::mbar_init;
using b200::mbar_expect_tx;
using b200::mbar_wait;
using b200::fence_proxy_async_smem;
using b200::tma_bulk_g2s;

// the emulated barrier is a phase counter in its 8 bytes: invalidating it clears them
__device__ __forceinline__ void mbar_inval(uint32_t mbar) { memset(emu::smem_ptr(mbar, 8), 0, 8); }

}  // namespace detail
}  // namespace lz
}  // namespace device
}  // namespace nvcomp
