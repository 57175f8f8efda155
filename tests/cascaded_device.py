"""ctypes view of build/tests/libcascaded_device.so: warp-per-chunk kernels over the warp-level Cascaded device API
(include/nvcomp/device/cascaded.cuh), in the batched C API's layout (device arrays of pointers and sizes).  Used by
tests/test_cascaded_device_gpu.py and tools/cascaded_device_bench.py.

Options are passed as a tuple (chunk_size, type, num_RLEs, num_deltas, use_bp); `region` is each decompressing or
visiting warp's shared-memory workspace in bytes."""
from __future__ import annotations

import ctypes as C
import os

import torch

from nvcomp_b200.batched import Batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "tests", "libcascaded_device.so")

_P, _Z, _I = C.c_void_p, C.c_size_t, C.c_int
_OPTS = [_Z, _I, _I, _I, _I]


class CascadedDevice:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make`")
        lib = C.CDLL(LIB_PATH)
        lib.cascaded_dev_max_compressed_bytes.argtypes = [_Z] + _OPTS
        lib.cascaded_dev_compress_smem_bytes.argtypes = _OPTS
        lib.cascaded_dev_decompress_smem_bytes.argtypes = _OPTS
        for name in ("max_compressed_bytes", "compress_smem_bytes", "decompress_smem_bytes",
                     "max_decompress_smem_bytes", "max_chunk_bytes", "smem_alignment"):
            getattr(lib, f"cascaded_dev_{name}").restype = _Z
        lib.cascaded_dev_compress.argtypes = [_P] * 5 + [_Z] + _OPTS + [_P]
        lib.cascaded_dev_decompress.argtypes = [_P] * 6 + [_Z, _Z, _P]
        lib.cascaded_dev_visit.argtypes = [_P] * 6 + [_Z, _I, _Z, _P]
        lib.cascaded_dev_mixed.argtypes = ([_P] * 5 + [_Z] + _OPTS + [_P] * 6 + [_Z] + [_P] * 6 + [_Z, _Z, _P])
        lib.cascaded_dev_fused_sum.argtypes = [_P] * 4 + [_Z, _Z, _P]
        lib.cascaded_dev_check.argtypes = [_P] * 3 + [_Z, _Z, _P]
        lib.cascaded_dev_sum_i64.argtypes = [_P] * 3 + [_Z, _P]
        lib.cascaded_dev_decompressed_size.argtypes = [_P] * 3 + [_Z, _P]
        self.lib = lib

    def max_compressed_bytes(self, n: int, opts) -> int:
        return self.lib.cascaded_dev_max_compressed_bytes(n, *opts)

    def compress_smem_bytes(self, opts) -> int:
        return self.lib.cascaded_dev_compress_smem_bytes(*opts)

    def decompress_smem_bytes(self, opts) -> int:
        return self.lib.cascaded_dev_decompress_smem_bytes(*opts)

    def max_decompress_smem_bytes(self) -> int:
        return self.lib.cascaded_dev_max_decompress_smem_bytes()

    def max_chunk_bytes(self) -> int:
        return self.lib.cascaded_dev_max_chunk_bytes()

    def smem_alignment(self) -> int:
        return self.lib.cascaded_dev_smem_alignment()

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    @staticmethod
    def _check(err: int, what: str) -> None:
        if err != 0:
            raise RuntimeError(f"{what}: cudaError {err}")

    def compress_async(self, inp: Batch, out: Batch, status: torch.Tensor, opts) -> None:
        """Compress inp into out (out.sizes receives the compressed sizes)."""
        self._check(self.lib.cascaded_dev_compress(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                                   out.sizes.data_ptr(), status.data_ptr(), len(inp), *opts,
                                                   self._stream()), "cascaded_dev_compress")

    def decompress_async(self, comp: Batch, out: Batch, actual: torch.Tensor, status: torch.Tensor,
                         region: int) -> None:
        """Decompress comp into out (capacities = out.sizes)."""
        self._check(self.lib.cascaded_dev_decompress(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                                     out.sizes.data_ptr(), actual.data_ptr(), status.data_ptr(),
                                                     len(comp), region, self._stream()), "cascaded_dev_decompress")

    def visit_async(self, comp: Batch, elem_type: int, sums: torch.Tensor, hashes: torch.Tensor, visits: torch.Tensor,
                    status: torch.Tensor, region: int) -> None:
        """for_each_block with the element type elem_type (an nvcompType_t): per chunk the wrapping u64 sum, the
        order-sensitive hash and the number of visits (see tests/cpp/cascaded_device_kernels.cu)."""
        self._check(self.lib.cascaded_dev_visit(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), sums.data_ptr(),
                                                hashes.data_ptr(), visits.data_ptr(), status.data_ptr(), len(comp),
                                                elem_type, region, self._stream()), "cascaded_dev_visit")

    def mixed_async(self, inp: Batch, cout: Batch, cstatus: torch.Tensor, opts, comp: Batch, dout: Batch,
                    actual: torch.Tensor, dstatus: torch.Tensor, vcomp: Batch, sums: torch.Tensor,
                    hashes: torch.Tensor, visits: torch.Tensor, vstatus: torch.Tensor, region: int) -> None:
        self._check(self.lib.cascaded_dev_mixed(
            inp.ptrs.data_ptr(), inp.sizes.data_ptr(), cout.ptrs.data_ptr(), cout.sizes.data_ptr(),
            cstatus.data_ptr(), len(inp), *opts, comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
            dout.ptrs.data_ptr(), dout.sizes.data_ptr(), actual.data_ptr(), dstatus.data_ptr(), len(comp),
            vcomp.ptrs.data_ptr(), vcomp.sizes.data_ptr(), sums.data_ptr(), hashes.data_ptr(), visits.data_ptr(),
            vstatus.data_ptr(), len(vcomp), region, self._stream()), "cascaded_dev_mixed")

    def fused_sum_async(self, comp: Batch, sums: torch.Tensor, status: torch.Tensor, region: int) -> None:
        self._check(self.lib.cascaded_dev_fused_sum(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), sums.data_ptr(),
                                                    status.data_ptr(), len(comp), region, self._stream()),
                    "cascaded_dev_fused_sum")

    def check_async(self, comp: Batch, ok: torch.Tensor, region: int) -> None:
        """for_each_block<int64>'s checking pass alone: ok[c] = 1 when chunk c would be visited."""
        self._check(self.lib.cascaded_dev_check(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), ok.data_ptr(),
                                                len(comp), region, self._stream()), "cascaded_dev_check")

    def sum_i64_async(self, data: Batch, sizes: torch.Tensor, sums: torch.Tensor) -> None:
        self._check(self.lib.cascaded_dev_sum_i64(data.ptrs.data_ptr(), sizes.data_ptr(), sums.data_ptr(), len(data),
                                                  self._stream()), "cascaded_dev_sum_i64")

    def decompressed_size(self, comp: Batch) -> torch.Tensor:
        sizes = torch.full((max(len(comp), 1),), -1, dtype=torch.int64, device="cuda")
        self._check(self.lib.cascaded_dev_decompressed_size(comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                                            sizes.data_ptr(), len(comp), self._stream()),
                    "cascaded_dev_decompressed_size")
        return sizes[:len(comp)]
