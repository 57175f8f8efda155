"""ctypes view of build/tests/libans_device.so: warp-per-chunk kernels over the warp-level ANS device API
(include/nvcomp/device/ans.cuh), in the batched C API's layout (device arrays of pointers and sizes).  Used by
tests/test_ans_device_gpu.py and tools/ans_device_bench.py."""
from __future__ import annotations

import ctypes as C
import os

import torch

from nvcomp_b200.batched import Batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "tests", "libans_device.so")

_P, _Z = C.c_void_p, C.c_size_t


class AnsDevice:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make`")
        lib = C.CDLL(LIB_PATH)
        for name in ("max_compressed_bytes", "compress_temp_bytes"):
            getattr(lib, f"ans_dev_{name}").argtypes = [_Z]
        for name in ("max_compressed_bytes", "max_chunk_bytes", "decompress_smem_bytes", "compress_smem_bytes",
                     "smem_alignment", "compress_temp_bytes"):
            getattr(lib, f"ans_dev_{name}").restype = _Z
        lib.ans_dev_decompress.argtypes = [_P] * 6 + [_Z, _P]
        lib.ans_dev_compress.argtypes = [_P] * 5 + [_Z, _P, _P]
        lib.ans_dev_mixed.argtypes = [_P] * 5 + [_Z, _P] + [_P] * 6 + [_Z, _P]
        lib.ans_dev_fused.argtypes = [_P] * 8 + [_Z, _P]
        lib.ans_dev_decompressed_size.argtypes = [_P] * 3 + [_Z, _P]
        self.lib = lib

    def max_compressed_bytes(self, n: int) -> int:
        return self.lib.ans_dev_max_compressed_bytes(n)

    def max_chunk_bytes(self) -> int:
        return self.lib.ans_dev_max_chunk_bytes()

    def compress_temp(self, batch: int) -> torch.Tensor:
        return torch.empty(self.lib.ans_dev_compress_temp_bytes(batch), dtype=torch.uint8, device="cuda")

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    @staticmethod
    def _check(err: int, what: str) -> None:
        if err != 0:
            raise RuntimeError(f"{what}: cudaError {err}")

    def compress_async(self, inp: Batch, out: Batch, status: torch.Tensor, tmp: torch.Tensor) -> None:
        """Compress inp into out (out.sizes receives the compressed sizes)."""
        self._check(self.lib.ans_dev_compress(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                              out.sizes.data_ptr(), status.data_ptr(), len(inp), tmp.data_ptr(),
                                              self._stream()), "ans_dev_compress")

    def decompress_async(self, comp: Batch, out: Batch, actual: torch.Tensor, status: torch.Tensor) -> None:
        """Decompress comp into out (capacities = out.sizes)."""
        self._check(self.lib.ans_dev_decompress(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                                out.sizes.data_ptr(), actual.data_ptr(), status.data_ptr(),
                                                len(comp), self._stream()), "ans_dev_decompress")

    def mixed_async(self, inp: Batch, cout: Batch, cstatus: torch.Tensor, tmp: torch.Tensor, comp: Batch,
                    dout: Batch, actual: torch.Tensor, dstatus: torch.Tensor) -> None:
        self._check(self.lib.ans_dev_mixed(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), cout.ptrs.data_ptr(),
                                           cout.sizes.data_ptr(), cstatus.data_ptr(), len(inp), tmp.data_ptr(),
                                           comp.ptrs.data_ptr(), comp.sizes.data_ptr(), dout.ptrs.data_ptr(),
                                           dout.sizes.data_ptr(), actual.data_ptr(), dstatus.data_ptr(), len(comp),
                                           self._stream()), "ans_dev_mixed")

    def fused_async(self, comp: Batch, out: Batch, actual: torch.Tensor, status: torch.Tensor, sums: torch.Tensor,
                    hists: torch.Tensor) -> None:
        self._check(self.lib.ans_dev_fused(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                           out.sizes.data_ptr(), actual.data_ptr(), status.data_ptr(),
                                           sums.data_ptr(), hists.data_ptr(), len(comp), self._stream()),
                    "ans_dev_fused")

    def decompressed_size(self, comp: Batch) -> torch.Tensor:
        sizes = torch.full((max(len(comp), 1),), -1, dtype=torch.int64, device="cuda")
        self._check(self.lib.ans_dev_decompressed_size(comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                                       sizes.data_ptr(), len(comp), self._stream()),
                    "ans_dev_decompressed_size")
        return sizes[:len(comp)]
