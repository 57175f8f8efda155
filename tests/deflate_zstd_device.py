"""ctypes view of build/tests/libdeflate_zstd_device.so: warp-per-chunk kernels over the warp-level Deflate, Gzip and
Zstd device APIs (include/nvcomp/device/deflate.cuh, gzip.cuh, zstd.cuh), in the batched C API's layout (device arrays
of pointers and sizes).  Used by tests/test_deflate_device_gpu.py, tests/test_zstd_device_gpu.py and
tools/deflate_zstd_device_bench.py.

`kind` is "deflate", "gzip" or "zstd".  A `ticket` is a zeroed int64 device tensor: the kernel's warps then pull chunks
from it (persistent grid, one wave of resident CTAs) instead of taking a static stride."""
from __future__ import annotations

import ctypes as C
import os

import torch

from nvcomp_b200.batched import Batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "tests", "libdeflate_zstd_device.so")

_P, _Z, _I = C.c_void_p, C.c_size_t, C.c_int
CODEC = {"deflate": 0, "gzip": 1, "zstd": 2}
CONSTANTS = ("deflate_decompress_smem", "deflate_compress_smem_0", "deflate_compress_smem_1",
             "deflate_compress_smem_2", "deflate_compress_smem_3", "deflate_compress_smem_neg1",
             "deflate_max_compress_chunk", "deflate_alignment", "gzip_decompress_smem", "gzip_alignment",
             "zstd_decompress_smem", "zstd_alignment")


def _ptr(t):
    return None if t is None else t.data_ptr()


class DeflateZstdDevice:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make`")
        lib = C.CDLL(LIB_PATH)
        lib.dz_dev_constants.argtypes = [_P]
        lib.dz_dev_region_bytes.restype = _Z
        lib.dz_dev_max_compressed_bytes.argtypes = [_Z]
        lib.dz_dev_max_compressed_bytes.restype = _Z
        lib.dz_dev_compress.argtypes = [_P] * 5 + [_Z, _I, _P, _P]
        lib.dz_dev_decompress.argtypes = [_I] + [_P] * 6 + [_Z, _P, _P]
        lib.dz_dev_decompress_sum.argtypes = [_I] + [_P] * 6 + [_Z, _P, _P]
        lib.dz_dev_sum.argtypes = [_P] * 3 + [_Z, _P, _P]
        lib.dz_dev_decompressed_size.argtypes = [_I] + [_P] * 3 + [_Z, _P]
        lib.dz_dev_reuse.argtypes = [_I] + [_P] * 8 + [_Z, _P]
        lib.dz_dev_mixed.argtypes = [_P] * 5 + [_Z] + ([_P] * 6 + [_Z]) * 3 + [_I, _P]
        self.lib = lib

    def constants(self) -> dict:
        """The sizes and alignments the three headers publish (see dz_dev_constants)."""
        out = (C.c_size_t * len(CONSTANTS))()
        self.lib.dz_dev_constants(out)
        return dict(zip(CONSTANTS, list(out)))

    def region_bytes(self) -> int:
        """Shared memory each warp of the test kernels owns (algo-1 compression aside)."""
        return self.lib.dz_dev_region_bytes()

    def max_compressed_bytes(self, n: int) -> int:
        return self.lib.dz_dev_max_compressed_bytes(n)

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    @staticmethod
    def _check(err: int, what: str) -> None:
        if err != 0:
            raise RuntimeError(f"{what}: cudaError {err}")

    def compress_async(self, inp: Batch, out: Batch, status: torch.Tensor | None, algo: int = 0,
                       ticket: torch.Tensor | None = None) -> None:
        """deflate::compress_warp on every chunk of inp into out (out.sizes receives the compressed sizes)."""
        self._check(self.lib.dz_dev_compress(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                             out.sizes.data_ptr(), _ptr(status), len(inp), algo, _ptr(ticket),
                                             self._stream()), "dz_dev_compress")

    def decompress_async(self, kind: str, comp: Batch, out: Batch, actual: torch.Tensor | None,
                         status: torch.Tensor | None, ticket: torch.Tensor | None = None) -> None:
        """decompress_warp on every chunk of comp into out (capacities = out.sizes)."""
        self._check(self.lib.dz_dev_decompress(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                               out.ptrs.data_ptr(), out.sizes.data_ptr(), _ptr(actual), _ptr(status),
                                               len(comp), _ptr(ticket), self._stream()), "dz_dev_decompress")

    def decompress_sum_async(self, kind: str, comp: Batch, out: Batch, sums: torch.Tensor, status: torch.Tensor,
                             ticket: torch.Tensor | None = None) -> None:
        """decompress_warp, then the same warp sums the chunk's 32-bit words (u64, wrapping)."""
        self._check(self.lib.dz_dev_decompress_sum(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                                   out.ptrs.data_ptr(), out.sizes.data_ptr(), sums.data_ptr(),
                                                   status.data_ptr(), len(comp), _ptr(ticket), self._stream()),
                    "dz_dev_decompress_sum")

    def sum_async(self, data: Batch, sizes: torch.Tensor, sums: torch.Tensor,
                  ticket: torch.Tensor | None = None) -> None:
        """One warp per chunk: the u64 sum of its 32-bit words, sizes[c] bytes."""
        self._check(self.lib.dz_dev_sum(data.ptrs.data_ptr(), sizes.data_ptr(), sums.data_ptr(), len(data),
                                        _ptr(ticket), self._stream()), "dz_dev_sum")

    def decompressed_size(self, kind: str, comp: Batch) -> torch.Tensor:
        """decompressed_size_warp, one warp per chunk."""
        sizes = torch.full((max(len(comp), 1),), -1, dtype=torch.int64, device="cuda")
        self._check(self.lib.dz_dev_decompressed_size(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                                      sizes.data_ptr(), len(comp), self._stream()),
                    "dz_dev_decompressed_size")
        return sizes[:len(comp)]

    def reuse_async(self, kind: str, comp: Batch, out: Batch, actual: torch.Tensor, status: torch.Tensor,
                    mismatch: torch.Tensor, canary_bad: torch.Tensor) -> None:
        """One warp decodes comp in order with one region and overwrites the region with 0xA5 after every call (see
        tests/cpp/deflate_zstd_device_kernels.cu, reuse_kernel)."""
        self._check(self.lib.dz_dev_reuse(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                          out.ptrs.data_ptr(), out.sizes.data_ptr(), actual.data_ptr(),
                                          status.data_ptr(), mismatch.data_ptr(), canary_bad.data_ptr(), len(comp),
                                          self._stream()), "dz_dev_reuse")

    def mixed_async(self, roles, algo: int = 0) -> None:
        """Four warps per CTA: roles = [(inp, out, status) Deflate compress, then (comp, out, actual, status) for
        Deflate, Gzip and Zstd decompression]."""
        inp, out, st = roles[0]
        args = [inp.ptrs.data_ptr(), inp.sizes.data_ptr(), out.ptrs.data_ptr(), out.sizes.data_ptr(), st.data_ptr(),
                len(inp)]
        for comp, out, actual, st in roles[1:]:
            args += [comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.ptrs.data_ptr(), out.sizes.data_ptr(),
                     actual.data_ptr(), st.data_ptr(), len(comp)]
        self._check(self.lib.dz_dev_mixed(*args, algo, self._stream()), "dz_dev_mixed")
