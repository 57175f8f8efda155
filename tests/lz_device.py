"""ctypes view of build/tests/liblz_device.so: warp-per-chunk kernels over the warp-level LZ4 and Snappy device APIs
(include/nvcomp/device/lz4.cuh, snappy.cuh), in the batched C API's layout (device arrays of pointers and sizes).
Used by tests/test_lz_device_gpu.py and tools/lz_device_bench.py.

`kind` is "lz4" or "snappy".  A `ticket` is a zeroed int64 device tensor: the kernel's warps then pull chunks from it
(persistent grid, one wave of resident CTAs) instead of taking a static stride."""
from __future__ import annotations

import ctypes as C
import os

import torch

from nvcomp_b200.batched import Batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "tests", "liblz_device.so")

_P, _Z, _I = C.c_void_p, C.c_size_t, C.c_int
CODEC = {"lz4": 0, "snappy": 1}


def _ptr(t):
    return None if t is None else t.data_ptr()


class LzDevice:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make`")
        lib = C.CDLL(LIB_PATH)
        lib.lz_dev_constants.argtypes = [_I, _P]
        lib.lz_dev_region_bytes.restype = _Z
        lib.lz_dev_max_compressed_bytes.argtypes = [_I, _Z]
        lib.lz_dev_max_compressed_bytes.restype = _Z
        lib.lz_dev_compress.argtypes = [_I] + [_P] * 5 + [_Z, _I, _P, _P]
        lib.lz_dev_decompress.argtypes = [_I] + [_P] * 6 + [_Z, _P, _P]
        lib.lz_dev_decompress_sum.argtypes = [_I] + [_P] * 6 + [_Z, _P, _P]
        lib.lz_dev_sum.argtypes = [_P] * 3 + [_Z, _P, _P]
        lib.lz_dev_decompressed_size.argtypes = [_I] + [_P] * 3 + [_Z, _P]
        lib.lz_dev_hygiene.argtypes = [_I] + [_P] * 8 + [_Z, _P]
        lib.lz_dev_mixed.argtypes = ([_P] * 5 + [_Z]) * 2 + ([_P] * 6 + [_Z]) * 2 + [_I, _P]
        self.lib = lib

    def constants(self, kind: str) -> dict:
        """kMaxChunkBytes, kSmemAlignment, kDecompressSmemBytes, kCompressSmemBytes of the codec's header."""
        out = (C.c_size_t * 4)()
        self.lib.lz_dev_constants(CODEC[kind], out)
        return dict(zip(("max_chunk", "alignment", "decompress_smem", "compress_smem"), list(out)))

    def region_bytes(self) -> int:
        """Shared memory each warp of the test kernels owns."""
        return self.lib.lz_dev_region_bytes()

    def max_compressed_bytes(self, kind: str, n: int) -> int:
        return self.lib.lz_dev_max_compressed_bytes(CODEC[kind], n)

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    @staticmethod
    def _check(err: int, what: str) -> None:
        if err != 0:
            raise RuntimeError(f"{what}: cudaError {err}")

    def compress_async(self, kind: str, inp: Batch, out: Batch, status: torch.Tensor, data_type: int = 0,
                       ticket: torch.Tensor | None = None) -> None:
        """compress_warp on every chunk of inp into out (out.sizes receives the compressed sizes).  data_type: the LZ4
        option (ignored for Snappy)."""
        self._check(self.lib.lz_dev_compress(CODEC[kind], inp.ptrs.data_ptr(), inp.sizes.data_ptr(),
                                             out.ptrs.data_ptr(), out.sizes.data_ptr(), _ptr(status), len(inp),
                                             data_type, _ptr(ticket), self._stream()), "lz_dev_compress")

    def decompress_async(self, kind: str, comp: Batch, out: Batch, actual: torch.Tensor | None,
                         status: torch.Tensor | None, ticket: torch.Tensor | None = None) -> None:
        """decompress_warp on every chunk of comp into out (capacities = out.sizes)."""
        self._check(self.lib.lz_dev_decompress(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                               out.ptrs.data_ptr(), out.sizes.data_ptr(), _ptr(actual), _ptr(status),
                                               len(comp), _ptr(ticket), self._stream()), "lz_dev_decompress")

    def decompress_sum_async(self, kind: str, comp: Batch, out: Batch, sums: torch.Tensor, status: torch.Tensor,
                             ticket: torch.Tensor | None = None) -> None:
        """decompress_warp, then the same warp sums the chunk's 32-bit words (u64, wrapping)."""
        self._check(self.lib.lz_dev_decompress_sum(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                                   out.ptrs.data_ptr(), out.sizes.data_ptr(), sums.data_ptr(),
                                                   status.data_ptr(), len(comp), _ptr(ticket), self._stream()),
                    "lz_dev_decompress_sum")

    def sum_async(self, data: Batch, sizes: torch.Tensor, sums: torch.Tensor,
                  ticket: torch.Tensor | None = None) -> None:
        """One warp per chunk: the u64 sum of its 32-bit words, sizes[c] bytes."""
        self._check(self.lib.lz_dev_sum(data.ptrs.data_ptr(), sizes.data_ptr(), sums.data_ptr(), len(data),
                                        _ptr(ticket), self._stream()), "lz_dev_sum")

    def decompressed_size(self, kind: str, comp: Batch) -> torch.Tensor:
        """lz4::decompressed_size_warp (one warp per chunk) or snappy::decompressed_size (one thread per chunk)."""
        sizes = torch.full((max(len(comp), 1),), -1, dtype=torch.int64, device="cuda")
        self._check(self.lib.lz_dev_decompressed_size(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                                      sizes.data_ptr(), len(comp), self._stream()),
                    "lz_dev_decompressed_size")
        return sizes[:len(comp)]

    def hygiene_async(self, kind: str, comp: Batch, out: Batch, actual: torch.Tensor, status: torch.Tensor,
                      mismatch: torch.Tensor, canary_bad: torch.Tensor) -> None:
        """One warp decodes comp in order with one region and overwrites / reads back the region after every call
        (see tests/cpp/lz_device_kernels.cu, hygiene_kernel)."""
        self._check(self.lib.lz_dev_hygiene(CODEC[kind], comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                                            out.ptrs.data_ptr(), out.sizes.data_ptr(), actual.data_ptr(),
                                            status.data_ptr(), mismatch.data_ptr(), canary_bad.data_ptr(), len(comp),
                                            self._stream()), "lz_dev_hygiene")

    def mixed_async(self, roles, data_type: int = 0) -> None:
        """Four warps per CTA: roles = [(inp, out, status) LZ4 compress, (inp, out, status) Snappy compress,
        (comp, out, actual, status) LZ4 decompress, (comp, out, actual, status) Snappy decompress]."""
        args = []
        for k, r in enumerate(roles):
            if k < 2:
                inp, out, st = r
                args += [inp.ptrs.data_ptr(), inp.sizes.data_ptr(), out.ptrs.data_ptr(), out.sizes.data_ptr(),
                         st.data_ptr(), len(inp)]
            else:
                comp, out, actual, st = r
                args += [comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.ptrs.data_ptr(), out.sizes.data_ptr(),
                         actual.data_ptr(), st.data_ptr(), len(comp)]
        self._check(self.lib.lz_dev_mixed(*args, data_type, self._stream()), "lz_dev_mixed")
