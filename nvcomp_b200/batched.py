"""Host-side mirror of the low-level batched interface (LLIF).

Same call order and argument meaning as the reference's
``nvcompBatched<Fmt>{CompressGetTempSize, CompressGetMaxOutputChunkSize,
CompressAsync, DecompressGetTempSize, GetDecompressSizeAsync, DecompressAsync}``
(reference ``doc/lowlevel_c_quickstart.md``; ``benchmarks/benchmark_template_chunked.cuh:420-530``).
Every function here ends in exactly one call through the C ABI of
``libnvcomp.so`` with raw device pointers; torch only owns the memory and the
stream.  No compute happens in Python and nothing falls back to the CPU.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Sequence

import numpy as np
import torch

from . import _lib
from ._lib import DEFAULT_OPTS, Status


class NvcompError(RuntimeError):
    def __init__(self, fn: str, status: int):
        try:
            name = Status(status).name
        except ValueError:
            name = str(status)
        super().__init__(f"{fn} returned {name}")
        self.status = status


def _check(fn: str, st: int) -> None:
    if st != 0:
        raise NvcompError(fn, st)


def _stream_handle(stream: torch.cuda.Stream | None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return s.cuda_stream


@dataclass
class Batch:
    """A device-resident batch in the layout every LLIF call takes: one slab plus
    device arrays of chunk pointers and chunk sizes (the reference's BatchData,
    ``benchmarks/benchmark_template_chunked.cuh:162-264``)."""

    slab: torch.Tensor    # uint8, device
    ptrs: torch.Tensor    # int64 (void*), device
    sizes: torch.Tensor   # int64 (size_t), device
    offsets: np.ndarray   # host copy of the byte offset of each chunk in slab

    def __len__(self) -> int:
        return int(self.ptrs.numel())

    def to_host(self, sizes: Sequence[int] | None = None) -> list[bytes]:
        host = self.slab.cpu().numpy()
        szs = self.sizes.cpu().numpy() if sizes is None else np.asarray(sizes)
        return [host[o:o + int(n)].tobytes() for o, n in zip(self.offsets, szs)]


def _as_u8(x) -> np.ndarray:
    if isinstance(x, (bytes, bytearray, memoryview)):
        return np.frombuffer(x, dtype=np.uint8)
    return np.ascontiguousarray(x).view(np.uint8).reshape(-1)


def make_batch(chunks: Sequence, device: str | torch.device = "cuda", align: int = 16,
               pad_to: int | None = None, misalign: int = 0) -> Batch:
    """Upload host chunks into one device slab; chunk starts are `align`-byte
    aligned (+ `misalign` bytes, to exercise unaligned pointers)."""
    arrs = [_as_u8(c) for c in chunks]
    offs, cur = [], 0
    for a in arrs:
        cur = (cur + align - 1) // align * align + misalign
        offs.append(cur)
        cur += max(len(a), pad_to or 0)
    total = max(cur, 1) + 64
    host = np.zeros(total, dtype=np.uint8)
    for o, a in zip(offs, arrs):
        host[o:o + len(a)] = a
    slab = torch.from_numpy(host).to(device)
    offsets = np.asarray(offs, dtype=np.int64)
    ptrs = torch.from_numpy(offsets + slab.data_ptr()).to(device)
    sizes = torch.tensor([len(a) for a in arrs], dtype=torch.int64, device=device)
    return Batch(slab, ptrs, sizes, offsets)


def empty_batch(n: int, stride: int, device: str | torch.device = "cuda", align: int = 16,
                misalign: int = 0, fill: int | None = None) -> Batch:
    """n output buffers of `stride` bytes each (compressed outputs, decompressed outputs)."""
    stride_al = (stride + align - 1) // align * align + (align if misalign else 0)
    total = max(n * stride_al, 1) + 64 + misalign
    slab = torch.empty(total, dtype=torch.uint8, device=device)
    if fill is not None:
        slab.fill_(fill)
    offsets = np.arange(n, dtype=np.int64) * stride_al + misalign
    # make the slab base 16-byte aligned relative offsets meaningful
    ptrs = torch.from_numpy(offsets + slab.data_ptr()).to(device)
    sizes = torch.full((n,), stride, dtype=torch.int64, device=device)
    return Batch(slab, ptrs, sizes, offsets)


class Codec:
    """One format's six LLIF entry points, bound to raw pointers.  Gzip, Zstd and LZ4Frame
    (``_lib.DECODE_ONLY_FORMATS``) have only the decompression half: their compress methods raise
    NotImplementedError."""

    def __init__(self, fmt: str, opts=None):
        self.decode_only = fmt in _lib.DECODE_ONLY_FORMATS
        if fmt not in _lib.FORMATS and not self.decode_only:
            raise ValueError(f"unknown format {fmt}")
        if self.decode_only and opts is not None:
            raise ValueError(f"{fmt} is decode-only and takes no options")
        self.fmt = fmt
        self.lib = _lib.load()
        self.opts = None if self.decode_only else (opts if opts is not None else DEFAULT_OPTS[fmt]())

    def _fn(self, name: str):
        return getattr(self.lib, f"nvcompBatched{self.fmt}{name}")

    def _compress_fn(self, name: str):
        if self.decode_only:
            raise NotImplementedError(f"{self.fmt} is decode-only in this library: {name} is not available "
                                      "(compress on the host, e.g. with zlib, and decode on the GPU)")
        return self._fn(name)

    # --- host-only size queries -------------------------------------------------
    def compress_get_temp_size(self, batch_size: int, max_chunk: int) -> int:
        out = C.c_size_t(0)
        _check("CompressGetTempSize",
               self._compress_fn("CompressGetTempSize")(batch_size, max_chunk, self.opts, C.byref(out)))
        return out.value

    def compress_get_max_output_chunk_size(self, max_chunk: int) -> int:
        out = C.c_size_t(0)
        _check("CompressGetMaxOutputChunkSize",
               self._compress_fn("CompressGetMaxOutputChunkSize")(max_chunk, self.opts, C.byref(out)))
        return out.value

    def decompress_get_temp_size(self, batch_size: int, max_chunk: int) -> int:
        out = C.c_size_t(0)
        _check("DecompressGetTempSize", self._fn("DecompressGetTempSize")(batch_size, max_chunk, C.byref(out)))
        return out.value

    # --- async device calls -----------------------------------------------------
    def compress_async(self, in_ptrs: int, in_bytes: int, max_chunk: int, batch: int, temp: int,
                       temp_bytes: int, out_ptrs: int, out_bytes: int, stream: int) -> None:
        _check("CompressAsync", self._compress_fn("CompressAsync")(
            in_ptrs, in_bytes, max_chunk, batch, temp, temp_bytes, out_ptrs, out_bytes, self.opts, stream))

    def get_decompress_size_async(self, comp_ptrs: int, comp_bytes: int, out_sizes: int, batch: int,
                                  stream: int) -> None:
        _check("GetDecompressSizeAsync", self._fn("GetDecompressSizeAsync")(
            comp_ptrs, comp_bytes, out_sizes, batch, stream))

    def decompress_async(self, comp_ptrs: int, comp_bytes: int, out_caps: int, actual: int, batch: int,
                         temp: int, temp_bytes: int, out_ptrs: int, statuses: int, stream: int) -> None:
        _check("DecompressAsync", self._fn("DecompressAsync")(
            comp_ptrs, comp_bytes, out_caps, actual, batch, temp, temp_bytes, out_ptrs, statuses, stream))

    # --- conveniences over torch-owned memory ------------------------------------
    def compress(self, inp: Batch, max_chunk: int | None = None,
                 stream: torch.cuda.Stream | None = None) -> Batch:
        n = len(inp)
        if max_chunk is None:
            max_chunk = int(inp.sizes.max().item()) if n else 0
        tb = self.compress_get_temp_size(n, max_chunk)
        temp = torch.empty(max(tb, 1), dtype=torch.uint8, device=inp.slab.device)
        max_out = self.compress_get_max_output_chunk_size(max_chunk)
        out = empty_batch(n, max_out, device=inp.slab.device)
        self.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), max_chunk, n, temp.data_ptr(), tb,
                            out.ptrs.data_ptr(), out.sizes.data_ptr(), _stream_handle(stream))
        out._keep = temp  # keep workspace alive until the stream drains
        return out

    def get_decompress_size(self, comp: Batch, stream: torch.cuda.Stream | None = None) -> torch.Tensor:
        n = len(comp)
        out = torch.zeros(max(n, 1), dtype=torch.int64, device=comp.slab.device)
        self.get_decompress_size_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.data_ptr(), n,
                                       _stream_handle(stream))
        return out[:n]

    def decompress(self, comp: Batch, out: Batch, max_chunk: int | None = None, want_actual: bool = True,
                   want_status: bool = True, stream: torch.cuda.Stream | None = None,
                   temp: torch.Tensor | None = None):
        """Decompress comp -> out (capacities = out.sizes).  Returns (actual, statuses)
        device tensors (None when not requested)."""
        n = len(comp)
        dev = comp.slab.device
        if max_chunk is None:
            max_chunk = int(out.sizes.max().item()) if n else 0
        tb = self.decompress_get_temp_size(n, max_chunk)
        if temp is None:
            temp = torch.empty(max(tb, 1), dtype=torch.uint8, device=dev)
        actual = torch.zeros(max(n, 1), dtype=torch.int64, device=dev) if want_actual else None
        status = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev) if want_status else None
        self.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(),
                              actual.data_ptr() if want_actual else None, n, temp.data_ptr(), tb,
                              out.ptrs.data_ptr(), status.data_ptr() if want_status else None,
                              _stream_handle(stream))
        out._keep = temp
        return (actual[:n] if want_actual else None), (status[:n] if want_status else None)
