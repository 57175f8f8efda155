"""ctypes binding of the C ABI exported by libnvcomp.so (include/nvcomp/*.h)."""
from __future__ import annotations

import ctypes as C
import enum
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

FORMATS = ("LZ4", "Snappy", "Cascaded", "Bitcomp", "ANS", "Deflate")

# formats this library decodes but does not encode (streams from zlib, gzip, libzstd, Parquet / ORC writers, ...):
# the three decompression entry points below are the ones they implement (include/nvcomp/gzip.h, zstd.h, lz4frame.h)
DECODE_ONLY_FORMATS = ("Gzip", "Zstd", "LZ4Frame")
DECODE_ENTRY_POINTS = ("DecompressGetTempSize", "GetDecompressSizeAsync", "DecompressAsync")

# the six (+2 Ex) entry points every format exports -- SURVEY.md section 8b
ENTRY_POINTS = (
    "CompressGetTempSize",
    "CompressGetTempSizeEx",
    "CompressGetMaxOutputChunkSize",
    "CompressAsync",
    "DecompressGetTempSize",
    "DecompressGetTempSizeEx",
    "GetDecompressSizeAsync",
    "DecompressAsync",
)


class Status(enum.IntEnum):
    Success = 0
    ErrorInvalidValue = 10
    ErrorNotSupported = 11
    ErrorCannotDecompress = 12
    ErrorBadChecksum = 13
    ErrorCannotVerifyChecksums = 14
    ErrorOutputBufferTooSmall = 15
    ErrorWrongHeaderLength = 16
    ErrorAlignment = 17
    ErrorChunkSizeTooLarge = 18
    ErrorCudaError = 1000
    ErrorInternal = 10000


class Type(enum.IntEnum):
    CHAR = 0
    UCHAR = 1
    SHORT = 2
    USHORT = 3
    INT = 4
    UINT = 5
    LONGLONG = 6
    ULONGLONG = 7
    BITS = 0xFF


class LZ4Opts(C.Structure):
    _fields_ = [("data_type", C.c_int)]


class SnappyOpts(C.Structure):
    _fields_ = [("reserved", C.c_int)]


class CascadedOpts(C.Structure):
    _fields_ = [("chunk_size", C.c_size_t), ("type", C.c_int), ("num_RLEs", C.c_int),
                ("num_deltas", C.c_int), ("use_bp", C.c_int)]


class BitcompOpts(C.Structure):
    _fields_ = [("algorithm_type", C.c_int), ("data_type", C.c_int)]


class ANSOpts(C.Structure):
    _fields_ = [("type", C.c_int)]


class DeflateOpts(C.Structure):
    _fields_ = [("algo", C.c_int)]     # 0 high throughput, 1 high compression, 2 entropy only


OPTS = {"LZ4": LZ4Opts, "Snappy": SnappyOpts, "Cascaded": CascadedOpts,
        "Bitcomp": BitcompOpts, "ANS": ANSOpts, "Deflate": DeflateOpts}

DEFAULT_OPTS = {
    "LZ4": lambda: LZ4Opts(Type.CHAR),
    "Snappy": lambda: SnappyOpts(0),
    "Cascaded": lambda: CascadedOpts(4096, Type.INT, 2, 1, 1),
    "Bitcomp": lambda: BitcompOpts(0, Type.UCHAR),
    "ANS": lambda: ANSOpts(0),
    "Deflate": lambda: DeflateOpts(0),
}


def lib_path() -> str:
    return os.path.join(_HERE, "lib", "libnvcomp.so")


def _declare(lib: C.CDLL) -> None:
    vp, sz, szp = C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)
    for fmt in FORMATS:
        opts = OPTS[fmt]
        sigs = {
            "CompressGetTempSize": [sz, sz, opts, szp],
            "CompressGetTempSizeEx": [sz, sz, opts, szp, sz],
            "CompressGetMaxOutputChunkSize": [sz, opts, szp],
            "CompressAsync": [vp, vp, sz, sz, vp, sz, vp, vp, opts, vp],
            "DecompressGetTempSize": [sz, sz, szp],
            "DecompressGetTempSizeEx": [sz, sz, szp, sz],
            "GetDecompressSizeAsync": [vp, vp, vp, sz, vp],
            "DecompressAsync": [vp, vp, vp, vp, sz, vp, sz, vp, vp, vp],
        }
        for name, args in sigs.items():
            fn = getattr(lib, f"nvcompBatched{fmt}{name}")
            fn.argtypes = args
            fn.restype = C.c_int
    decode_sigs = {
        "DecompressGetTempSize": [sz, sz, szp],
        "GetDecompressSizeAsync": [vp, vp, vp, sz, vp],
        "DecompressAsync": [vp, vp, vp, vp, sz, vp, sz, vp, vp, vp],
    }
    for fmt in DECODE_ONLY_FORMATS:
        for name in DECODE_ENTRY_POINTS:
            fn = getattr(lib, f"nvcompBatched{fmt}{name}")
            fn.argtypes = decode_sigs[name]
            fn.restype = C.c_int


def load() -> C.CDLL:
    """Load libnvcomp.so.  Fails loudly: there is no CPU or torch fallback."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `make` or `python -c 'import __graft_entry__ as g; g.build()'`. "
            "nvcomp_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    _declare(lib)
    _LIB = lib
    return lib
