import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def _ensure_built():
    need = [os.path.join(ROOT, "oracle", "liboracle.so"), os.path.join(ROOT, "nvcomp_b200", "lib", "libnvcomp.so")]
    if not all(os.path.exists(p) for p in need):
        subprocess.run(["make", "-C", ROOT, "-j4"], check=True, stdout=subprocess.DEVNULL)


class Oracle:
    """ctypes view of oracle/liboracle.so -- the CPU checker (tests only)."""

    def __init__(self):
        _ensure_built()
        self.lib = C.CDLL(os.path.join(ROOT, "oracle", "liboracle.so"))
        u8p, sz = C.c_char_p, C.c_size_t
        for name in ("lz4", "snappy", "cascaded", "bitcomp", "ans"):
            for op, args in (("decompress", [u8p, sz, u8p, sz]), ("decompressed_size", [u8p, sz])):
                fn = getattr(self.lib, f"oracle_{name}_{op}", None)
                if fn is not None:
                    fn.argtypes, fn.restype = args, C.c_long
        for name in ("lz4", "snappy"):
            fn = getattr(self.lib, f"oracle_{name}_compress")
            fn.argtypes, fn.restype = [u8p, sz, u8p, sz], C.c_long
            fn = getattr(self.lib, f"oracle_{name}_bound")
            fn.argtypes, fn.restype = [sz], sz

        self.lib.oracle_cascaded_compress.argtypes = [u8p, sz, u8p, sz, sz, C.c_uint, C.c_int, C.c_int, C.c_int]
        self.lib.oracle_cascaded_compress.restype = C.c_long
        self.lib.oracle_bitcomp_compress.argtypes = [u8p, sz, u8p, sz, C.c_uint, C.c_uint]
        self.lib.oracle_bitcomp_compress.restype = C.c_long
        self.lib.oracle_ans_compress.argtypes = [u8p, sz, u8p, sz]
        self.lib.oracle_ans_compress.restype = C.c_long

    def compress_typed(self, codec: str, data: bytes, **kw) -> bytes:
        cap = 24 * len(data) + 262144
        out = C.create_string_buffer(cap)
        if codec == "cascaded":
            r = self.lib.oracle_cascaded_compress(data, len(data), out, cap, kw.get("chunk_size", 4096), kw["type"],
                                                  kw["num_RLEs"], kw["num_deltas"], kw["use_bp"])
        elif codec == "bitcomp":
            r = self.lib.oracle_bitcomp_compress(data, len(data), out, cap, kw["algo"], kw["type"])
        else:
            r = self.lib.oracle_ans_compress(data, len(data), out, cap)
        assert r >= 0, (codec, kw)
        return out.raw[:r]

    def decompress(self, codec: str, data: bytes, cap: int):
        out = C.create_string_buffer(max(cap, 1))
        r = getattr(self.lib, f"oracle_{codec}_decompress")(data, len(data), out, cap)
        return None if r < 0 else out.raw[:r]

    def size(self, codec: str, data: bytes) -> int:
        return getattr(self.lib, f"oracle_{codec}_decompressed_size")(data, len(data))

    def compress(self, codec: str, data: bytes) -> bytes:
        cap = getattr(self.lib, f"oracle_{codec}_bound")(len(data))
        out = C.create_string_buffer(cap)
        r = getattr(self.lib, f"oracle_{codec}_compress")(data, len(data), out, cap)
        assert r >= 0
        return out.raw[:r]


class LibLZ4:
    """liblz4 1.9.4 -- the CPU codec the reference itself links (examples/lz4_cpu_*.cu)."""

    def __init__(self):
        self.lib = C.CDLL("liblz4.so.1")
        self.lib.LZ4_compress_default.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
        self.lib.LZ4_compress_HC.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int]
        self.lib.LZ4_decompress_safe.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]

    def compress(self, data: bytes, hc: int = 0) -> bytes:
        cap = self.lib.LZ4_compressBound(len(data))
        out = C.create_string_buffer(max(cap, 1))
        if hc:
            n = self.lib.LZ4_compress_HC(data, out, len(data), cap, hc)
        else:
            n = self.lib.LZ4_compress_default(data, out, len(data), cap)
        assert n > 0 or len(data) == 0
        return out.raw[:n]

    def decompress(self, data: bytes, cap: int):
        out = C.create_string_buffer(max(cap, 1))
        n = self.lib.LZ4_decompress_safe(data, out, len(data), cap)
        return None if n < 0 else out.raw[:n]


@pytest.fixture(scope="session")
def oracle():
    return Oracle()


@pytest.fixture(scope="session")
def liblz4():
    try:
        return LibLZ4()
    except OSError:
        pytest.skip("liblz4.so.1 not available")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


def sample_inputs(seed=123):
    """Small, varied chunks used by several parity tests (name -> bytes)."""
    from nvcomp_b200 import datagen
    rng = np.random.default_rng(seed)
    out = {
        "empty": b"",
        "one": b"x",
        "short12": b"abcdefghijkl",
        "short13": b"abcdefghijklm",
        "zeros_64k": bytes(65536),
        "zeros_1000": bytes(1000),
        "random_64k": rng.integers(0, 256, 65536, dtype=np.uint8).tobytes(),
        "random_777": rng.integers(0, 256, 777, dtype=np.uint8).tobytes(),
        "text": (b"the quick brown fox jumps over the lazy dog. " * 300)[:12345],
        "period3": (b"abc" * 30000)[:65536],
        "period7": (b"1234567" * 10000)[:65536],
        "period33": (bytes(range(33)) * 2000)[:65536],
        "period100": (bytes(range(100)) * 700)[:65536],
        "period600": (rng.integers(0, 256, 600, dtype=np.uint8).tobytes() * 120)[:65536],
        "runlength_i32": datagen.runlength_i32(1, seed=7)[0].tobytes(),
        "price_walk": datagen.tabular_f32(1, seed=8, column=0)[0].tobytes(),
        "lowcard": datagen.tabular_f32(1, seed=9, column=1)[0].tobytes(),
        "clustered": datagen.tabular_f32(1, seed=10, column=2)[0].tobytes(),
        "sensor": datagen.tabular_f32(1, seed=11, column=3)[0].tobytes(),
        "sorted_i64": datagen.sorted_i64(1, seed=12)[0].tobytes(),
        "lowentropy": datagen.lowentropy_bytes(1, seed=13)[0].tobytes(),
        "gen_data3": datagen.snappy_synth(1, 3, seed=0)[0].tobytes(),
        "ragged_40001": datagen.runlength_i32(1, seed=14)[0].tobytes()[:40001],
    }
    return out
