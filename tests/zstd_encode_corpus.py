"""The warp-level Zstd encoder (include/nvcomp/device/detail/zstd_encode.cuh) in the host warp emulator, and the
inputs its tests share: tests/test_zstd_encode_emu.py checks the emulated frames, tests/test_zstd_compress_device_gpu.py
holds the GPU's frames to them byte for byte."""
import ctypes as C
import glob
import os
import subprocess

import numpy as np

from conftest import ROOT, sample_inputs

FAULT = -2


class EmuZstdEncoder:
    def __init__(self):
        subprocess.run(["make", "-C", ROOT, "tests/emu/libemu_lz.so"], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "libemu_lz.so"))
        self.lib.emu_zstd_compress.restype = C.c_long
        self.lib.emu_zstd_compress.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.c_uint, C.c_char_p, C.c_char_p,
                                               C.c_size_t]
        self.lib.emu_zstd_enc_bound.restype = C.c_size_t
        self.lib.emu_zstd_enc_bound.argtypes = [C.c_size_t]
        self.lib.emu_zstd_enc_smem.restype = C.c_size_t

    def bound(self, n: int) -> int:
        return self.lib.emu_zstd_enc_bound(n)

    def compress(self, data: bytes, in_mis: int = 0, out_mis: int = 0) -> bytes:
        """One frame; the emulator also checks that nothing past the frame was written."""
        out = C.create_string_buffer(max(self.bound(len(data)), 1))
        msg = C.create_string_buffer(256)
        r = self.lib.emu_zstd_compress(data, len(data), in_mis, out_mis, out, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        return out.raw[:r]


def fibonacci_bytes(n=65536, seed=5):
    """Literal frequencies in Fibonacci proportion over 22 symbols: an unlimited Huffman code would be 21 bits deep,
    so the 11-bit limit binds."""
    fib = [1, 1]
    while len(fib) < 22:
        fib.append(fib[-1] + fib[-2])
    scale = n / sum(fib)
    counts = [max(1, int(f * scale)) for f in fib]
    counts[-1] += n - sum(counts)
    data = np.repeat(np.arange(22, dtype=np.uint8) * 11, counts)
    np.random.default_rng(seed).shuffle(data)
    return data.tobytes()


def edge_inputs():
    rng = np.random.default_rng(77)
    text = b"It was the best of times, it was the worst of times, it was the age of wisdom. " * 1000
    tile = np.tile(rng.integers(0, 120, 300, dtype=np.uint8), 60).tobytes()[:16384]   # no 'x' in it
    payload = rng.integers(0, 256, 200, dtype=np.uint8).tobytes()
    keys = rng.integers(0, 256, (316, 8), dtype=np.uint8)
    keys[:, 0] = np.arange(316) % 256
    keys[:, 7] = np.arange(316) % 251
    records = b"".join(k.tobytes() + payload for k in keys)
    far = rng.integers(0, 256, 65532, dtype=np.uint8).tobytes()
    half = rng.integers(0, 256, 10000, dtype=np.uint8).tobytes()
    skew = np.minimum(rng.geometric(0.03, 65536) - 1, 255).astype(np.uint8)
    return {
        "len0": b"",
        "len1": b"Q",
        "len255": text[:255],
        "len256": text[:256],
        "len65536": text[:65536],
        "equal65536": b"\x5a" * 65536,
        "equal300": b"\x01" * 300,
        "random65536": rng.integers(0, 256, 65536, dtype=np.uint8).tobytes(),
        "random1000": rng.integers(0, 256, 1000, dtype=np.uint8).tobytes(),
        "fibonacci": fibonacci_bytes(),
        "alphabet256": skew.tobytes(),                                  # highest literal 255: FSE weights
        "alphabet100": (skew % 100).astype(np.uint8).tobytes(),         # highest literal < 128
        "alphabet12": (rng.geometric(0.4, 65536) % 12).astype(np.uint8).tobytes(),
        "periodic": (rng.integers(0, 256, 37, dtype=np.uint8).tobytes() * 2000)[:65536],
        "periodic_mix": b"".join(rng.integers(0, 256, 8, dtype=np.uint8).tobytes() * int(k)
                                 for k in rng.integers(1, 9, 3000))[:65536],
        "rle_literals": tile + (b"xx" + tile[:16382]) * 3,              # blocks 2-4: literals "xx"
        "records": records[:65536],                                      # matches of 131-258 bytes: one ML code
        "distance65532": far + far[:4],
        "match_across_block": half + half + half[:5000],
        "text_17000": text[:17000],
    }


def golden_inputs():
    out = {}
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*.raw"))):
        with open(p, "rb") as f:
            out[os.path.basename(p)[:-4]] = f.read()
    # chunk 218 of datagen.tabular_f32(10000): a match without literals whose offset sits in two repeat slots
    with open(os.path.join(ROOT, "tests", "golden", "zstd_encode_rep_slots.bin"), "rb") as f:
        out["zstd_encode_rep_slots"] = f.read()
    return out


def corpus():
    return {**{f"sample:{k}": v for k, v in sample_inputs().items()},
            **{f"golden:{k}": v for k, v in golden_inputs().items()},
            **{f"edge:{k}": v for k, v in edge_inputs().items()}}
