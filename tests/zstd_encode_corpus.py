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
        self.lib.emu_zstd_parse.restype = C.c_long
        self.lib.emu_zstd_parse.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]

    def bound(self, n: int) -> int:
        return self.lib.emu_zstd_enc_bound(n)

    def parse(self, data: bytes):
        """The matcher's parse with the encoder's arguments, before block cutting:
        [(literal run, offset, length), ..., (trailing literals, 0, 0)]."""
        cap = 3 * (len(data) // 4 + 2)
        t = (C.c_uint32 * cap)()
        msg = C.create_string_buffer(256)
        r = self.lib.emu_zstd_parse(data, len(data), t, cap, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        assert 0 < r <= cap, r
        return [tuple(t[i:i + 3]) for i in range(0, r, 3)]

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


def literal_run(m, seed, n=8192):
    """m random bytes, then their last 64 bytes repeated up to n: one literal run, then one long match."""
    y = np.random.default_rng(seed).integers(0, 256, m, dtype=np.uint8).tobytes()
    return (y + y[-64:] * (n // 64 + 1))[:n]


def short_runs(c, a, last, seed):
    """64 random bytes, then c pieces of `a` random literals (`last` in the final piece) and an 8-byte copy from the
    first 64 bytes: about one sequence per piece."""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 256, 64, dtype=np.uint8)
    parts = [r.tobytes()]
    for i in range(c):
        j = int(rng.integers(0, 56))
        parts.append(rng.integers(0, 256, a if i < c - 1 else last, dtype=np.uint8).tobytes() + r[j:j + 8].tobytes())
    return b"".join(parts)


def copy_pieces(c, seed):
    """256 random bytes, then c pieces of one random literal and an 8-byte copy from them."""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 256, 256, dtype=np.uint8)
    parts = [r.tobytes()]
    for _ in range(c):
        j = int(rng.integers(0, 240))
        parts.append(bytes([int(rng.integers(0, 256))]) + r[j:j + 8].tobytes())
    parts.append(rng.integers(0, 256, 16, dtype=np.uint8).tobytes())
    return b"".join(parts)


def tail_repeat(n, k, seed):
    """n random bytes whose last k repeat the first k."""
    y = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()
    return y[:n - k] + y[:k]


def skewed_literals(seed, n=400):
    """n bytes from a geometric distribution over a random subset of the symbols below 128."""
    rng = np.random.default_rng(seed)
    nsym = int(rng.integers(3, 40))
    syms = rng.choice(int(rng.integers(nsym, 128)), nsym, replace=False)
    p = rng.geometric(float(rng.uniform(0.05, 0.5)), n) % nsym
    return syms[p].astype(np.uint8).tobytes()


def one_literal_block():
    """Block 1: 1 000 random bytes, then "ab" repeated; block 2: the byte that ends that match, then the 1 000 bytes
    again: its literals section holds exactly one literal."""
    r = np.random.default_rng(5).integers(0, 256, 1000, dtype=np.uint8).tobytes()
    return r + (b"ab" * 9000)[:16384 - 1000] + b"a" + r


def boundary_inputs():
    """Inputs whose first block sits on one side of a stream-rule boundary (the seeds and sizes were searched for
    with the matcher and tests/zstd_encode_model.py; tests/test_zstd_encode_model.py asserts each boundary is hit)."""
    rng = np.random.default_rng(1)
    raw_first = bytearray(rng.integers(0, 256, 16384, dtype=np.uint8).tobytes())
    raw_first[9000:9005] = raw_first[100:105]          # a 5-byte match that does not pay for itself
    raw_then_repeat = (bytes(raw_first) + rng.integers(0, 256, 40, dtype=np.uint8).tobytes() + bytes([7]) * 200 +
                       rng.integers(0, 256, 40, dtype=np.uint8).tobytes())
    return {
        "raw_lits31": literal_run(31, 31),                        # Raw literals, 1-byte header
        "raw_lits32": literal_run(32, 32),                        # 2-byte header
        "raw_lits4095": short_runs(160, 25, 14, 4095),            # 2-byte header
        "raw_lits4096": short_runs(158, 25, 46, 4096),            # 3-byte header
        "huf_lits255": (np.random.default_rng(1000).integers(0, 32, 255, dtype=np.uint8).tobytes() * 9)[:2048],
        "huf_lits256": (np.random.default_rng(1000).integers(0, 32, 256, dtype=np.uint8).tobytes() * 8)[:2048],
        "huf_lits16384": np.random.default_rng(0).integers(0, 128, 16384, dtype=np.uint8).tobytes(),   # no match
        "nseq127": copy_pieces(114, 7),
        "nseq128": copy_pieces(115, 7),
        "body_block_minus1": tail_repeat(600, 10, 0),             # Compressed body of 599 bytes
        "body_equals_block": tail_repeat(600, 8, 162),            # Compressed body of 600 bytes: Raw
        "raw_then_repeat": raw_then_repeat,
        "one_literal_block": one_literal_block(),                 # Raw and RLE literals of the same size
        "weights_tie": skewed_literals(242),                      # direct and FSE weights of the same size
        "table_cost_tie": copy_pieces(6, 1),                      # ML: Predefined and FSE of the same cost
        # 4 sequences, OF codes 0, 0, 0, 1: an FSE table at accuracy log 5
        "fse_four_sequences": b"abx" + b"x" * 20 + b"cdy" + b"y" * 20 + b"efz" + b"z" * 20 + b"gh" + b"klmn" * 6 +
                              b"pqrstuvw",
    }


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
        **boundary_inputs(),
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
