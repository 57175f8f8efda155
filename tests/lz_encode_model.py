"""A plain model of the LZ4 and Snappy streams the warp-per-chunk matcher writes (include/nvcomp/device/detail/
lz77_compress.cuh with lz4_encode.cuh / snappy_encode.cuh), and the emulated encoder those headers run in.

check_lz4 / check_snappy parse a stream back into (literal run, offset, length) sequences and hold it to the
encoder's rules:
  - every offset is in [1, min(position, 65535)], every match is >= 4 bytes and equal to its source;
  - LZ4: a match starts before n - 12 and ends at or before n - 5; Snappy: a match starts before n - 4;
  - every match is maximal: it stops at the first mismatch or at the end limit, rounded down to a multiple of the
    candidate stride s (the LZ4 data_type: 1, 2 or 4 bytes), and its start, length and offset are multiples of s;
  - Snappy: the preamble varint is n.
Then they write the sequences again with a restatement of each emitter, and that must be the stream byte for byte:
for LZ4 the token nibbles, the 255-runs and the final literal-only sequence; for Snappy the literal tag forms, copy-1
for lengths 4-11 at offsets < 2048 and copy-2 otherwise, 64-byte copies for long matches and the 60-byte tail split."""
import ctypes as C
import glob
import os
import subprocess

import numpy as np

from conftest import ROOT, sample_inputs

FAULT = -2
MAX_OFFSET = 65535
CODEC = {"lz4": 0, "snappy": 1}


def lz4_bound(n: int) -> int:
    return n + n // 255 + 16


def snappy_bound(n: int) -> int:
    return 32 + n + n // 6


BOUND = {"lz4": lz4_bound, "snappy": snappy_bound}


# (kind, candidate stride): LZ4 at every data_type stride, Snappy at 1
VARIANTS = [("lz4", 1), ("lz4", 2), ("lz4", 4), ("snappy", 1)]


class EmuLzEncoder:
    """The matcher and both emitters in the host warp emulator (tests/emu/emu_lz_encode.cpp)."""

    def __init__(self):
        subprocess.run(["make", "-C", ROOT, "tests/emu/libemu_lz.so"], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "libemu_lz.so"))
        self.lib.emu_lz_compress.restype = C.c_long
        self.lib.emu_lz_compress.argtypes = [C.c_int, C.c_uint, C.c_char_p, C.c_size_t, C.c_uint, C.c_uint,
                                             C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        self.lib.emu_lz_parse.restype = C.c_long
        self.lib.emu_lz_parse.argtypes = [C.c_int, C.c_uint, C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                          C.c_char_p, C.c_size_t]

    def compress(self, kind: str, data: bytes, step: int = 1, in_mis: int = 0, out_mis: int = 0) -> bytes:
        """One stream into a buffer of exactly the codec's bound; the emulator also checks that nothing past the
        stream was written."""
        cap = BOUND[kind](len(data))
        out = C.create_string_buffer(cap)
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz_compress(CODEC[kind], step, data, len(data), in_mis, out_mis, out, cap, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        return out.raw[:r]

    def parse(self, kind: str, data: bytes, step: int = 1):
        """The matcher's parse: [(literal run, offset, length), ..., (trailing literals, 0, 0)]."""
        cap = 3 * (len(data) // 4 + 2)
        t = (C.c_uint32 * cap)()
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz_parse(CODEC[kind], step, data, len(data), t, cap, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        assert 0 < r <= cap, r
        return [tuple(t[i:i + 3]) for i in range(0, r, 3)]


# ---------------------------------------------------------------------------------------------------------------------
# stream -> sequences
# ---------------------------------------------------------------------------------------------------------------------
def _lz4_len(s: bytes, i: int, base: int):
    """A 4-bit length field of value `base`, followed by 255-runs when it is 15."""
    n = base
    if base == 15:
        while True:
            assert i < len(s), "length run past the end of the block"
            b = s[i]
            i += 1
            n += b
            if b != 255:
                break
    return n, i


def parse_lz4(s: bytes):
    """An LZ4 block -> [(literal run, offset, length), ..., (trailing literals, 0, 0)]."""
    seqs, i = [], 0
    while True:
        assert i < len(s), "block ends without a literal-only sequence"
        tok = s[i]
        i += 1
        ll, i = _lz4_len(s, i, tok >> 4)
        i += ll
        assert i <= len(s), "literals past the end of the block"
        if i == len(s):
            assert tok & 15 == 0, "the last sequence has a match length"
            seqs.append((ll, 0, 0))
            return seqs
        assert i + 2 <= len(s), "offset past the end of the block"
        off = s[i] | (s[i + 1] << 8)
        i += 2
        ml, i = _lz4_len(s, i, tok & 15)
        seqs.append((ll, off, ml + 4))


def _varint(s: bytes):
    v, i = 0, 0
    while True:
        b = s[i]
        v |= (b & 127) << (7 * i)
        i += 1
        if b < 128:
            return v, i


def parse_snappy(s: bytes):
    """A Snappy stream -> (preamble length, [(literal run, offset, length), ..., (trailing literals, 0, 0)]).
    Consecutive copies at one offset with no literal between are one match: the encoder splits only long matches,
    and a maximal match is never followed by another at its own offset."""
    n, i = _varint(s)
    seqs, ll = [], 0
    while i < len(s):
        tag = s[i]
        kind = tag & 3
        if kind == 0:
            m = tag >> 2
            i += 1
            if m >= 60:
                nb = m - 59
                m = int.from_bytes(s[i:i + nb], "little")
                i += nb
            ll += m + 1
            i += m + 1
            assert i <= len(s), "literal past the end of the stream"
            continue
        if kind == 1:
            length, off = 4 + ((tag >> 2) & 7), ((tag >> 5) << 8) | s[i + 1]
            i += 2
        elif kind == 2:
            length, off = 1 + (tag >> 2), s[i + 1] | (s[i + 2] << 8)
            i += 3
        else:
            raise AssertionError("copy-4 element: the encoder never writes one")
        assert i <= len(s), "copy past the end of the stream"
        if ll == 0 and seqs and seqs[-1][1] == off:
            seqs[-1] = (seqs[-1][0], off, seqs[-1][2] + length)
        else:
            seqs.append((ll, off, length))
        ll = 0
    seqs.append((ll, 0, 0))
    return n, seqs


# ---------------------------------------------------------------------------------------------------------------------
# sequences -> stream (each emitter restated)
# ---------------------------------------------------------------------------------------------------------------------
def _lz4_ext(rem: int) -> bytes:
    return b"\xff" * (rem // 255) + bytes([rem % 255])


def emit_lz4(data: bytes, seqs) -> bytes:
    out, pos = bytearray(), 0
    for ll, off, ml in seqs:
        mc = ml - 4 if ml else 0
        out.append((min(ll, 15) << 4) | min(mc, 15))
        if ll >= 15:
            out += _lz4_ext(ll - 15)
        out += data[pos:pos + ll]
        pos += ll + ml
        if ml:
            out += bytes([off & 255, off >> 8])
            if mc >= 15:
                out += _lz4_ext(mc - 15)
    return bytes(out)


def _snappy_copy(off: int, length: int) -> bytes:
    if 4 <= length < 12 and off < 2048:
        return bytes([1 | ((length - 4) << 2) | ((off >> 8) << 5), off & 255])
    return bytes([2 | ((length - 1) << 2), off & 255, off >> 8])


def emit_snappy(data: bytes, seqs) -> bytes:
    n = len(data)
    out = bytearray()
    while n >= 128:
        out.append((n & 127) | 128)
        n >>= 7
    out.append(n)
    pos = 0
    for ll, off, ml in seqs:
        if ll:
            m = ll - 1
            if m < 60:
                out.append(m << 2)
            else:
                nb = (m.bit_length() + 7) // 8
                out.append((59 + nb) << 2)
                out += m.to_bytes(nb, "little")
            out += data[pos:pos + ll]
        pos += ll + ml
        while ml > 67:             # 64-byte copies until 4..67 bytes are left
            out += _snappy_copy(off, 64)
            ml -= 64
        if ml > 64:                # 65..67: 60 bytes, then 5..7
            out += _snappy_copy(off, 60)
            ml -= 60
        if ml:
            out += _snappy_copy(off, ml)
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# the rules
# ---------------------------------------------------------------------------------------------------------------------
def _common_len(data: bytes, p: int, c: int, limit: int) -> int:
    """Bytes from p equal to the bytes from c (c < p, so an overlapping source reads the input itself), up to limit."""
    n = 0
    while p + n + 64 <= limit and data[p + n:p + n + 64] == data[c + n:c + n + 64]:
        n += 64
    while p + n < limit and data[p + n] == data[c + n]:
        n += 1
    return n


def check_sequences(data: bytes, seqs, start_limit: int, tail_literals: int, step: int = 1) -> None:
    """The matcher's rules for a parse of `data`: a match starts at p < n - start_limit and ends at or before
    n - tail_literals."""
    n = len(data)
    assert seqs and seqs[-1][1:] == (0, 0), "the parse ends with its trailing literals"
    pos = 0
    for k, (ll, off, ml) in enumerate(seqs[:-1]):
        p = pos + ll
        tag = f"sequence {k} at {p}: literals {ll}, offset {off}, length {ml}"
        assert 1 <= off <= min(p, MAX_OFFSET), tag
        assert ml >= 4, tag
        assert p < n - start_limit, tag
        assert p + ml <= n - tail_literals, tag
        full = _common_len(data, p, p - off, n - tail_literals)
        assert full >= ml, f"{tag}: bytes differ from the source after {full}"
        assert ml == full - full % step, f"{tag}: not maximal (the bytes agree for {full})"
        assert p % step == 0 and off % step == 0, f"{tag}: not aligned to the stride {step}"
        pos = p + ml
    assert pos + seqs[-1][0] == n, "the parse does not cover the input"


def check_lz4(stream: bytes, data: bytes, step: int = 1):
    """Hold an LZ4 block of `data` to the encoder's rules; returns its sequences."""
    seqs = parse_lz4(stream)
    check_sequences(data, seqs, 12, 5, step)
    assert emit_lz4(data, seqs) == stream, "the LZ4 emitter restated writes other bytes"
    return seqs


def check_snappy(stream: bytes, data: bytes):
    """Hold a Snappy stream of `data` to the encoder's rules; returns its sequences."""
    n, seqs = parse_snappy(stream)
    assert n == len(data), f"preamble says {n} bytes, the input has {len(data)}"
    check_sequences(data, seqs, 4, 0, 1)
    assert emit_snappy(data, seqs) == stream, "the Snappy emitter restated writes other bytes"
    return seqs


def check(kind: str, stream: bytes, data: bytes, step: int = 1):
    return check_lz4(stream, data, step) if kind == "lz4" else check_snappy(stream, data)


# ---------------------------------------------------------------------------------------------------------------------
# the inputs the emulated and the GPU encoders share
# ---------------------------------------------------------------------------------------------------------------------
def period_input(period: int, seed: int = 41) -> bytes:
    """Random bytes that repeat with the given period for 4 096 bytes more: a match at offset `period` if it is
    <= 65 535, and nothing to match otherwise."""
    block = np.random.default_rng(seed + period).integers(0, 256, period, dtype=np.uint8).tobytes()
    return block + block[:4096]


def corpus():
    """name -> bytes: the sample and golden inputs, a 64 KB slice of every datagen dataset, the sizes 0-80 (a
    period-5 pattern, so the end-of-chunk limits bind), 4 095-4 097, 65 535-65 537 and 2^17 +- 1 (slices of the
    datasets), and periods 65 534-65 537 around the largest offset."""
    from nvcomp_b200 import datagen
    out = {f"sample:{k}": v for k, v in sample_inputs().items()}
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*.raw"))):
        with open(p, "rb") as f:
            out[f"golden:{os.path.basename(p)[:-4]}"] = f.read()
    mixed = b""
    for name, gen in datagen.DATASETS.items():
        raw = gen(3)[1:].tobytes()
        out[f"slice:{name}"] = raw[:65536]
        mixed += raw[:32768]
    for n in range(81):
        out[f"size:{n}"] = (b"vwxyz" * 17)[:n]
    for n in (4095, 4096, 4097, 65535, 65536, 65537, (1 << 17) - 1, (1 << 17) + 1):
        out[f"size:{n}"] = (mixed * 2)[:n]
    for period in (65534, 65535, 65536, 65537):
        out[f"period:{period}"] = period_input(period)
    return out
