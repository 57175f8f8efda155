"""CPU: the warp-level Deflate / Gzip decoder of nvcomp_b200/csrc (inflate_decode.cuh) executed in the host warp
emulator (tests/emu: 32 fibers, rendezvous at every warp intrinsic, bounds-checked shared and vector accesses, guard
pages around the global buffers), with zlib as the oracle.  The hand-built streams of tests/deflate_writer.py are
pinned to zlib first, so every verdict here is zlib's."""
import ctypes as C
import os
import subprocess
import zlib

import pytest

import deflate_writer as W
from conftest import ROOT, sample_inputs

INPUTS = sample_inputs()
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}
BAD, FAULT, CHECKSUM = -1, -2, -3


class Emu:
    def __init__(self):
        subprocess.run(["make", "-C", ROOT, "tests/emu/libemu_lz.so"], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "libemu_lz.so"))
        self.lib.emu_inflate.restype = C.c_int
        self.lib.emu_inflate.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint,
                                         C.c_uint, C.c_int, C.c_char_p, C.c_size_t]

    def run(self, gz: bool, comp: bytes, cap: int, count_only=False, in_mis=0, out_mis=0, reps=1):
        """bytes on success, else BAD / CHECKSUM (count_only: the decoded length or BAD)."""
        out = C.create_string_buffer(max(cap, 1))
        msg = C.create_string_buffer(256)
        r = self.lib.emu_inflate(int(gz), int(count_only), comp, len(comp), out, cap, in_mis, out_mis, reps, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        if r < 0 or count_only:
            return r
        return out.raw[:r]


@pytest.fixture(scope="module")
def emu():
    return Emu()


def _check(emu, gz, comp, cap, **kw):
    """The emulated decoder's verdict and bytes equal zlib's."""
    verdict, want = W.zlib_expect(comp, gz, cap)
    got = emu.run(gz, comp, cap, **kw)
    if verdict == "ok":
        assert got == want
    else:
        assert got == (CHECKSUM if verdict == "checksum" else BAD), verdict


# 1. the writer is pinned to zlib
def test_writer_valid_streams_pinned_to_zlib():
    for name, s, want in W.valid_streams():
        assert W.zlib_expect(s, False, len(want)) == ("ok", want), name
    for name, s, want in W.gzip_streams():
        assert W.zlib_expect(s, True, len(want)) == ("ok", want), name


def test_writer_invalid_streams_pinned_to_zlib():
    for rule, s in W.invalid_streams():
        assert W.zlib_expect(s, False, 1 << 20)[0] == "bad", rule
    for rule, s, verdict in W.invalid_gzip():
        assert W.zlib_expect(s, True, 1 << 20)[0] == verdict, rule


def test_writer_code284_extra31_verdict():
    """Length code 284 with extra value 31 spells 258 (zlib's encoder uses 285 for it): zlib 1.3 accepts it."""
    s, want = W.code284_extra31()
    assert W.zlib_expect(s, False, len(want)) == ("ok", want)
    assert want[-258:] == bytes([5]) * 258


# 2. zlib's own streams
@pytest.mark.parametrize("name", sorted(INPUTS))
def test_emulated_decoder_matches_zlib(emu, name):
    data = INPUTS[name]
    for gz in (False, True):
        for level in (0, 1, 6, 9):
            for strategy in STRATEGIES.values():
                for mem_level in (1, 9):
                    comp = W.compress(data, gz, level, strategy, mem_level)
                    assert emu.run(gz, comp, len(data)) == data, (gz, level, strategy, mem_level)


def test_emulated_decoder_flush_points(emu):
    """Z_SYNC_FLUSH / Z_FULL_FLUSH end a block and add an empty stored block."""
    for name in ("text", "price_walk", "random_64k", "zeros_64k"):
        data = INPUTS[name]
        n = len(data)
        for mode in (zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
            flushes = [(0, mode), (n // 3, mode), (n // 3, mode), (n // 2 + 7, mode), (n, mode)]
            for gz in (False, True):
                for level in (1, 6):
                    comp = W.compress(data, gz, level, flushes=flushes)
                    assert emu.run(gz, comp, n) == data, (name, mode, gz, level)


# 3. alignment, capacity, size query
@pytest.mark.parametrize("mis", [0, 1, 7, 15])
def test_emulated_decoder_misaligned_buffers(emu, mis):
    for name in ("text", "price_walk", "period7", "random_777", "runlength_i32"):
        data = INPUTS[name]
        for gz in (False, True):
            for level in (0, 6):
                comp = W.compress(data, gz, level)
                assert emu.run(gz, comp, len(data), in_mis=mis, out_mis=(mis * 5) % 16) == data
                assert emu.run(gz, comp, len(data), in_mis=(mis * 3) % 16, out_mis=mis) == data


def test_emulated_decoder_capacity_and_size_query(emu):
    for name in ("one", "text", "zeros_64k", "random_64k", "sensor", "ragged_40001"):
        data = INPUTS[name]
        for gz in (False, True):
            for level in (0, 1, 9):
                comp = W.compress(data, gz, level)
                assert emu.run(gz, comp, len(data)) == data
                assert emu.run(gz, comp, len(data) - 1) == BAD
                assert emu.run(gz, comp, 0, count_only=True) == len(data)
    assert emu.run(False, W.compress(b"", False), 0) == b""
    assert emu.run(True, W.compress(b"", True), 0) == b""


# 4. hand-built edge streams
def test_emulated_decoder_edge_streams(emu):
    for name, s, want in W.valid_streams():
        assert emu.run(False, s, len(want)) == want, name
        assert emu.run(False, s, len(want), reps=2) == want, name         # fixed tables reused by the warp
        assert emu.run(False, s, 0, count_only=True) == len(want), name
        assert emu.run(False, s + b"\xff\x00junk", len(want) + 5) == want, name
        gz = W.gzip_member(s, want, name=b"edge")
        assert emu.run(True, gz, len(want)) == want, name
    s, want = W.code284_extra31()
    assert emu.run(False, s, len(want)) == want
    for name, s, want in W.gzip_streams():
        assert emu.run(True, s, len(want)) == want, name
        assert emu.run(True, s, 0, count_only=True) == len(want), name


def test_emulated_decoder_rejections(emu):
    for rule, s in W.invalid_streams():
        assert emu.run(False, s, 1 << 16) == BAD, rule
        assert emu.run(False, s, 0, count_only=True) == BAD, rule
    for rule, s, verdict in W.invalid_gzip():
        want = CHECKSUM if verdict == "checksum" else BAD
        assert emu.run(True, s, 1 << 16) == want, rule
        # the size query cannot check the CRC-32 (it produces no bytes), but it checks ISIZE
        size = emu.run(True, s, 0, count_only=True)
        if rule == "bad_crc":
            assert size == 3000, rule
        else:
            assert size == BAD, rule


# 5. corruption campaign
def test_emulated_decoder_corruption_campaign(emu):
    """3000 seeded corruptions of zlib streams: the emulated decoder gives zlib's verdict (and bytes when accepted),
    with no emulator fault and no access outside the buffers."""
    corpus = W.corruption_corpus(2024, 3000)
    for i, (gz, s, cap) in enumerate(corpus):
        _check(emu, gz, s, cap, in_mis=i % 16, out_mis=(i * 7) % 16)
