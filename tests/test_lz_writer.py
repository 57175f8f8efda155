"""CPU: the hand-built LZ4 / Snappy streams of tests/lz_writer.py (shapes no encoder emits, one invalid stream per
rejection rule) and a seeded corruption corpus, pinned to the oracle, to liblz4 / pyarrow where those accept, and run
through the warp-level decoders in the host emulator -- single chunks in every mode and misalignment, chunk sequences
decoded by one warp with one ring and one mbarrier phase (as the kernels' chunk loop runs them), and the LZ4 size
query."""
import ctypes as C
import zlib

import numpy as np
import pytest

import lz_writer as W
from conftest import sample_inputs
from test_lz_emu import Emu, MODES

VALID = W.valid_streams()
INVALID = W.invalid_streams()
ALL = {**VALID, **INVALID}
BIG = 1 << 18          # streams whose output exceeds this are run at fewer misalignments in the emulator

# Streams the oracle accepts and liblz4's LZ4_decompress_safe rejects: liblz4 enforces the end-of-block rules (the last
# match starts >= 12 bytes before the end and >= 5 literal bytes follow it) relative to the output capacity, so a
# block whose final sequence is short decodes only with spare capacity (or not at all).  The oracle -- and this
# library -- follow the format's grammar (DESIGN §4).  At exact capacity:
LIBLZ4_REJECTS = {
    "lz4_edge_64-2", "lz4_edge_1024-2", "lz4_edge_1024-1", "lz4_edge_1024+0", "lz4_edge_1024+2", "lz4_edge_2048-2",
    "lz4_edge_2048+3", "lz4_end_lit_0", "lz4_final_zero_literals", "lz4_match_4", "lz4_match_18", "lz4_match_19",
    "lz4_match_274", "lz4_match_60000", "lz4_off_eq_op_1", "lz4_off_eq_op_2", "lz4_off_eq_op_9", "lz4_off_eq_op_17",
    "lz4_off_eq_op_100", "lz4_serial_match_192", "lz4_serial_match_193",
}
# Invalid streams liblz4 accepts: a match with offset 0 far enough from the block end passes its checks (the match
# source is the output position itself).  The format has no offset 0; the oracle and this library reject it.
LIBLZ4_ACCEPTS = {"lz4_off0_window"}


class SeqEmu(Emu):
    def __init__(self):
        super().__init__()
        sz, szp = C.c_size_t, C.POINTER(C.c_size_t)
        f = self.lib.emu_lz_decode_seq
        f.restype = C.c_int
        f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, szp, szp, C.c_char_p, szp, szp, C.c_uint, C.c_uint,
                      C.POINTER(C.c_longlong), C.c_char_p, sz]
        self.lib.emu_lz4_walk.restype = C.c_longlong
        self.lib.emu_lz4_walk.argtypes = [C.c_char_p, sz, C.c_uint, C.c_char_p, sz]
        self.lib.emu_lz_fails_in_flight.restype = C.c_int
        self.lib.emu_lz_fails_in_flight.argtypes = [C.c_int, C.c_char_p, sz, sz, C.c_char_p, sz]
        self.lib.emu_lz_bucket.restype = C.c_int
        self.lib.emu_lz_bucket.argtypes = [C.c_ulonglong, C.c_ulonglong]

    def decode_seq(self, codec, chunks, caps, mode="block", in_mis=0, out_mis=0):
        """[(bytes | None)] per chunk, decoded in order by one emulated warp."""
        k = len(chunks)
        arr = lambda xs: (C.c_size_t * k)(*xs)
        in_off = np.cumsum([0] + [len(c) for c in chunks])[:-1].tolist()
        out_off = np.cumsum([0] + list(caps))[:-1].tolist()
        dst = C.create_string_buffer(max(sum(caps), 1))
        prod = (C.c_longlong * k)()
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz_decode_seq(0 if codec == "lz4" else 1, MODES[mode], k, b"".join(chunks), arr(in_off),
                                       arr([len(c) for c in chunks]), dst, arr(out_off), arr(caps), in_mis, out_mis,
                                       prod, msg, 256)
        assert r != -2, f"emulator fault: {msg.value.decode()}"
        return [None if prod[i] < 0 else dst.raw[out_off[i]:out_off[i] + prod[i]] for i in range(k)]

    def fails_in_flight(self, codec, comp, cap):
        """1: the dense decoder rejects the stream with a staged-block copy in flight, 0: rejects it with none,
        2: accepts it."""
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz_fails_in_flight(0 if codec == "lz4" else 1, comp, len(comp), cap, msg, 256)
        assert r != -2, f"emulator fault: {msg.value.decode()}"
        return r

    def lz4_size(self, comp, in_mis=0):
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz4_walk(comp, len(comp), in_mis, msg, 256)
        assert r != -2, f"emulator fault: {msg.value.decode()}"
        return r


@pytest.fixture(scope="module")
def emu():
    return SeqEmu()


# Restatement of csrc/lz_sched.cuh (the GPU tests use it to steer chunks to a kernel and a cost bucket):
# lz_chunk_is_light and lz_bucket.  test_scheduler_restatement_matches_lz_sched ties it to the header.
def is_light(cap, n):
    return cap >= 4 * n or n + (cap >> 6) >= cap


def bucket(cap, n):
    if is_light(cap, n):
        return 0 if cap >= 4 * n else 1
    return 2 + 3 - min(n >> 14, 3)


def test_scheduler_restatement_matches_lz_sched(emu):
    """is_light / bucket equal lz_sched.cuh's lz_bucket (compiled from the header into the emulator library) around
    every threshold: 4x, the 1/64 incompressible margin and the 16 KB dense-bucket steps."""
    ns = {0, 1, 2, 63, 64, 65, 1000, 4095}
    for k in range(1, 6):
        ns |= {(k << 14) - 1, k << 14, (k << 14) + 1}
    for n in sorted(ns):
        caps = {0, 1, n, n + 1, 4 * n - 1, 4 * n, 4 * n + 1, 65536, 1 << 24}
        for c in range(max(n - 2, 0), n + 3):
            caps |= {c + (c >> 6), 64 * n // 63 - 1, 64 * n // 63, 64 * n // 63 + 1, 64 * n // 63 + 2}
        for cap in sorted(x for x in caps if x >= 0):
            assert emu.lib.emu_lz_bucket(cap, n) == bucket(cap, n), (cap, n)


def _oracle_size(oracle, codec, comp):
    r = oracle.size(codec, comp)
    return r if r >= 0 else -1


# ---------------------------------------------------------------------------------------------------------------------
# the writers against the oracle, liblz4 and pyarrow
# ---------------------------------------------------------------------------------------------------------------------
def test_writer_covers_the_issue_shapes():
    """The named shapes exist (a writer change that drops one fails here, not silently)."""
    for name in ("lz4_lit_0", "lz4_lit_14", "lz4_lit_15", "lz4_lit_270", "lz4_match_4", "lz4_match_18", "lz4_match_19",
                 "lz4_match_274", "lz4_match_60000", "lz4_off_1", "lz4_off_17", "lz4_off_33", "lz4_off_4097",
                 "lz4_off_65535", "lz4_final_zero_literals", "lz4_only_empty_final", "lz4_edge_1024+0",
                 "lz4_serial_lit_193", "lz4_serial_match_193", "lz4_chain_16000", "lz4_far_1mb", "lz4_far_16mb",
                 "snappy_varint_0_x4", "snappy_varint_4byte", "snappy_littag_63_1", "snappy_copy1_all",
                 "snappy_copy2_off65535", "snappy_copy4", "snappy_run_p8_k35"):
        assert name in VALID, name
    for name in ("lz4_off0", "lz4_off_op_plus_1", "lz4_ext_runs_off_end", "lz4_over_cap_by_1_literal",
                 "lz4_over_cap_by_1_match", "snappy_off0_copy2", "snappy_off_op_plus_1_copy4",
                 "snappy_preamble_larger", "snappy_preamble_smaller_match", "snappy_over_cap_by_1_literal",
                 "snappy_over_cap_by_1_match", "snappy_varint_6_bytes"):
        assert name in INVALID, name
    assert len(VALID["lz4_far_16mb"].out) > 16_000_000 and len(VALID["lz4_chain_16000"].comp) > 16000 * 3


def test_writer_streams_match_oracle(oracle):
    for name, c in VALID.items():
        n = len(c.out)
        assert oracle.decompress(c.codec, c.comp, n) == c.out, name
        assert oracle.decompress(c.codec, c.comp, n + 1) == c.out, name
        assert oracle.size(c.codec, c.comp) == n, name
        if n:
            assert oracle.decompress(c.codec, c.comp, n - 1) is None, name
    for name, c in INVALID.items():
        assert oracle.decompress(c.codec, c.comp, c.cap) is None, name


def test_writer_lz4_streams_vs_liblz4(liblz4):
    rejects = set()
    for name, c in VALID.items():
        if c.codec != "lz4":
            continue
        got = liblz4.decompress(c.comp, len(c.out))
        if got is None:
            rejects.add(name)
        else:
            assert got == c.out, name
    assert rejects == LIBLZ4_REJECTS
    accepts = {name for name, c in INVALID.items() if c.codec == "lz4" and liblz4.decompress(c.comp, c.cap) is not None}
    assert accepts == LIBLZ4_ACCEPTS


def test_writer_snappy_streams_vs_pyarrow():
    import pyarrow as pa
    codec = pa.Codec("snappy")
    for name, c in VALID.items():
        if c.codec != "snappy" or not c.out:
            continue
        assert codec.decompress(c.comp, decompressed_size=len(c.out)).to_pybytes() == c.out, name
    for name, c in INVALID.items():
        if c.codec != "snappy" or c.cap == 0:
            continue
        try:
            got = codec.decompress(c.comp, decompressed_size=c.cap).to_pybytes()
        except (OSError, pa.ArrowException):
            got = None
        assert got is None or len(got) != c.cap, name


# ---------------------------------------------------------------------------------------------------------------------
# the emulated decoders
# ---------------------------------------------------------------------------------------------------------------------
MIS = [(i, (7 * i + 3) % 16) for i in range(16)]       # every input and every output misalignment 0..15


@pytest.mark.parametrize("mode", sorted(MODES))
def test_emulator_writer_streams(emu, oracle, mode):
    """Every writer stream, valid and invalid, at every input and output misalignment: the oracle's verdict and bytes
    at its capacity; the invalid ones also at 64 KB, the valid ones also at exact - 1, at 4x the compressed size (the
    other kernel) and at 64 KB."""
    for name, c in ALL.items():
        mis = MIS if len(c.out or b"") <= BIG else MIS[:2]
        for in_mis, out_mis in mis:
            got = emu.decode(c.codec, c.comp, c.cap, mode, in_mis, out_mis)
            assert got == c.out, (name, mode, in_mis, out_mis)
        if c.out is None:
            assert emu.decode(c.codec, c.comp, 65536, mode, 5, 11) == oracle.decompress(c.codec, c.comp, 65536), name
            continue
        for cap in {max(len(c.out) - 1, 0), max(len(c.out), 4 * len(c.comp)), 65536}:
            want = oracle.decompress(c.codec, c.comp, cap)
            assert emu.decode(c.codec, c.comp, cap, mode, 5, 11) == want, (name, mode, cap)


def test_emulator_lz4_size_query(emu, oracle):
    """lz4_walk_chunk (the LZ4 size query) on every LZ4 writer stream and corrupted copies of them: the oracle's size,
    -1 where the oracle finds the block malformed."""
    rng = np.random.default_rng(3)
    for name, c in ALL.items():
        if c.codec != "lz4":
            continue
        assert emu.lz4_size(c.comp, int(rng.integers(0, 16))) == _oracle_size(oracle, "lz4", c.comp), name
        for _ in range(4):
            _, bad = W.mutate(rng, "lz4", c.comp)
            assert emu.lz4_size(bad) == _oracle_size(oracle, "lz4", bad), name


def _dense_lz4(rng, n_out=20000, bad_at=None, seed_lits=16):
    """A dense LZ4 block (short literals, short near matches: the block path), optionally with one sequence whose
    offset is op + 1 after `bad_at` output bytes."""
    w = W.Lz4().seq(rng.integers(0, 256, seed_lits, dtype=np.uint8).tobytes(), 4, 4)
    placed = False
    while len(w.out) < n_out:
        ll = int(rng.integers(0, 4))
        lits = rng.integers(0, 256, ll, dtype=np.uint8).tobytes()
        if bad_at is not None and not placed and len(w.out) >= bad_at:
            w.seq(lits, len(w.out) + ll + 1, 4)
            placed = True
            continue
        w.seq(lits, int(rng.integers(1, min(200, len(w.out)) + 1)), int(rng.integers(4, 10)))
    return w.end(b"tail!").case()


def _dense_snappy(rng, n_out=20000, bad_at=None):
    s = W.Snappy().lit(rng.integers(0, 256, 16, dtype=np.uint8).tobytes())
    placed = False
    while len(s.out) < n_out:
        if bad_at is not None and not placed and len(s.out) >= bad_at:
            s.copy1(min(len(s.out) + 1, 2047), 4) if len(s.out) < 2047 else s.copy2(len(s.out) + 1, 4)
            placed = True
            continue
        s.lit(rng.integers(0, 256, int(rng.integers(1, 4)), dtype=np.uint8).tobytes())
        s.copy1(int(rng.integers(1, min(2047, len(s.out)) + 1)), int(rng.integers(4, 12)))
    return s.case()


@pytest.mark.parametrize("codec", ["lz4", "snappy"])
@pytest.mark.parametrize("mode", ["adaptive", "block"])
def test_emulator_chunk_sequence_after_failure(emu, oracle, codec, mode):
    """One warp decodes a run of chunks with one ring, one mbarrier and one tma_parity.  Chunks that fail in the middle
    of a staged block -- a bad offset or the capacity running out while the next block's copy is in flight -- must
    leave the phase right for the valid chunk behind them (lz_decode_stream drains the copy)."""
    rng = np.random.default_rng(17)
    make = _dense_lz4 if codec == "lz4" else _dense_snappy
    chunks, caps = [], []
    for k in range(6):
        good = make(rng)
        bad = make(rng, bad_at=int(rng.integers(3000, 15000)))
        assert bad.out is None and good.out is not None
        chunks += [good.comp, bad.comp, good.comp]
        caps += [len(good.out), len(good.out) * 2, len(good.out) - int(rng.integers(1, 9000))]   # last: over capacity
    chunks += [VALID[f"{codec}_dense_far" if codec == "lz4" else "snappy_dense_mixed"].comp]
    caps += [len(VALID["lz4_dense_far" if codec == "lz4" else "snappy_dense_mixed"].out)]
    want = [oracle.decompress(codec, c, cap) for c, cap in zip(chunks, caps)]
    assert sum(w is None for w in want) == 12
    # the failing chunks really fail with the next block's copy in flight (what lz_decode_stream must drain)
    in_flight = [emu.fails_in_flight(codec, c, cap) for c, cap, w in zip(chunks, caps, want) if w is None]
    assert in_flight.count(1) >= 6, in_flight
    for in_mis, out_mis in [(0, 0), (3, 9), (15, 1)]:
        got = emu.decode_seq(codec, chunks, caps, mode, in_mis, out_mis)
        for i, (g, w) in enumerate(zip(got, want)):
            assert g == w, (i, in_mis, out_mis)


# ---------------------------------------------------------------------------------------------------------------------
# corruption corpus
# ---------------------------------------------------------------------------------------------------------------------
def cpu_producers(oracle, liblz4):
    import pyarrow as pa
    snap = pa.Codec("snappy")
    return {
        ("lz4", "liblz4"): liblz4.compress,
        ("lz4", "lz4hc12"): lambda d: liblz4.compress(d, 12),
        ("lz4", "oracle"): lambda d: oracle.compress("lz4", d),
        ("snappy", "oracle"): lambda d: oracle.compress("snappy", d),
        ("snappy", "pyarrow"): lambda d: snap.compress(d).to_pybytes() if d else b"\x00",
    }


def corpus_inputs():
    from nvcomp_b200 import datagen
    ins = list(sample_inputs().values())
    for name in ("runlength_i32", "tabular_f32", "snappy_synth", "lz4_mixed", "lowentropy_bytes", "sorted_i64"):
        ins += [r.tobytes() for r in datagen.DATASETS[name](2)]
    return ins


def test_emulator_corruption_corpus(emu, oracle, liblz4):
    """4000 seeded corruptions of producer streams (bit flips, truncations, appended bytes, single-byte inserts and
    deletes, rewritten Snappy preambles): the oracle's verdict and bytes, and the
    oracle's size from the LZ4 size query, at the capacities the GPU test uses (lz_writer.corpus_cap)."""
    corpus = W.corruption_corpus(cpu_producers(oracle, liblz4), corpus_inputs())
    assert len(corpus) == 4000
    kinds = {}
    for i, (codec, prod, kind, comp, n) in enumerate(corpus):
        kinds[kind] = kinds.get(kind, 0) + 1
        cap = W.corpus_cap(i, comp, n)
        want = oracle.decompress(codec, comp, cap)
        mode = ("adaptive", "block", "direct")[i % 3]
        got = emu.decode(codec, comp, cap, mode, i % 16, (i * 5) % 16)
        assert got == want, (i, codec, prod, kind, mode, zlib.crc32(comp))
        if codec == "lz4" and i % 4 == 1:
            assert emu.lz4_size(comp) == _oracle_size(oracle, "lz4", comp), (i, prod, kind)
    assert min(kinds.values()) > 200 and len(kinds) == 6, kinds
