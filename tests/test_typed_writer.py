"""CPU: the hand-built typed streams (tests/typed_writer.py) against the oracle, the writer against the encoders, and the
corruption campaign's mutator.  tests/test_typed_oracle_gpu.py runs the same streams on the GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import typed_model as tm
import typed_writer as W

CODECS = ("cascaded", "bitcomp", "ans")


@pytest.mark.parametrize("name", sorted(W.VALID))
def test_valid_case_decodes_to_its_bytes(oracle, name):
    c = W.VALID[name]
    assert oracle.decompress(c.codec, c.comp, c.cap) == c.out
    assert oracle.size(c.codec, c.comp) == len(c.out)
    if c.out:
        assert oracle.decompress(c.codec, c.comp, c.cap - 1) is None


@pytest.mark.parametrize("name", sorted(W.INVALID))
def test_invalid_case_is_rejected(oracle, name):
    c = W.INVALID[name]
    assert oracle.decompress(c.codec, c.comp, c.cap) is None


def test_every_codec_has_cases():
    for codec in CODECS:
        assert sum(c.codec == codec for c in W.VALID.values()) >= 8, codec
        assert sum(c.codec == codec for c in W.INVALID.values()) >= 14, codec
        assert any(c.header for c in W.INVALID.values() if c.codec == codec), codec
        assert any(not c.header for c in W.INVALID.values() if c.codec == codec), codec


def test_run_length_table(oracle):
    """The control chunk (INT, R=1, D=0, one partition, values {5, 7}) decodes to [5, 5, 5, 7]; a zero-length run, a
    run minimum of 2^32 + 2 and lengths that wrap 32 bits are rejected."""
    ctl = W.VALID["csc_control"]
    assert oracle.decompress("cascaded", ctl.comp, 16) == np.array([5, 5, 5, 7], np.uint32).tobytes()
    for name in ("csc_run_zero_length", "csc_run_min_above_capacity", "csc_run_length_wraps_32"):
        assert oracle.decompress("cascaded", W.INVALID[name].comp, 64) is None, name
        assert oracle.decompress("cascaded", W.INVALID[name + "_layer1"].comp, 64) is None, name


@pytest.mark.parametrize("type_id", sorted(tm.TYPE_SIZE))
@pytest.mark.parametrize("layers", [(0, 0, 1), (1, 0, 1), (1, 1, 1), (2, 1, 0), (3, 2, 1), (0, 2, 1)])
def test_writer_reproduces_cascaded_encoder(oracle, type_id, layers):
    R, D, bp = layers
    for part in (512, 4096):
        for name, raw in tm.edge_chunks(type_id, part):
            want = oracle.compress_typed("cascaded", raw, chunk_size=part, type=type_id, num_RLEs=R, num_deltas=D,
                                         use_bp=bp)
            assert W.cascaded_from_fields(raw, type_id, part, R, D, bp) == want, (name, part)


@pytest.mark.parametrize("type_id", sorted(tm.TYPE_SIZE))
@pytest.mark.parametrize("algo", [0, 1])
def test_writer_reproduces_bitcomp_encoder(oracle, type_id, algo):
    for name, raw in tm.bitcomp_edge_chunks(type_id):
        assert W.bitcomp_from_fields(raw, algo, type_id) == oracle.compress_typed("bitcomp", raw, algo=algo,
                                                                                  type=type_id), name


def test_writer_reproduces_ans_encoder(oracle):
    for name, raw in tm.ans_edge_chunks(big=False):
        assert W.ans_from_fields(raw) == oracle.compress_typed("ans", raw), name


@pytest.fixture(scope="module")
def sources():
    return W.campaign_sources()


@pytest.mark.parametrize("codec", CODECS)
def test_mutator_is_seeded_and_reaches_every_field_class(sources, codec):
    """The campaign the GPU test runs: the same streams for the same seed, different ones for another, and every field
    class of the format hit many times."""
    a = W.corruption_campaign(sources, codec)
    assert a == W.corruption_campaign(sources, codec)
    assert [x[2] for x in a[:50]] != [x[2] for x in W.corruption_campaign(sources, codec, seed=6)[:50]]
    counts = {k: sum(x[1] == k for x in a) for k in W.CLASSES[codec]}
    assert min(counts.values()) >= 50, counts
    srcs = {s[0] for s in sources[codec]}
    assert len({x[0] for x in a}) >= min(len(srcs), 100)


def _oracle_rules():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "typed_oracle.c")).read()
    return set(re.findall(r'broken\("(\w+)"', src))


def test_every_oracle_rule_has_a_case():
    """Each rejection rule of the typed oracle is what an invalid case breaks (alone, or with the rules it implies)."""
    rules = _oracle_rules()
    named = {r for c in W.INVALID.values() for r in c.rules}
    assert named <= rules, named - rules
    assert rules <= named, rules - named


@pytest.mark.parametrize("name", sorted(n for n, c in W.INVALID.items() if c.rules))
def test_invalid_case_breaks_only_its_rules(oracle, name):
    """With the case's rules skipped and its missing bytes present past its end, the oracle decodes it: no other rule
    rejects it; with any one of them applied it is rejected.  (The stream and output buffers get room for what a
    rule-less decode reads and writes.)"""
    c = W.INVALID[name]
    buf = C.create_string_buffer(c.comp + c.beyond + bytes(1 << 20), len(c.comp) + len(c.beyond) + (1 << 20))
    out = C.create_string_buffer(c.cap + (1 << 21))
    fn = getattr(oracle.lib, f"oracle_{c.codec}_decompress")
    assert fn(buf, len(c.comp), out, c.cap) < 0
    try:
        for k in range(len(c.rules) + 1):       # all its rules skipped: decodes; any one of them kept: rejected
            skip = [r for i, r in enumerate(c.rules) if i != k]
            names = C.create_string_buffer(",".join(skip).encode())  # the oracle keeps the pointer: keep it alive
            oracle.lib.oracle_typed_skip_rules(names)
            r = fn(buf, len(c.comp), out, c.cap)
            assert (r >= 0) == (k == len(c.rules)), (skip, r)
    finally:
        oracle.lib.oracle_typed_skip_rules(None)
