"""CPU: the oracle's Cascaded / Bitcomp / ANS encoders agree with the plain reference model in typed_model.py on every
edge input, for every element type and a spread of layer / partition options.  The oracle writes into a buffer full
of 0xA5 here, so a byte it leaves unwritten (a pad, a stream's last word) shows up as a mismatch."""
import ctypes as C

import pytest

import typed_model as tm

TYPES = sorted(tm.TYPE_SIZE)
LAYERS = [(0, 0), (1, 0), (0, 1), (1, 1), (2, 1), (1, 2), (3, 2), (0, 7), (7, 0), (7, 7)]
PARTS = [512, 520, 1000, 8192, 16384]


def oracle_compress(oracle, kind: str, data: bytes, **kw) -> bytes:
    """oracle.compress_typed() into a buffer pre-filled with 0xA5 instead of zeros."""
    cap = 24 * len(data) + 262144
    out = C.create_string_buffer(b"\xa5" * cap, cap)
    lib = oracle.lib
    if kind == "cascaded":
        r = lib.oracle_cascaded_compress(data, len(data), out, cap, kw["chunk_size"], kw["type"], kw["num_RLEs"],
                                         kw["num_deltas"], kw["use_bp"])
    elif kind == "bitcomp":
        r = lib.oracle_bitcomp_compress(data, len(data), out, cap, kw["algo"], kw["type"])
    else:
        r = lib.oracle_ans_compress(data, len(data), out, cap)
    assert r >= 0, (kind, kw)
    return out.raw[:r]


def _check_cascaded(oracle, chunks, type_id, part, r, d, bp):
    kw = dict(chunk_size=part, type=type_id, num_RLEs=r, num_deltas=d, use_bp=bp)
    for name, data in chunks:
        s = oracle_compress(oracle, "cascaded", data, **kw)
        want = tm.cascaded_model(data, type_id, part, r, d, bp)
        got = tm.parse_cascaded(s)
        assert len(s) == want["size"], (name, kw)
        assert got == want, (name, kw)
        assert oracle.decompress("cascaded", s, len(data)) == data, (name, kw)


@pytest.mark.parametrize("bp", [0, 1])
@pytest.mark.parametrize("layers", LAYERS)
@pytest.mark.parametrize("type_id", TYPES)
def test_cascaded_oracle_matches_model(oracle, type_id, layers, bp):
    _check_cascaded(oracle, tm.edge_chunks(type_id), type_id, 4096, *layers, bp)


@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("type_id", TYPES)
def test_cascaded_oracle_matches_model_partition_sizes(oracle, type_id, part):
    chunks = tm.edge_chunks(type_id, part)
    for r, d in [(1, 1), (7, 7)]:
        _check_cascaded(oracle, chunks, type_id, part, r, d, 1)
    _check_cascaded(oracle, chunks, type_id, part, 2, 1, 0)


def test_cascaded_header_pad_is_zero(oracle):
    """An odd partition count leaves 4 bytes between the offset table and the first partition: they are zero."""
    data = bytes(range(256)) * 48                           # 3 partitions of 4096 bytes
    s = oracle_compress(oracle, "cascaded", data, chunk_size=4096, type=1, num_RLEs=1, num_deltas=1, use_bp=1)
    assert tm._u32(s, 16) == 3 and tm._u32(s, 20) == 40
    assert s[36:40] == bytes(4)


@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("type_id", TYPES)
def test_bitcomp_oracle_matches_model(oracle, type_id, algo):
    for name, data in tm.bitcomp_edge_chunks(type_id):
        s = oracle_compress(oracle, "bitcomp", data, algo=algo, type=type_id)
        want = tm.bitcomp_model(data, algo, type_id)
        assert len(s) == want["size"], name
        assert tm.parse_bitcomp(s) == want, name
        assert oracle.decompress("bitcomp", s, len(data)) == data, name


def test_ans_oracle_matches_model(oracle):
    seen = set()
    for name, data in tm.ans_edge_chunks():
        s = oracle_compress(oracle, "ans", data)
        want = tm.ans_model(data)
        assert len(s) == want["size"], name
        assert tm.parse_ans(s) == want, name
        assert oracle.decompress("ans", s, len(data)) == data, name
        seen.add(want["header"][2])
        if name == "two_symbols_one_rare":
            assert want["freq"][0] == 4095 and want["freq"][1] == 1
        if name == "16MB":
            assert want["header"][3] == 1024
    assert seen == {0, 1, 2}                                # every mode is reached
