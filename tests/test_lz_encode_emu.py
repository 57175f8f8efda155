"""CPU: the warp-per-chunk LZ77 matcher with the LZ4 and Snappy emitters (include/nvcomp/device/detail/
lz77_compress.cuh, lz4_encode.cuh, snappy_encode.cuh), run in the host warp emulator (tests/emu: 32 fibers,
rendezvous at every warp intrinsic, guard pages around the global buffers).

Every stream must pass the stream-rules model of tests/lz_encode_model.py (valid, maximal, stride-aligned matches
inside the end-of-chunk limits, and the emitters' exact element forms), decode under liblz4 at exact capacity or
pyarrow, fit the codec's bound, and be the same at every input and output misalignment.  Ratio floors per dataset
catch a matcher that still writes valid streams but finds fewer matches."""
import numpy as np
import pytest

import lz_encode_model as M
from nvcomp_b200 import datagen

INPUTS = M.corpus()
NAMES = sorted(INPUTS)


@pytest.fixture(scope="module")
def enc():
    return M.EmuLzEncoder()


@pytest.fixture(scope="module")
def snappy():
    pa = pytest.importorskip("pyarrow")
    return pa.Codec("snappy")


def _id(v):
    return f"{v[0]}{v[1]}"


@pytest.mark.parametrize("variant", M.VARIANTS, ids=_id)
@pytest.mark.parametrize("name", NAMES)
def test_stream_rules(name, variant, enc, liblz4, snappy):
    kind, step = variant
    data = INPUTS[name]
    stream = enc.compress(kind, data, step)
    assert len(stream) <= M.BOUND[kind](len(data))
    seqs = M.check(kind, stream, data, step)
    assert seqs == enc.parse(kind, data, step), "the stream is not the matcher's parse"
    if kind == "lz4":
        assert liblz4.decompress(stream, len(data)) == data
    elif data:
        assert snappy.decompress(stream, decompressed_size=len(data)).to_pybytes() == data
    if not data:
        assert stream == b"\x00"      # LZ4: one empty literal-only token; Snappy: the preamble varint 0


@pytest.mark.parametrize("name", NAMES)
def test_misaligned_same_bytes(name, enc):
    k = 1 + NAMES.index(name) % 15
    for kind, step in M.VARIANTS:
        assert enc.compress(kind, INPUTS[name], step, in_mis=k, out_mis=16 - k) == enc.compress(kind, INPUTS[name],
                                                                                                  step)


@pytest.mark.parametrize("name", ["sample:price_walk", "sample:runlength_i32", "size:77"])
def test_every_misalignment(name, enc):
    for kind, step in M.VARIANTS:
        want = enc.compress(kind, INPUTS[name], step)
        for k in range(16):
            assert enc.compress(kind, INPUTS[name], step, in_mis=k, out_mis=15 - k) == want, (kind, step, k)


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
@pytest.mark.parametrize("period", [65534, 65535, 65536, 65537])
def test_largest_offset(period, kind, enc):
    """Data that repeats after `period` bytes is matched at that offset up to 65 535, and not at all beyond it."""
    data = INPUTS[f"period:{period}"]
    seqs = M.check(kind, enc.compress(kind, data), data)[:-1]
    if period <= M.MAX_OFFSET:
        assert any(off == period for _, off, _ in seqs) and sum(ml for *_, ml in seqs) >= 4000, seqs
    else:
        assert seqs == []


def test_model_rejects_near_misses():
    """The model fails streams that decode but break one rule: a match one byte short, a Snappy copy-2 where copy-1
    fits, a stride-2 match at an odd position, an LZ4 match that starts 12 bytes before the end."""
    rng = np.random.default_rng(1)
    head, tail = rng.integers(0, 256, (2, 40), dtype=np.uint8)
    assert head[8] != tail[0]
    data = head.tobytes() + head[:8].tobytes() + tail.tobytes()
    seqs = [(40, 40, 8), (40, 0, 0)]
    short = [(40, 40, 7), (41, 0, 0)]
    for kind, emit in (("lz4", M.emit_lz4), ("snappy", M.emit_snappy)):
        M.check(kind, emit(data, seqs), data)
        with pytest.raises(AssertionError, match="not maximal"):
            M.check(kind, emit(data, short), data)
    good = M.emit_snappy(data, seqs)
    copy1 = M._snappy_copy(40, 8)
    assert len(copy1) == 2 and good.count(copy1) == 1
    copy2 = bytes([2 | (7 << 2), 40, 0])
    with pytest.raises(AssertionError, match="restated"):
        M.check("snappy", good.replace(copy1, copy2), data)
    period3 = INPUTS["sample:period3"][:600]
    M.check("lz4", M.emit_lz4(period3, [(3, 3, 592), (5, 0, 0)]), period3)
    with pytest.raises(AssertionError, match="stride"):
        M.check("lz4", M.emit_lz4(period3, [(3, 3, 592), (5, 0, 0)]), period3, step=2)
    late = INPUTS["size:40"]
    M.check("lz4", M.emit_lz4(late, [(27, 5, 8), (5, 0, 0)]), late)
    with pytest.raises(AssertionError, match="sequence 0 at 28"):
        M.check("lz4", M.emit_lz4(late, [(28, 5, 7), (5, 0, 0)]), late)


# Floors on each dataset's ratio, 8 x 64 KB chunks, just under what the matcher reaches (liblz4 1.9.4 default and
# pyarrow Snappy reach: runlength_i32 52.58 / 16.88, tabular_f32 1.673 / 1.946, sorted_i64 2.625 / 2.580,
# lowentropy_bytes 1.489 / 1.971, random_bytes 0.996 / 1.000, snappy_synth 1.443 / 2.128, lz4_mixed 3.253 / 3.521).
# A dropped candidate path fails them: without the intra-group candidates runlength_i32 falls far below its floor.
RATIO_FLOOR = {
    "runlength_i32": (52.2, 16.8),
    "tabular_f32": (1.66, 1.93),
    "sorted_i64": (2.37, 2.45),
    "lowentropy_bytes": (1.47, 1.99),
    "random_bytes": (0.995, 0.999),
    "snappy_synth": (1.43, 2.12),
    "lz4_mixed": (3.23, 3.49),
}


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
@pytest.mark.parametrize("dataset", sorted(RATIO_FLOOR))
def test_ratio_floor(dataset, kind, enc):
    chunks = [r.tobytes() for r in datagen.DATASETS[dataset](8)]
    ratio = sum(map(len, chunks)) / sum(len(enc.compress(kind, c)) for c in chunks)
    floor = RATIO_FLOOR[dataset][kind == "snappy"]
    assert ratio >= floor, f"{dataset} {kind}: {ratio:.4f} < {floor}"
