"""-m gpu: the warp-level Zstd device API (include/nvcomp/device/zstd.cuh) through the kernels of
tests/cpp/deflate_zstd_device_kernels.cu.

decompress_warp must return the batched call's status, size and bytes for every chunk and capacity, exactly, and
libzstd's verdict -- with the one documented difference (zstd_writer.four_stream_end_mismatch) allowed against libzstd
only, never against the batched call.  decompressed_size_warp must agree with GetDecompressSizeAsync.  Every output sits
in a guarded buffer (tests/gpu_util.py), the region must be reusable between calls, and a fused decode-and-sum must give
numpy's sums."""
import pytest

import zstd_writer as W
from test_deflate_device_gpu import (BAD_CHECKSUM, CANNOT_DECOMPRESS, INPUTS, OK, _codec, dev_decompress, edge_caps,
                                     match_batched, match_batched_sizes, run_fused_sum, run_huge_sizes, run_reuse,
                                     zstd_golden)
from gpu_util import gpu_decompress

pytestmark = pytest.mark.gpu
STATUS = {"ok": OK, "bad": CANNOT_DECOMPRESS, "checksum": BAD_CHECKSUM}


@pytest.fixture(scope="module")
def zs():
    z = W.libzstd_or_none()
    if z is None:
        pytest.skip("libzstd 1.5.5 (libzstd.so.1) not available: the verdicts are pinned to that release")
    return z


def corpus(zs):
    """(raw, stream): libzstd at six settings and pyarrow at three levels over every sample input, and the hand-built
    valid streams of zstd_writer (the corpus of test_zstd_gpu.py)."""
    from test_zstd_gpu import corpus as batched_corpus
    return batched_corpus(zs)


def corruptions(zs, count=3000):
    bases = []
    for name in ("text", "price_walk", "lowentropy", "clustered", "period33", "short13", "runlength_i32"):
        data = INPUTS[name]
        for level, ck, cs in ((1, True, True), (3, False, False), (19, True, False), (-5, False, True)):
            bases.append(zs.compress(data, level, checksum=ck, content_size=cs))
    return [W.corrupt(bases[seed % len(bases)], seed) for seed in range(count)]


def match_libzstd(zs, chunks, caps, **kw):
    """match_batched (device == batched, exactly), then both against libzstd.  Returns the number of chunks under the
    four-stream exemption."""
    outs, a, s = match_batched("zstd", chunks, caps, **kw)
    exempt = 0
    for i, (c, cap) in enumerate(zip(chunks, caps)):
        verdict, want = zs.expect(c, cap)
        if s[i] == CANNOT_DECOMPRESS and verdict != "bad" and W.four_stream_end_mismatch(c):
            exempt += 1
            continue
        assert s[i] == STATUS[verdict], (i, verdict, int(s[i]))
        if verdict == "ok":
            assert int(a[i]) == len(want) and outs[i] == want, i
    return exempt


def test_golden_vectors():
    """The committed libzstd vectors decode without libzstd present."""
    pairs = zstd_golden()
    outs, a, s = match_batched("zstd", [c for _, c in pairs], [len(r) for r, _ in pairs], what="golden")
    assert (s == OK).all() and outs == [r for r, _ in pairs]


def test_sizes_of_2_32_or_more():
    pairs = zstd_golden()[:6]
    run_huge_sizes("zstd", [c for _, c in pairs], [len(r) for r, _ in pairs])


def test_corpus_and_mutations(zs):
    pairs = corpus(zs) + zstd_golden()
    muts = W.mutations(zs, INPUTS)
    chunks = [c for _, c in pairs] + [c for _, c, _ in muts]
    caps = [len(r) for r, _ in pairs] + [1 << 20] * len(muts)
    match_libzstd(zs, chunks, caps, what="corpus")


def test_corruptions(zs):
    """3000 seeded corruptions."""
    chunks = corruptions(zs)
    exempt = match_libzstd(zs, chunks, [1 << 16] * len(chunks), in_mis=5, out_mis=12, what="corruptions")
    assert exempt <= 150, exempt


def test_capacity_edges(zs):
    pairs = corpus(zs)[::4]
    chunks, caps = edge_caps([c for _, c in pairs], [len(r) for r, _ in pairs])
    match_libzstd(zs, chunks, caps, what="caps")


def test_misalignment(zs):
    """Input and output misalignments 0-15 (each input offset with a different output offset)."""
    pairs = corpus(zs)[::9] + zstd_golden()[::3]
    chunks, caps = [c for _, c in pairs], [len(r) for r, _ in pairs]
    for m in range(16):
        outs, a, s = match_batched("zstd", chunks, caps, in_mis=m, out_mis=(7 * m + 3) % 16, what="misalign")
        assert (s == OK).all() and outs == [r for r, _ in pairs], m


def test_big_chunks(zs):
    from nvcomp_b200 import datagen
    big = datagen.tabular_f32(256, seed=21).tobytes()[:16 << 20]
    mb = big[:1 << 20]
    raws = [big, mb, mb]
    chunks = [zs.compress(big, 3, window_log=24, checksum=True), zs.compress(mb, 19, checksum=True),
              zs.compress(mb, 1, window_log=20)]
    outs, a, s = match_batched("zstd", chunks, [len(r) for r in raws], in_mis=3, out_mis=1, what="big")
    assert (s == OK).all() and outs == raws
    assert match_batched_sizes("zstd", chunks) == [len(r) for r in raws]


def test_null_actual(zs):
    pairs = corpus(zs)[::5]
    chunks = [c for _, c in pairs] + corruptions(zs, 100)
    caps = [len(r) for r, _ in pairs] + [1 << 16] * 100
    _, _, s = dev_decompress("zstd", chunks, caps, want_actual=False)
    _, _, bs, _ = gpu_decompress(_codec("zstd"), chunks, caps)
    assert s.tolist() == bs.tolist()


def test_decompressed_size(zs):
    chunks = [c for _, c in corpus(zs)] + [c for _, c, _ in W.mutations(zs, INPUTS)] + corruptions(zs)
    match_batched_sizes("zstd", chunks)
    match_batched_sizes("zstd", chunks[::7], in_mis=9)


def test_region_reuse(zs):
    pairs = corpus(zs)[::6] + zstd_golden()
    chunks = [c for _, c in pairs] + corruptions(zs, 200)
    caps = [len(r) for r, _ in pairs] + [1 << 16] * 200
    chunks, caps = chunks + chunks[:20], caps + [max(c - 1, 0) for c in caps[:20]]
    outs, a, s = run_reuse("zstd", chunks, caps)
    wouts, wa, ws = match_batched("zstd", chunks, caps, in_mis=3, out_mis=5, what="reuse")
    assert s.tolist() == ws.tolist() and a.tolist() == wa.tolist()
    assert [o if st == OK else b"" for o, st in zip(outs, s)] == [o if st == OK else b"" for o, st in zip(wouts, ws)]
    assert (s == OK).sum() >= len(pairs) and (s != OK).sum() >= 20


def test_fused_sum():
    pairs = zstd_golden()
    run_fused_sum("zstd", [c for _, c in pairs], [r for r, _ in pairs])
