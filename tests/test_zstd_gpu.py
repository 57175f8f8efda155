"""GPU: batched Zstd decompression through the C ABI (nvcompBatchedZstd*), held to libzstd's verdicts and bytes on
libzstd's and pyarrow's streams, the hand-built and mutated streams of tests/zstd_writer.py, the committed golden
vectors and a seeded corruption campaign.  Every call runs on guarded output buffers (gpu_util.gpu_decompress):
nothing may be written outside a chunk, and a successful chunk writes exactly `actual` bytes."""
import json
import os

import numpy as np
import pytest
import torch

import zstd_writer as W
from conftest import sample_inputs
from gpu_util import FILL, gpu_decompress
from nvcomp_b200.batched import Codec, empty_batch, make_batch

pytestmark = pytest.mark.gpu

INPUTS = sample_inputs()
STATUS = {"ok": 0, "bad": 12, "checksum": 13}


@pytest.fixture(scope="module")
def zs():
    z = W.libzstd_or_none()
    if z is None:
        pytest.skip("libzstd 1.5.5 (libzstd.so.1) not available: the verdicts are pinned to that release")
    return z


@pytest.fixture(scope="module")
def codec():
    return Codec("Zstd")


def _pyarrow(data, level):
    pa = pytest.importorskip("pyarrow")
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def corpus(zs):
    out = []
    for name in sorted(INPUTS):
        data = INPUTS[name]
        for level, strategy, wl, ck, cs in ((-5, None, 17, False, True), (1, None, 17, True, True),
                                            (3, None, 10, False, False), (9, 6, 17, True, False),
                                            (19, 9, 17, False, True), (22, None, 10, True, True)):
            out.append((data, zs.compress(data, level, strategy, wl, ck, cs)))
        out += [(data, _pyarrow(data, level)) for level in (1, 3, 19)]
    for name, s, want in W.valid_streams(zs, INPUTS):
        out.append((want, s))
    return out


def golden():
    gdir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    with open(os.path.join(gdir, "zstd_manifest.json")) as f:
        vecs = json.load(f)["vectors"]
    out = []
    for v in vecs:
        with open(os.path.join(gdir, v["raw"]), "rb") as f:
            raw = f.read()
        with open(os.path.join(gdir, v["comp"]), "rb") as f:
            out.append((raw, f.read()))
    return out


def assert_matches_libzstd(zs, codec, streams, caps, **kw):
    """Statuses, sizes and bytes equal libzstd's.  Returns how many chunks fell under the one documented difference
    (W.four_stream_end_mismatch: rejected here, decoded by libzstd)."""
    outs, actual, status, _ = gpu_decompress(codec, streams, caps, **kw)
    exempt = 0
    for i, (s, cap) in enumerate(zip(streams, caps)):
        verdict, want = zs.expect(s, cap)
        if status[i] == STATUS["bad"] and verdict != "bad" and W.four_stream_end_mismatch(s):
            assert actual[i] == 0, i
            exempt += 1
            continue
        assert status[i] == STATUS[verdict], (i, verdict, int(status[i]))
        if verdict == "ok":
            assert int(actual[i]) == len(want) and outs[i] == want, i
        else:
            assert actual[i] == 0, i
    return exempt


@pytest.mark.parametrize("misalign", [0, 1, 7])
def test_zstd_decodes_corpus_and_golden(zs, codec, misalign):
    pairs = corpus(zs) + golden()
    streams = [s for _, s in pairs]
    caps = [len(d) for d, _ in pairs]
    outs, actual, status, _ = gpu_decompress(codec, streams, caps, misalign=misalign)
    assert (status == 0).all(), np.flatnonzero(status)
    for i, (d, _) in enumerate(pairs):
        assert int(actual[i]) == len(d) and outs[i] == d, i


def test_zstd_hand_built_and_mutated_streams(zs, codec):
    muts = W.mutations(zs, INPUTS)
    streams = [s for _, s, _ in muts]
    assert_matches_libzstd(zs, codec, streams, [1 << 20] * len(streams))
    for (rule, s, verdict) in muts:
        assert zs.expect(s, 1 << 20)[0] == verdict, rule


def test_zstd_capacity_edges(zs, codec):
    streams, caps = [], []
    for name in ("one", "text", "zeros_64k", "random_64k", "sensor", "ragged_40001"):
        data = INPUTS[name]
        s = zs.compress(data, 3, checksum=True)
        for cap in (len(data), max(len(data) - 1, 0), 0):
            streams.append(s)
            caps.append(cap)
    assert_matches_libzstd(zs, codec, streams, caps)


def test_zstd_optional_arguments(zs, codec):
    data = [INPUTS[k] for k in ("text", "price_walk", "zeros_1000", "random_777")]
    streams = [zs.compress(d, 3) for d in data]
    caps = [len(d) for d in data]
    outs, a, s, _ = gpu_decompress(codec, streams, caps, want_actual=False)
    assert a is None and (s == 0).all() and outs == data
    outs, a, s, _ = gpu_decompress(codec, streams, caps, want_status=False)
    assert s is None and outs == data
    # no workspace (static chunk stride), and actual aliasing the capacities
    comp = make_batch(streams)
    out = empty_batch(len(data), max(caps), fill=FILL)
    out.sizes.copy_(torch.tensor(caps, dtype=torch.int64, device="cuda"))
    status = torch.full((len(data),), -1, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(), out.sizes.data_ptr(),
                           len(data), None, 0, out.ptrs.data_ptr(), status.data_ptr(), stream)
    torch.cuda.synchronize()
    assert (status == 0).all() and out.sizes.cpu().tolist() == caps
    assert out.to_host(np.asarray(caps)) == data
    # an empty batch is a no-op
    codec.decompress_async(0, 0, 0, 0, 0, None, 0, 0, 0, stream)
    codec.get_decompress_size_async(0, 0, 0, 0, stream)
    assert codec.decompress_get_temp_size(10, 1 << 16) == 256


def test_zstd_size_query(zs, codec):
    pairs = corpus(zs)[:200]
    streams = [s for _, s in pairs]
    streams += [W.corrupt(s, seed) for seed, s in enumerate(streams)]
    sizes = codec.get_decompress_size(make_batch(streams)).cpu().tolist()
    for s, n in zip(streams, sizes):
        verdict, want = zs.expect(s, 1 << 25)
        if n == 0 and verdict != "bad" and W.four_stream_end_mismatch(s):
            continue                   # the one documented difference (W.four_stream_end_mismatch)
        if verdict == "ok":
            assert n == len(want)
        elif verdict == "bad":
            assert n == 0
        # a checksum verdict: the size query produces no bytes, so it cannot see the checksum


def test_zstd_mixed_producer_batch_2000(zs, codec):
    pairs = corpus(zs) + golden()
    rng = np.random.default_rng(4)
    pick = [pairs[i] for i in rng.integers(0, len(pairs), 2000)]
    outs, actual, status, _ = gpu_decompress(codec, [s for _, s in pick], [len(d) for d, _ in pick])
    assert (status == 0).all()
    assert all(o == d for o, (d, _) in zip(outs, pick))


def test_zstd_ragged_and_large_chunks(zs, codec):
    from nvcomp_b200 import datagen
    big = datagen.tabular_f32(256, seed=21).tobytes()[:16 << 20]
    mb = big[:1 << 20]
    rng = np.random.default_rng(9)
    ragged = [big[int(o):int(o) + int(n)] for o, n in zip(rng.integers(0, 1 << 20, 40), rng.integers(0, 200000, 40))]
    datas = [big, mb, mb] + ragged
    streams = [zs.compress(big, 3, window_log=24, checksum=True), zs.compress(mb, 19, checksum=True),
               zs.compress(mb, 1, window_log=20)] + [zs.compress(d, 3) for d in ragged]
    outs, actual, status, _ = gpu_decompress(codec, streams, [len(d) for d in datas], misalign=3)
    assert (status == 0).all()
    assert all(o == d for o, d in zip(outs, datas))


def test_zstd_corruption_campaign(zs, codec):
    """3000 seeded corruptions: statuses equal libzstd's verdicts, bytes equal on success, canaries intact.  The one
    exception: a 4-stream Huffman literal stream that does not end exactly on its first bit is rejected where libzstd
    may decode it (W.four_stream_end_mismatch); those cases are counted and must stay rare."""
    bases = []
    for name in ("text", "price_walk", "lowentropy", "clustered", "period33", "short13", "runlength_i32"):
        data = INPUTS[name]
        for level, ck, cs in ((1, True, True), (3, False, False), (19, True, False), (-5, False, True)):
            bases.append(zs.compress(data, level, checksum=ck, content_size=cs))
    streams = [W.corrupt(bases[seed % len(bases)], seed) for seed in range(3000)]
    exempt = assert_matches_libzstd(zs, codec, streams, [1 << 16] * len(streams), misalign=5)
    print(f"3000 corruptions: {exempt} four-stream end mismatches")
    assert exempt <= 150, exempt


def test_zstd_respects_stream_order(zs, codec):
    """The inputs are written by a kernel on a non-default stream just before the decode on that stream."""
    data = [INPUTS[k] for k in ("text", "price_walk", "lowcard", "random_64k")]
    streams = [zs.compress(d, 3, checksum=True) for d in data]
    side = torch.cuda.Stream()
    comp = make_batch(streams)
    host = comp.slab.clone()
    out = empty_batch(len(data), max(len(d) for d in data), fill=0)
    out.sizes.copy_(torch.tensor([len(d) for d in data], dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        comp.slab.zero_()
        comp.slab.copy_(host)          # the decoder must see these bytes, not the zeros
        actual, status = codec.decompress(comp, out, stream=side)
    side.synchronize()
    assert (status == 0).all() and actual.cpu().tolist() == [len(d) for d in data]
    assert out.to_host(actual.cpu().numpy()) == data
