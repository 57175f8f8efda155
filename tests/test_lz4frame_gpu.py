"""GPU: nvcompBatchedLZ4FrameDecompressAsync and nvcompBatchedLZ4FrameGetDecompressSizeAsync held to the host warp
emulator (and through it to liblz4's LZ4F_decompress) byte for byte and status for status, on the hand-built frames,
producer frames and a corruption sample of tests/test_lz4frame_emu.py, in one batch and across batch positions; plus
10 000 x 64 KB pyarrow frames, a 32 MB chunk of 4 MB-block frames, a 0-byte chunk, temp / actual / statuses null,
actual aliasing caps, canaries past every output and two calls on two streams."""
import numpy as np
import pytest
import torch

import lz4frame_writer as F
from nvcomp_b200.batched import Codec, make_batch
from test_lz4frame_emu import FrameEmu, campaign_seeds, mutate, producer_frames, producer_inputs

pytestmark = pytest.mark.gpu
CANARY = 0xAB
PAD = 32


@pytest.fixture(scope="module")
def lz4f():
    return F.LibLZ4F()


@pytest.fixture(scope="module")
def cases(lz4f):
    return _cases(lz4f)


_CACHE = {}


def _cases(lz4f):
    """(name, chunk, cap, emulator status, emulator bytes, emulator size), built once per session"""
    if "cases" in _CACHE:
        return _CACHE["cases"]
    emu = FrameEmu()
    # every fourth FLG / BD combination (the emulator test runs them all) and every other frame of the writer
    chunks = {k: v for i, (k, v) in enumerate(F.corpus(lz4f).items())
              if k[:2] not in ("b4", "b5", "b6", "b7") or i % 4 == 0}
    inputs = {k: v for k, v in producer_inputs().items() if len(v) <= 1 << 17}
    chunks.update(producer_frames(lz4f, inputs, prefs=[dict(bsid=4, linked=True), dict(bsid=5, linked=False,
                                                                                       content_sum=True,
                                                                                       block_sum=True)]))
    rng = np.random.default_rng(11)
    seeds = list(campaign_seeds(lz4f).values())
    for i in range(300):
        c = mutate(rng, seeds[int(rng.integers(0, len(seeds)))])
        if not F.has_offset0_match(c):            # (liblz4 accepts offset-0 matches: see test_lz4frame_emu.py)
            chunks[f"corrupt_{i}"] = c
    out = []
    for name, chunk in chunks.items():
        err, dec = lz4f.decode(chunk)
        n = len(dec)
        for cap in sorted({n, max(n - 1, 0)}) if err is None else [n + 64]:
            st, got = emu.decode(chunk, cap)
            assert (st, got) == lz4f.verdict(chunk, cap), name
            out.append((name, chunk, cap, st, got, emu.size(chunk)))
    _CACHE["cases"] = out
    return out


def run(cases, order, stream=None, temp=True, want_actual=True, want_status=True, alias=False):
    codec = Codec("LZ4Frame")
    sel = [cases[i] for i in order]
    comp = make_batch([c[1] for c in sel])
    out = make_batch([bytes([CANARY]) * (c[2] + PAD) for c in sel])
    caps = torch.tensor([c[2] for c in sel], dtype=torch.int64, device="cuda")
    n = len(sel)
    sh = (stream or torch.cuda.current_stream()).cuda_stream
    tb = codec.decompress_get_temp_size(n, 1 << 20)
    tmp = torch.zeros(tb, dtype=torch.uint8, device="cuda")
    actual = caps.clone() if alias else torch.full((n,), -7, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(),
                               actual.data_ptr() if alias else caps.data_ptr(),
                               actual.data_ptr() if want_actual else None, n, tmp.data_ptr() if temp else None,
                               tb if temp else 0, out.ptrs.data_ptr(), status.data_ptr() if want_status else None, sh)
    return sel, comp, out, actual, status


def check(sel, out, actual, status, want_actual=True, want_status=True):
    torch.cuda.synchronize()
    slab = out.slab.cpu().numpy()
    act = actual.cpu().tolist()
    sts = status.cpu().tolist()
    for i, (name, chunk, cap, st, got, _) in enumerate(sel):
        if want_status:
            assert sts[i] == st, (name, cap, sts[i], st)
        if want_actual:
            assert act[i] == (len(got) if st == 0 else 0), (name, act[i])
        o = int(out.offsets[i])
        if st == 0:
            assert slab[o:o + len(got)].tobytes() == got, name
            assert (slab[o + len(got):o + cap + PAD] == CANARY).all(), (name, "written past actual")
        else:
            assert (slab[o + cap:o + cap + PAD] == CANARY).all(), (name, "written past cap")


def test_batch_equals_emulator(cases):
    order = list(range(len(cases)))
    sel, _, out, actual, status = run(cases, order)
    check(sel, out, actual, status)


def test_batch_positions(cases):
    rng = np.random.default_rng(5)
    order = rng.permutation(len(cases)).tolist()
    sel, _, out, actual, status = run(cases, order)
    check(sel, out, actual, status)
    order = [i for i in range(len(cases)) for _ in range(2)][::-1]
    sel, _, out, actual, status = run(cases, order, temp=False)
    check(sel, out, actual, status)


def test_null_actual_status_and_alias(cases):
    order = list(range(0, len(cases), 3))
    sel, _, out, actual, status = run(cases, order, want_actual=False)
    check(sel, out, actual, status, want_actual=False)
    sel, _, out, actual, status = run(cases, order, want_status=False)
    check(sel, out, actual, status, want_status=False)
    sel, _, out, actual, status = run(cases, order, alias=True)
    check(sel, out, actual, status)


def test_size_query_equals_emulator(cases):
    codec = Codec("LZ4Frame")
    comp = make_batch([c[1] for c in cases])
    sizes = codec.get_decompress_size(comp).cpu().tolist()
    assert sizes == [c[5] for c in cases]


def test_two_streams(cases):
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = run(cases, list(range(0, len(cases), 2)), stream=s1)
    b = run(cases, list(range(1, len(cases), 2)), stream=s2)
    for sel, _, out, actual, status in (a, b):
        check(sel, out, actual, status)


def test_zero_byte_chunk_and_compress_is_unavailable():
    codec = Codec("LZ4Frame")
    comp = make_batch([b"", b""])
    out = make_batch([bytes([CANARY]) * 16, bytes([CANARY]) * 16])
    actual, status = codec.decompress(comp, out)
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [0, 0] and actual.cpu().tolist() == [0, 0]
    assert (out.slab.cpu().numpy()[:32] == CANARY).all()
    assert codec.get_decompress_size(comp).cpu().tolist() == [0, 0]
    with pytest.raises(NotImplementedError):
        codec.compress_get_max_output_chunk_size(65536)


def test_ten_thousand_pyarrow_frames():
    import pyarrow as pa
    from nvcomp_b200 import datagen
    data = np.concatenate([datagen.tabular_f32(5000, seed=31).view(np.uint8),
                           datagen.runlength_i32(5000, seed=32).view(np.uint8)])
    pc = pa.Codec("lz4")
    chunks = [pc.compress(row.tobytes()).to_pybytes() for row in data]
    codec = Codec("LZ4Frame")
    comp = make_batch(chunks)
    out = make_batch([bytes(65536 + 16)] * len(chunks))
    out.sizes = torch.full((len(chunks),), 65536, dtype=torch.int64, device="cuda")
    sizes = codec.get_decompress_size(comp)
    actual, status = codec.decompress(comp, out)
    torch.cuda.synchronize()
    assert (status == 0).all().item() and (actual == 65536).all().item() and (sizes == 65536).all().item()
    slab = out.slab.cpu().numpy()
    got = np.stack([slab[o:o + 65536] for o in out.offsets])
    assert np.array_equal(got, data)


def test_32mb_chunk_of_4mb_block_frames(lz4f):
    from nvcomp_b200 import datagen
    data = np.concatenate([datagen.tabular_f32(256, seed=41).view(np.uint8).reshape(-1),
                           datagen.runlength_i32(256, seed=42).view(np.uint8).reshape(-1)]).tobytes()
    assert len(data) == 32 << 20
    chunk = b"".join(lz4f.compress_frame(data[i:i + (8 << 20)], 7, i % (16 << 20) == 0, True, i % 2 == 0, True)
                     for i in range(0, len(data), 8 << 20))
    codec = Codec("LZ4Frame")
    comp = make_batch([chunk])
    out = make_batch([bytes(len(data) + 16)])
    out.sizes = torch.tensor([len(data)], dtype=torch.int64, device="cuda")
    actual, status = codec.decompress(comp, out)
    sizes = codec.get_decompress_size(comp)
    torch.cuda.synchronize()
    assert status.item() == 0 and actual.item() == len(data) and sizes.item() == len(data)
    assert out.slab[:len(data)].cpu().numpy().tobytes() == data
