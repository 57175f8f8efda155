"""-m gpu: Cascaded, Bitcomp and ANS decoding held to the oracle through the C ABI -- the hand-built streams of
tests/typed_writer.py (legal streams no encoder writes, and one stream per rejection rule) and a seeded corruption
campaign over real encoder streams, in mixed batches.  Status, `actual` and the bytes must be the oracle's for every
stream and capacity; gpu_util.gpu_decompress also checks the canaries around every output and that a success wrote
exactly `actual` bytes.  The size query, the 8-byte alignment of the streams and the warp-level ANS device API
(decompress_warp) are held to the same verdicts."""
import pytest
import torch

import typed_writer as W

pytestmark = pytest.mark.gpu
FMT = {"cascaded": "Cascaded", "bitcomp": "Bitcomp", "ans": "ANS"}
CODECS = sorted(FMT)


def _codec(codec):
    from nvcomp_b200.batched import Codec
    return Codec(FMT[codec])


def _want(oracle, codec, chunks, caps):
    return [oracle.decompress(codec, c, cap) for c, cap in zip(chunks, caps)]


def _diverging(want, outs, a, s):
    """Indices where the decoder's status / actual / bytes are not the oracle's verdict."""
    bad = []
    for i, w in enumerate(want):
        ok = (s[i] == 12 and a[i] == 0) if w is None else (s[i] == 0 and a[i] == len(w) and outs[i] == w)
        if not ok:
            bad.append(i)
    return bad


def _check(oracle, codec, chunks, caps, names, in_mis=0, out_mis=0):
    from gpu_util import gpu_decompress
    want = _want(oracle, codec, chunks, caps)
    outs, a, s, _ = gpu_decompress(_codec(codec), chunks, caps, in_misalign=in_mis, out_misalign=out_mis)
    bad = _diverging(want, outs, a, s)
    assert not bad, [(names[i], caps[i], int(s[i]), int(a[i]), None if want[i] is None else len(want[i]))
                     for i in bad[:20]]
    return want


def _writer_batch(codec):
    """Every valid case at capacities exact, exact - 1 and 0; every invalid case at its capacity and 0."""
    chunks, caps, names = [], [], []
    for name, c in W.VALID.items():
        if c.codec == codec:
            for cap in sorted({c.cap, max(c.cap - 1, 0), 0}):
                chunks.append(c.comp); caps.append(cap); names.append(name)
    for name, c in W.INVALID.items():
        if c.codec == codec:
            for cap in (c.cap, 0):
                chunks.append(c.comp); caps.append(cap); names.append(name)
    return chunks, caps, names


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("in_mis,out_mis", [(0, 0), (0, 8), (8, 0), (8, 8)])
def test_writer_cases(oracle, codec, in_mis, out_mis):
    chunks, caps, names = _writer_batch(codec)
    _check(oracle, codec, chunks, caps, names, in_mis, out_mis)


@pytest.fixture(scope="module")
def sources():
    return W.campaign_sources()


def _campaign(sources, codec):
    """3000 corrupted streams at capacities raw length, raw length + 64 and raw length - 1 in turn."""
    camp = W.corruption_campaign(sources, codec)
    chunks = [x[2] for x in camp]
    caps = [(n, n + 64, max(n - 1, 0))[i % 3] for i, (_, _, _, n) in enumerate(camp)]
    names = [f"{x[0]}:{x[1]}" for x in camp]
    return chunks, caps, names


@pytest.mark.parametrize("codec", CODECS)
def test_corruption_campaign(oracle, sources, codec):
    chunks, caps, names = _campaign(sources, codec)
    assert len(chunks) >= 3000
    want = _check(oracle, codec, chunks, caps, names)
    # both verdicts are well represented
    assert sum(w is None for w in want) >= 300 and sum(w is not None for w in want) >= 100


@pytest.mark.parametrize("codec", CODECS)
def test_size_query(oracle, sources, codec):
    """GetDecompressSizeAsync: the oracle's length for every stream the oracle decodes, 0 for a stream whose header is
    malformed."""
    from nvcomp_b200.batched import make_batch
    chunks, want = [], []
    for c in W.VALID.values():
        if c.codec == codec:
            chunks.append(c.comp); want.append(len(c.out))
    for c in W.INVALID.values():
        if c.codec == codec and c.header:
            chunks.append(c.comp); want.append(0)
    for _, _, bad, _ in W.corruption_campaign(sources, codec)[:1000]:
        r = oracle.decompress(codec, bad, 1 << 25)
        if r is not None:
            chunks.append(bad); want.append(len(r))
    sizes = _codec(codec).get_decompress_size(make_batch(chunks))
    torch.cuda.synchronize()
    got = sizes.cpu().tolist()
    bad = [i for i in range(len(want)) if got[i] != want[i]]
    assert not bad, [(i, got[i], want[i]) for i in bad[:20]]


@pytest.mark.parametrize("codec", CODECS)
def test_misaligned_streams_are_rejected(codec):
    """The streams are 8-byte aligned by definition: at 1 .. 7 bytes past that, status CannotDecompress, actual 0 and
    a size query of 0, for streams that decode when aligned."""
    from gpu_util import gpu_decompress
    from nvcomp_b200.batched import make_batch
    cases = [c for c in W.VALID.values() if c.codec == codec]
    chunks, caps = [c.comp for c in cases], [c.cap for c in cases]
    for mis in range(1, 8):
        _, a, s, _ = gpu_decompress(_codec(codec), chunks, caps, in_misalign=mis, out_misalign=0)
        assert (s == 12).all() and (a == 0).all(), (mis, s.tolist())
        sizes = _codec(codec).get_decompress_size(make_batch(chunks, misalign=mis))
        torch.cuda.synchronize()
        assert sizes.cpu().tolist() == [0] * len(chunks), mis


def _dev_decompress(dev, streams, caps):
    """decompress_warp into guarded outputs (gpu_util.guarded_decompress): (outputs of `actual` bytes, actual, status)."""
    from gpu_util import guarded_decompress

    def launch(comp, out, _max_chunk):
        actual = torch.full((max(len(caps), 1),), -1, dtype=torch.int64, device="cuda")
        status = torch.full((max(len(caps), 1),), -1, dtype=torch.int32, device="cuda")
        dev.decompress_async(comp, out, actual, status)
        return actual, status
    outs, a, s, _ = guarded_decompress(launch, "decompress_warp", streams, caps)
    return outs, a, s


def test_ans_device_api(oracle, sources):
    """The warp-level device API's decompress_warp shares the batched decoder's segment decode: the ANS writer cases and
    campaign get the oracle's verdicts there too."""
    from ans_device import AnsDevice
    dev = AnsDevice()
    chunks, caps, names = _writer_batch("ans")
    c2, k2, n2 = _campaign(sources, "ans")
    chunks, caps, names = chunks + c2, caps + k2, names + n2
    want = _want(oracle, "ans", chunks, caps)
    outs, a, s = _dev_decompress(dev, chunks, caps)
    bad = _diverging(want, outs, a, s)
    assert not bad, [(names[i], caps[i], int(s[i]), int(a[i])) for i in bad[:20]]
