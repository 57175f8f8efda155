"""-m gpu: the warp-level ANS device API (include/nvcomp/device/ans.cuh) against the batched C API and the oracle.

compress_warp must write the batched encoder's and the oracle's streams byte for byte; decompress_warp must return the
batched decoder's status, size and bytes for every chunk and capacity.  Every output sits in a guarded region
(tests/gpu_util.py): nothing may be written outside [out, out + capacity) or [out, out + max_compressed_bytes(n)),
and a successful decode writes exactly `actual` bytes.  A failed decode reports size 0; the bytes it left in the
output are not a result (a malformed stream can read stale words from the decoder's shared-memory ring), so only the
canaries are checked for those."""
import numpy as np
import pytest
import torch

import typed_model as tm
from conftest import sample_inputs

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="the ANS device API runs on a CUDA device")]

MB = 1 << 20
SIZES = [0, 1, 2, 31, 32, 33, 16383, 16384, 16385, 65536, MB, 16 * MB]


@pytest.fixture(scope="module")
def dev():
    from ans_device import AnsDevice
    return AnsDevice()


@pytest.fixture(scope="module")
def llif():
    from nvcomp_b200.batched import Codec
    return Codec("ANS")


@pytest.fixture(scope="module")
def llif_streams(llif):
    """The batched encoder's stream of every INPUTS chunk."""
    from gpu_util import gpu_compress
    return gpu_compress(llif, [v for _, v in INPUTS])[0]


def _inputs():
    """(name, bytes): edge chunks, the sample inputs, one chunk of every bench dataset, and the listed sizes up to
    1 MB as low-entropy, single-symbol (mode 2) and incompressible (mode 1) chunks."""
    from nvcomp_b200 import datagen
    out = list(tm.ans_edge_chunks(big=False))
    out += sorted(sample_inputs().items())
    out += [(f"bench_{k}", fn(1)[0].tobytes()) for k, fn in sorted(datagen.DATASETS.items())]
    rng = np.random.default_rng(4242)
    for n in SIZES[:-1]:
        out.append((f"geo_{n}", np.minimum(rng.geometric(0.3, n) - 1, 255).astype(np.uint8).tobytes()))
        out.append((f"const_{n}", bytes([0x5A]) * n))
        out.append((f"random_{n}", rng.integers(0, 256, n, dtype=np.uint8).tobytes()))
    return out


INPUTS = _inputs()
# 16 MB chunks go in batches of their own: a batched output slot is max_compressed_bytes(largest chunk)
_rng = np.random.default_rng(4343)
BIG = [("geo_16MB", np.minimum(_rng.geometric(0.3, SIZES[-1]) - 1, 255).astype(np.uint8).tobytes()),
       ("const_16MB", bytes([7]) * SIZES[-1]),
       ("random_16MB", _rng.integers(0, 256, SIZES[-1], dtype=np.uint8).tobytes())]


def dev_compress(dev, raws, misalign=0):
    """compress_warp every chunk (inputs at 16-byte aligned addresses + misalign) into guarded outputs of
    max_compressed_bytes(n).  Returns the streams."""
    from gpu_util import _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    inp = make_batch(raws, misalign=misalign)
    bounds = [dev.max_compressed_bytes(len(r)) for r in raws]
    out, allowed = _guarded_batch(bounds)
    status = torch.full((len(raws),), -1, dtype=torch.int32, device="cuda")
    dev.compress_async(inp, out, status, dev.compress_temp(len(raws)))
    torch.cuda.synchronize()
    sizes = out.sizes.cpu().numpy()
    assert (status.cpu().numpy() == 0).all()
    assert all(s <= b for s, b in zip(sizes, bounds)), "compressed size above max_compressed_bytes(n)"
    _check_canaries(out.slab.cpu().numpy(), allowed, out.offsets, "compress_warp")
    return out.to_host(sizes)


def dev_decompress(dev, streams, caps, in_misalign=0, out_misalign=0):
    """decompress_warp into guarded outputs.  Returns (outputs of `actual` bytes, actual, status)."""
    from gpu_util import FILL, _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    comp = make_batch(streams, misalign=in_misalign)
    out, allowed = _guarded_batch(caps, out_misalign)
    actual = torch.full((max(len(caps), 1),), -1, dtype=torch.int64, device="cuda")
    status = torch.full((max(len(caps), 1),), -1, dtype=torch.int32, device="cuda")
    dev.decompress_async(comp, out, actual, status)
    torch.cuda.synchronize()
    a, s = actual.cpu().numpy()[:len(caps)], status.cpu().numpy()[:len(caps)]
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, "decompress_warp")
    for i, (o, cap) in enumerate(zip(out.offsets, caps)):
        if s[i] == 0:
            assert (host[o + int(a[i]):o + cap] == FILL).all(), f"chunk {i} wrote past actual={int(a[i])}"
    return out.to_host(a), a, s


def assert_same_verdicts(dev, llif, streams, caps, in_misalign=0, out_misalign=0):
    """decompress_warp and the batched decoder agree on every chunk: status, actual, and the bytes of a success."""
    from gpu_util import gpu_decompress
    outs, a, s = dev_decompress(dev, streams, caps, in_misalign, out_misalign)
    louts, la, ls, _ = gpu_decompress(llif, streams, caps, in_misalign=in_misalign, out_misalign=out_misalign)
    for i in range(len(streams)):
        assert (s[i], a[i]) == (ls[i], la[i]), (i, s[i], a[i], ls[i], la[i])
        assert s[i] in (0, 12) and (s[i] == 0 or a[i] == 0), (i, s[i], a[i])
        if s[i] == 0:
            assert outs[i] == louts[i], i
    return outs, a, s


def test_constants_match_the_batched_api(dev, llif):
    for n in [0, 1, 16383, 16384, 16385, 65536, MB, 16 * MB]:
        assert dev.max_compressed_bytes(n) == llif.compress_get_max_output_chunk_size(n)
        assert dev.max_compressed_bytes(n) % 8 == 0
    assert dev.max_chunk_bytes() == 1 << 24


@pytest.mark.parametrize("misalign", range(8))
def test_streams_match_llif_and_oracle(dev, llif, llif_streams, oracle, misalign):
    from gpu_util import gpu_compress
    names, raws = [k for k, _ in INPUTS], [v for _, v in INPUTS]
    streams = dev_compress(dev, raws, misalign)
    lstreams = llif_streams if misalign == 0 else gpu_compress(llif, raws, misalign=misalign)[0]
    for name, raw, s, ls in zip(names, raws, streams, lstreams):
        assert s == ls, (name, len(raw), len(s), len(ls))
        if misalign == 0:
            assert s == oracle.compress_typed("ans", raw), name
    if misalign == 0:
        modes = {int.from_bytes(s[8:12], "little") for s in streams}
        assert modes == {0, 1, 2}, modes


@pytest.mark.parametrize("name,raw", BIG, ids=[k for k, _ in BIG])
def test_16mb_chunk(dev, llif, oracle, name, raw):
    """One 16 MB chunk (1024 segments): stream identity with the batched encoder and the oracle at two input
    misalignments, and decoding both ways."""
    from gpu_util import gpu_compress, gpu_decompress
    ls = gpu_compress(llif, [raw])[0][0]
    assert ls == oracle.compress_typed("ans", raw)
    for m in (0, 5):
        assert dev_compress(dev, [raw], m)[0] == ls, m
    outs, a, s = dev_decompress(dev, [ls], [len(raw)], out_misalign=3)
    assert (s[0], a[0]) == (0, len(raw)) and outs[0] == raw
    louts, la, lst, _ = gpu_decompress(llif, [ls], [len(raw)])
    assert (lst[0], la[0]) == (0, len(raw)) and louts[0] == raw


def test_decode_both_ways(dev, llif, llif_streams, oracle):
    """decompress_warp decodes the batched encoder's and the oracle's streams; the batched decoder decodes
    compress_warp's streams."""
    from gpu_util import gpu_decompress
    names, raws = [k for k, _ in INPUTS], [v for _, v in INPUTS]
    ostreams = [oracle.compress_typed("ans", r) for r in raws]
    dstreams = dev_compress(dev, raws)
    caps = [len(r) for r in raws]
    for streams in (llif_streams, ostreams):
        outs, a, s = dev_decompress(dev, streams, caps)
        for name, raw, o, ai, si in zip(names, raws, outs, a, s):
            assert (si, ai, o) == (0, len(raw), raw), name
    louts, la, ls, _ = gpu_decompress(llif, dstreams, caps)
    for name, raw, o, ai, si in zip(names, raws, louts, la, ls):
        assert (si, ai, o) == (0, len(raw), raw), name


@pytest.mark.parametrize("out_misalign", range(16))
def test_capacities_and_output_misalignment(dev, llif, llif_streams, out_misalign):
    """Capacities exact, exact - 1, 0 and 64 KB at every output misalignment."""
    raws = [v for _, v in INPUTS]
    streams, caps = [], []
    for s, r in zip(llif_streams, raws):
        n = len(r)
        for cap in {n, max(n - 1, 0), 0, 65536}:
            streams.append(s)
            caps.append(cap)
    _, a, s = assert_same_verdicts(dev, llif, streams, caps, out_misalign=out_misalign)
    for i, (cap, st) in enumerate(zip(caps, s)):
        n = int.from_bytes(streams[i][4:8], "little")
        assert (st == 0) == (n <= cap), (i, n, cap, st)


@pytest.mark.parametrize("seed", [7101, 7102, 7103])
def test_fuzzed_streams_get_the_batched_verdict(dev, llif, seed):
    """test_fuzz_gpu.py's recipe with new seeds: garbage, bit flips, truncations, extensions, plus every
    misaligned stream pointer."""
    from gpu_util import gpu_compress
    from nvcomp_b200.batched import make_batch
    inputs = sample_inputs()
    rng = np.random.default_rng(seed)
    names = ["text", "runlength_i32", "price_walk", "lowentropy", "sorted_i64", "period7", "ragged_40001",
             "random_777", "zeros_1000", "one", "empty"]
    raws = [inputs[n] for n in names] + [np.minimum(rng.geometric(0.3, 70000) - 1, 255).astype(np.uint8).tobytes()]
    goods, _ = gpu_compress(llif, raws)
    chunks, caps = [], []
    for n in [1, 2, 3, 7, 15, 16, 17, 64, 257, 528, 1000, 4096, 20000]:
        chunks.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes()); caps.append(65536)
    for g, r in zip(goods, raws):
        for _ in range(12):
            b = bytearray(g)
            for pos in rng.integers(0, len(b), rng.integers(1, 8)):
                b[pos] ^= 1 << rng.integers(0, 8)
            chunks.append(bytes(b)); caps.append(max(len(r), 1))
        for _ in range(3):
            chunks.append(g[: rng.integers(0, len(g))]); caps.append(max(len(r), 1))
        chunks.append(g + bytes(rng.integers(0, 256, 5, dtype=np.uint8))); caps.append(max(len(r), 1))
        chunks.append(g); caps.append(max(len(r), 1))
    _, _, s = assert_same_verdicts(dev, llif, chunks, caps)
    assert (s == 0).sum() >= len(goods) and (s == 12).any()
    comp = make_batch(chunks)
    assert dev.decompressed_size(comp).cpu().tolist() == llif.get_decompress_size(comp).cpu().tolist()
    for m in range(1, 8):
        _, _, s = assert_same_verdicts(dev, llif, goods, [max(len(r), 1) for r in raws], in_misalign=m)
        assert (s == 12).all(), m
        comp = make_batch(goods, misalign=m)
        assert dev.decompressed_size(comp).cpu().tolist() == [0] * len(goods)


def test_mixed_warps_in_one_cta(dev, llif):
    """Even warps compress one batch while the odd warps of the same CTAs decode another."""
    from gpu_util import gpu_compress
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import empty_batch, make_batch
    craws = [v for _, v in INPUTS if len(v) <= 65536] * 3
    draws = [r.tobytes() for r in datagen.lowentropy_bytes(200, seed=21)] + [v for _, v in INPUTS]
    lstreams, _ = gpu_compress(llif, craws)
    dstreams, _ = gpu_compress(llif, draws)
    inp = make_batch(craws)
    cout = empty_batch(len(craws), dev.max_compressed_bytes(max(len(r) for r in craws)))
    comp = make_batch(dstreams)
    dout = make_batch([bytes(len(r)) for r in draws])
    cst = torch.full((len(craws),), -1, dtype=torch.int32, device="cuda")
    actual = torch.full((len(draws),), -1, dtype=torch.int64, device="cuda")
    dst = torch.full((len(draws),), -1, dtype=torch.int32, device="cuda")
    dev.mixed_async(inp, cout, cst, dev.compress_temp(max(len(craws), len(draws))), comp, dout, actual, dst)
    torch.cuda.synchronize()
    assert (cst.cpu().numpy() == 0).all() and (dst.cpu().numpy() == 0).all()
    assert cout.to_host() == lstreams
    assert actual.cpu().tolist() == [len(r) for r in draws]
    assert dout.to_host() == draws


def test_fused_decode_and_reduce(dev, llif):
    """A kernel that decodes a chunk and reduces the decoded bytes (sum and histogram) in the same kernel."""
    from gpu_util import gpu_compress
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import make_batch
    raws = [r.tobytes() for r in datagen.lowentropy_bytes(300, seed=22)] + [v for _, v in INPUTS]
    streams, _ = gpu_compress(llif, raws)
    streams.append(streams[0][:100])                 # one that fails: reduced over 0 bytes
    raws.append(b"")
    comp = make_batch(streams)
    out = make_batch([bytes(max(len(r), 1)) for r in raws[:-1]] + [bytes(65536)])
    n = len(streams)
    actual = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    sums = torch.zeros(n, dtype=torch.int64, device="cuda")
    hists = torch.zeros(n * 256, dtype=torch.int32, device="cuda")
    dev.fused_async(comp, out, actual, status, sums, hists)
    torch.cuda.synchronize()
    st = status.cpu().numpy()
    assert (st[:-1] == 0).all() and st[-1] == 12
    assert actual.cpu().tolist() == [len(r) for r in raws]
    h = hists.cpu().numpy().reshape(n, 256)
    s = sums.cpu().numpy()
    for i, r in enumerate(raws):
        b = np.frombuffer(r, dtype=np.uint8)
        assert s[i] == int(b.sum(dtype=np.uint64)), i
        assert (h[i] == np.bincount(b, minlength=256)).all(), i


def test_chunk_too_large(dev):
    """n > kMaxChunkBytes: ChunkSizeTooLarge, comp_bytes 0, nothing written."""
    from gpu_util import FILL, _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    n = dev.max_chunk_bytes() + 1
    inp = make_batch([bytes(n), b"ab" * 100])
    out, allowed = _guarded_batch([dev.max_compressed_bytes(n), dev.max_compressed_bytes(200)])
    status = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    dev.compress_async(inp, out, status, dev.compress_temp(2))
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [18, 0]
    sizes = out.sizes.cpu().tolist()
    assert sizes == [0, 16 + 200]                  # "ab" * 100 is stored raw
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, "compress_warp")
    o = int(out.offsets[0])
    assert (host[o:o + dev.max_compressed_bytes(n)] == FILL).all()
