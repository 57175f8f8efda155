"""-m gpu: the warp-level Bitcomp device API (include/nvcomp/device/bitcomp.cuh) against the batched C API and the
oracle.

compress_warp must write the batched encoder's and the oracle's streams byte for byte; decompress_warp must return the
batched decoder's and the oracle's status, size and bytes for every chunk and capacity; for_each_block must hand every
element of a chunk the oracle decodes to the caller, in order, and call nothing for a chunk the oracle rejects.
Every output sits in a guarded region (tests/gpu_util.py): nothing may be written outside [out, out + capacity) or
[out, out + max_compressed_bytes(n)), and a successful decode writes exactly `actual` bytes."""
import numpy as np
import pytest
import torch

import typed_model as tm
import typed_writer as W

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="the Bitcomp device API runs on a CUDA device")]

MB = 1 << 20
TYPES = range(8)
ALGOS = (0, 1)
M64 = (1 << 64) - 1
NP_TYPE = {0: np.int8, 1: np.uint8, 2: np.int16, 3: np.uint16, 4: np.int32, 5: np.uint32, 6: np.int64, 7: np.uint64}


@pytest.fixture(scope="module")
def dev():
    from bitcomp_device import BitcompDevice
    return BitcompDevice()


def codec(algo=0, type_id=1):
    from nvcomp_b200._lib import BitcompOpts
    from nvcomp_b200.batched import Codec
    return Codec("Bitcomp", opts=BitcompOpts(algo, type_id))


def _inputs(type_id):
    """(name, bytes): the Bitcomp edge chunks of the type, a 64 KB slice of every bench dataset, and those slices cut
    to lengths that are not a multiple of the element size."""
    from nvcomp_b200 import datagen
    ts = tm.TYPE_SIZE[type_id]
    out = list(tm.bitcomp_edge_chunks(type_id))
    for k, fn in sorted(datagen.DATASETS.items()):
        raw = fn(1)[0].tobytes()[:65536]
        out.append((f"bench_{k}", raw))
        if ts > 1:
            out.append((f"bench_{k}_ragged", raw[:65536 - ts + 1 + len(k) % (ts - 1)]))
    return out


def dev_compress(dev, raws, algo, type_id, misalign=0):
    """compress_warp every chunk (inputs at 16-byte aligned addresses + misalign) into guarded outputs of
    max_compressed_bytes(n).  Returns (streams, status)."""
    from gpu_util import _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    inp = make_batch(raws, misalign=misalign)
    bounds = [dev.max_compressed_bytes(len(r), algo, type_id) for r in raws]
    out, allowed = _guarded_batch(bounds)
    status = torch.full((max(len(raws), 1),), -1, dtype=torch.int32, device="cuda")
    dev.compress_async(inp, out, status, algo, type_id)
    torch.cuda.synchronize()
    sizes = out.sizes.cpu().numpy()
    assert all(s <= b for s, b in zip(sizes, bounds)), "compressed size above max_compressed_bytes(n)"
    _check_canaries(out.slab.cpu().numpy(), allowed, out.offsets, "compress_warp")
    return out.to_host(sizes), status.cpu().numpy()[:len(raws)], out


def dev_decompress(dev, streams, caps, in_misalign=0, out_misalign=0):
    """decompress_warp into guarded outputs (gpu_util.guarded_decompress): (outputs of `actual` bytes, actual, status)."""
    from gpu_util import guarded_decompress

    def launch(comp, out, _max_chunk):
        actual = torch.full((max(len(caps), 1),), -1, dtype=torch.int64, device="cuda")
        status = torch.full((max(len(caps), 1),), -1, dtype=torch.int32, device="cuda")
        dev.decompress_async(comp, out, actual, status)
        return actual, status
    outs, a, s, _ = guarded_decompress(launch, "decompress_warp", streams, caps, in_misalign, out_misalign)
    return outs, a, s


def assert_verdicts(dev, oracle, streams, caps, names, in_misalign=0, out_misalign=0, use_oracle=True):
    """decompress_warp agrees with the batched decoder (and, for aligned pointers, the oracle) on every chunk: status,
    actual, and the bytes of a success."""
    from gpu_util import gpu_decompress
    outs, a, s = dev_decompress(dev, streams, caps, in_misalign, out_misalign)
    louts, la, ls, _ = gpu_decompress(codec(), streams, caps, in_misalign=in_misalign, out_misalign=out_misalign)
    bad = []
    for i in range(len(streams)):
        ok = (s[i], a[i]) == (ls[i], la[i]) and s[i] in (0, 12) and (s[i] == 0 or a[i] == 0)
        ok = ok and (s[i] != 0 or outs[i] == louts[i])
        if ok and use_oracle:
            w = oracle.decompress("bitcomp", streams[i], caps[i])
            ok = (s[i] == 12) if w is None else (s[i] == 0 and outs[i] == w)
        if not ok:
            bad.append(i)
    assert not bad, [(names[i], caps[i], int(s[i]), int(a[i]), int(ls[i]), int(la[i])) for i in bad[:20]]
    return outs, a, s


def _widen(data: bytes, type_id: int) -> np.ndarray:
    ts = tm.TYPE_SIZE[type_id]
    v = np.frombuffer(data[:len(data) // ts * ts], dtype=NP_TYPE[type_id])
    return v.astype(np.int64).view(np.uint64) if type_id in tm.SIGNED else v.astype(np.uint64)


def _mix64(x: np.ndarray) -> np.ndarray:
    x = x ^ (x >> np.uint64(30)); x = x * np.uint64(0xBF58476D1CE4E5B9)
    x = x ^ (x >> np.uint64(27)); x = x * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def expected_visit(data: bytes, type_id: int):
    """(sum, hash, visits) of the visit kernel for a chunk that decodes to `data` (see bitcomp_device_kernels.cu)."""
    w = _widen(data, type_id)
    n = len(w)
    if n == 0:
        return 0, 0, 0
    idx = np.arange(n, dtype=np.uint64)
    m = _mix64(w ^ (idx * np.uint64(0x9E3779B97F4A7C15)))
    h = 0
    for d in np.add.reduceat(m, np.arange(0, n, 128)):
        h = ((h ^ int(d)) * 0x100000001B3) & M64
    return int(w.sum(dtype=np.uint64)), h, (n + 127) // 128


def dev_visit(dev, streams, elem_type, misalign=0):
    from nvcomp_b200.batched import make_batch
    n = max(len(streams), 1)
    sums, hashes, visits = (torch.full((n,), -1, dtype=torch.int64, device="cuda") for _ in range(3))
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    dev.visit_async(make_batch(streams, misalign=misalign), elem_type, sums, hashes, visits, status)
    torch.cuda.synchronize()
    u = [t.cpu().numpy()[:len(streams)].view(np.uint64) for t in (sums, hashes, visits)]
    return u[0], u[1], u[2], status.cpu().numpy()[:len(streams)]


def _header_type_n(b: bytes):
    return (b[5], int.from_bytes(b[8:12], "little")) if len(b) >= 16 else (None, 0)


def assert_visits(dev, oracle, streams, names):
    """for_each_block over every stream, with the element type the stream declares: a stream the oracle decodes (with
    room for all of it) gives the numpy sum, hash and block count of the oracle's elements; any other gives
    CannotDecompress and no visit."""
    by_type = {}
    for s, name in zip(streams, names):
        t, n = _header_type_n(s)
        if n > 1 << 25:                             # a corrupted size no stream here can back: left to the other tests
            continue
        by_type.setdefault(t if t in NP_TYPE else 1, []).append((name, s, n))
    seen = {0: 0, 12: 0}
    for t, cases in sorted(by_type.items()):
        ss = [c[1] for c in cases]
        sums, hashes, visits, st = dev_visit(dev, ss, t)
        for i, (name, s, n) in enumerate(cases):
            w = oracle.decompress("bitcomp", s, n)
            if w is None:
                assert (st[i], visits[i]) == (12, 0), (name, int(st[i]), int(visits[i]))
            else:
                assert st[i] == 0, (name, int(st[i]))
                assert (int(sums[i]), int(hashes[i]), int(visits[i])) == expected_visit(w, t), name
            seen[int(st[i])] += 1
    return seen


# ------------------------------------------------------------------------------------------------------ constants
def test_constants_match_the_batched_api(dev):
    for algo in ALGOS:
        for t in TYPES:
            c = codec(algo, t)
            for n in [0, 1, 127, 128, 129, 65536, 1 << 24]:
                assert dev.max_compressed_bytes(n, algo, t) == c.compress_get_max_output_chunk_size(n), (algo, t, n)
    assert dev.max_chunk_bytes() == 1 << 24
    assert dev.compress_smem_bytes() == 132 * 8 and dev.compress_smem_bytes() % dev.smem_alignment() == 0
    assert dev.max_compressed_bytes((1 << 24) + 1, 0, 1) == 0
    assert dev.max_compressed_bytes(100, 2, 1) == 0 and dev.max_compressed_bytes(100, 0, 8) == 0


# -------------------------------------------------------------------------------------------------------- streams
@pytest.mark.parametrize("type_id", TYPES)
@pytest.mark.parametrize("algo", ALGOS)
def test_streams_match_llif_and_oracle(dev, oracle, algo, type_id):
    from gpu_util import gpu_compress
    ts = tm.TYPE_SIZE[type_id]
    items = _inputs(type_id)
    names, raws = [k for k, _ in items], [v for _, v in items]
    lstreams, _ = gpu_compress(codec(algo, type_id), raws)
    for misalign in sorted({0, ts, 8}):
        streams, st, _ = dev_compress(dev, raws, algo, type_id, misalign)
        assert (st == 0).all(), misalign
        for name, raw, s, ls in zip(names, raws, streams, lstreams):
            assert s == ls, (misalign, name, len(raw), len(s), len(ls))
    for name, raw, ls in zip(names, raws, lstreams):
        assert ls == oracle.compress_typed("bitcomp", raw, algo=algo, type=type_id), name


def test_invalid_opts_and_chunk_too_large(dev):
    """Invalid options: InvalidValue; n > kMaxChunkBytes: ChunkSizeTooLarge; both with comp_bytes 0 and nothing
    written."""
    from gpu_util import FILL, _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    for algo, t, n, want in ((2, 1, 100, 10), (-1, 1, 100, 10), (0, 8, 100, 10), (0, 7, (1 << 24) + 8, 18)):
        inp = make_batch([bytes(n)])
        out, allowed = _guarded_batch([4096])
        status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        dev.compress_async(inp, out, status, algo, t)
        torch.cuda.synchronize()
        assert (int(status[0]), int(out.sizes[0])) == (want, 0), (algo, t, n)
        host = out.slab.cpu().numpy()
        _check_canaries(host, allowed, out.offsets, "compress_warp")
        assert (host[int(out.offsets[0]):int(out.offsets[0]) + 4096] == FILL).all()


# ------------------------------------------------------------------------------------------------ decode verdicts
def _writer_cases():
    chunks, caps, names = [], [], []
    for name, c in list(W.VALID.items()) + list(W.INVALID.items()):
        if c.codec == "bitcomp":
            for cap in sorted({c.cap, max(c.cap - 1, 0), 0}):
                chunks.append(c.comp); caps.append(cap); names.append(name)
    return chunks, caps, names


@pytest.fixture(scope="module")
def campaign():
    camp = W.corruption_campaign(W.campaign_sources(), "bitcomp")
    return [x[2] for x in camp], [x[3] for x in camp], [f"{x[0]}:{x[1]}" for x in camp]


def test_writer_cases(dev, oracle):
    chunks, caps, names = _writer_cases()
    assert_verdicts(dev, oracle, chunks, caps, names)


def test_corruption_campaign(dev, oracle, campaign):
    streams, lens, names = campaign
    assert len(streams) >= 3000
    chunks, caps, cnames = [], [], []
    for s, n, name in zip(streams, lens, names):
        for cap in sorted({n, max(n - 1, 0), 0}):
            chunks.append(s); caps.append(cap); cnames.append(name)
    _, _, st = assert_verdicts(dev, oracle, chunks, caps, cnames)
    assert (st == 0).sum() >= 100 and (st == 12).sum() >= 300


def test_output_misalignment(dev, oracle):
    """Outputs 1 to 15 bytes past 16-byte alignment: a typed stream whose output is not aligned to its element is
    rejected as the batched decoder rejects it; the rest decode to the batched decoder's bytes."""
    cases = [c for c in W.VALID.values() if c.codec == "bitcomp"]
    from gpu_util import gpu_compress
    raws = [r for _, r in _inputs(6)[:12]]
    streams = [c.comp for c in cases] + gpu_compress(codec(0, 6), raws)[0] + gpu_compress(codec(1, 1), raws)[0]
    caps = [c.cap for c in cases] + [len(r) for r in raws] * 2
    names = [f"s{i}" for i in range(len(streams))]
    for m in range(1, 16):
        _, _, s = assert_verdicts(dev, oracle, streams, caps, names, out_misalign=m, use_oracle=False)
        for i, b in enumerate(streams):
            ts = tm.TYPE_SIZE[b[5]]
            assert (s[i] == 0) == (m % ts == 0), (m, i, ts, int(s[i]))


def test_misaligned_streams_and_size_query(dev, oracle, campaign):
    """Streams 1 to 7 bytes off their 8-byte alignment: CannotDecompress, actual 0, a size of 0.  Aligned: the size
    query gives the batched query's answer on every writer and campaign stream."""
    from nvcomp_b200.batched import make_batch
    cases = [c for c in W.VALID.values() if c.codec == "bitcomp"]
    chunks, caps = [c.comp for c in cases], [c.cap for c in cases]
    for m in range(1, 8):
        _, a, s = dev_decompress(dev, chunks, caps, in_misalign=m)
        assert (s == 12).all() and (a == 0).all(), (m, s.tolist())
        assert dev.decompressed_size(make_batch(chunks, misalign=m)).cpu().tolist() == [0] * len(chunks), m
        for t in (1, 2, 4, 6):
            _, _, visits, st = dev_visit(dev, chunks, t, misalign=m)
            assert (st == 12).all() and (visits == 0).all(), (m, t)
    streams = _writer_cases()[0] + campaign[0]
    comp = make_batch(streams)
    got = dev.decompressed_size(comp).cpu().tolist()
    want = codec().get_decompress_size(comp).cpu().tolist()
    assert got == want
    assert sum(g > 0 for g in got) >= 100 and sum(g == 0 for g in got) >= 20


# ------------------------------------------------------------------------------------------------- for_each_block
def test_for_each_block_writer_and_campaign(dev, oracle, campaign):
    names = [n for n, c in list(W.VALID.items()) + list(W.INVALID.items()) if c.codec == "bitcomp"]
    streams = [c.comp for c in list(W.VALID.values()) + list(W.INVALID.values()) if c.codec == "bitcomp"]
    seen = assert_visits(dev, oracle, streams + campaign[0], names + campaign[2])
    assert seen[0] >= 100 and seen[12] >= 300, seen


@pytest.mark.parametrize("type_id", TYPES)
def test_for_each_block_encoder_streams(dev, oracle, type_id):
    """Both algorithms' streams of every input, visited with the stream's type; with a type of another size the visit
    returns InvalidValue and calls nothing."""
    from gpu_util import gpu_compress
    items = _inputs(type_id)
    streams = []
    for algo in ALGOS:
        streams += gpu_compress(codec(algo, type_id), [v for _, v in items])[0]
    names = [k for k, _ in items] * 2
    seen = assert_visits(dev, oracle, streams, names)
    assert seen[12] == 0
    other = {1: 6, 2: 0, 4: 2, 8: 5}[tm.TYPE_SIZE[type_id]]
    _, _, visits, st = dev_visit(dev, streams, other)
    assert (st == 10).all() and (visits == 0).all()


# ------------------------------------------------------------------------------------------ concurrency and size
def test_mixed_warps_in_one_cta(dev, oracle):
    """Warps of the same CTAs compress one batch, decompress another and visit a third at once."""
    from gpu_util import gpu_compress
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import empty_batch, make_batch
    craws = [r.tobytes() for r in datagen.sorted_i64(150, seed=31)] + [v for _, v in _inputs(7)]
    draws = [r.tobytes() for r in datagen.runlength_i32(200, seed=32)]
    vraws = [r.tobytes() for r in datagen.sorted_i64(250, seed=33)] + [v for _, v in _inputs(6)]
    lstreams, _ = gpu_compress(codec(0, 7), craws)
    dstreams, _ = gpu_compress(codec(1, 4), draws)
    vstreams, _ = gpu_compress(codec(0, 6), vraws)
    inp = make_batch(craws)
    cout = empty_batch(len(craws), dev.max_compressed_bytes(max(len(r) for r in craws), 0, 7))
    comp, vcomp = make_batch(dstreams), make_batch(vstreams)
    dout = make_batch([bytes(len(r)) for r in draws])
    cst = torch.full((len(craws),), -1, dtype=torch.int32, device="cuda")
    actual = torch.full((len(draws),), -1, dtype=torch.int64, device="cuda")
    dst = torch.full((len(draws),), -1, dtype=torch.int32, device="cuda")
    sums, hashes, visits = (torch.full((len(vraws),), -1, dtype=torch.int64, device="cuda") for _ in range(3))
    vst = torch.full((len(vraws),), -1, dtype=torch.int32, device="cuda")
    dev.mixed_async(inp, cout, cst, 0, 7, comp, dout, actual, dst, vcomp, sums, hashes, visits, vst)
    torch.cuda.synchronize()
    assert (cst.cpu().numpy() == 0).all() and (dst.cpu().numpy() == 0).all() and (vst.cpu().numpy() == 0).all()
    assert cout.to_host() == lstreams
    assert actual.cpu().tolist() == [len(r) for r in draws]
    assert dout.to_host() == draws
    u = [t.cpu().numpy().view(np.uint64) for t in (sums, hashes, visits)]
    for i, r in enumerate(vraws):
        assert (int(u[0][i]), int(u[1][i]), int(u[2][i])) == expected_visit(r, 6), i


@pytest.mark.parametrize("algo,type_id", [(0, 6), (1, 5)])
def test_16mb_chunk(dev, oracle, algo, type_id):
    """A 16 MB chunk (the largest allowed): compress_warp's stream is the batched encoder's and the oracle's, and it
    round-trips through decompress_warp and for_each_block."""
    from gpu_util import gpu_compress
    rng = np.random.default_rng(77 + algo)
    n = 1 << 24
    ts = tm.TYPE_SIZE[type_id]
    if algo == 0:
        vals = np.cumsum(rng.integers(-50, 1000, n // ts)).astype(NP_TYPE[type_id])
    else:
        vals = (rng.integers(0, 1 << 20, n // ts) * (rng.random(n // ts) < 0.2)).astype(NP_TYPE[type_id])
    raw = vals.tobytes()
    ls = gpu_compress(codec(algo, type_id), [raw])[0][0]
    assert ls == oracle.compress_typed("bitcomp", raw, algo=algo, type=type_id)
    streams, st, _ = dev_compress(dev, [raw], algo, type_id)
    assert st[0] == 0 and streams[0] == ls
    outs, a, s = dev_decompress(dev, [ls], [n], out_misalign=ts)
    assert (s[0], a[0]) == (0, n) and outs[0] == raw
    sums, hashes, visits, vst = dev_visit(dev, [ls], type_id)
    assert vst[0] == 0 and (int(sums[0]), int(hashes[0]), int(visits[0])) == expected_visit(raw, type_id)
