"""-m gpu: the warp-level Cascaded device API (include/nvcomp/device/cascaded.cuh) against the batched C API and the
oracle.

compress_warp must write the batched encoder's and the oracle's streams byte for byte; decompress_warp must return the
batched decoder's and the oracle's status, size and bytes for every chunk and capacity; for_each_block must hand every
element of a chunk the oracle decodes to the caller, in order and in blocks that never cross a partition, and call
nothing for a chunk the oracle rejects.  Every output sits in a guarded region (tests/gpu_util.py): nothing may be
written outside [out, out + capacity) or [out, out + max_compressed_bytes(n)), and a successful decode writes exactly
`actual` bytes."""
import numpy as np
import pytest
import torch

import typed_model as tm
import typed_writer as W

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="the Cascaded device API runs on a CUDA device")]

TYPES = range(8)
M64 = (1 << 64) - 1
NP_TYPE = {0: np.int8, 1: np.uint8, 2: np.int16, 3: np.uint16, 4: np.int32, 5: np.uint32, 6: np.int64, 7: np.uint64}
BENCH_OPTS = (4096, 6, 1, 1, 1)          # (chunk_size, type, num_RLEs, num_deltas, use_bp) of bench.py --codec cascaded
# legal options the stream tests sweep: both partition-size extremes, a size that is not a power of two, 7/7 layers,
# no layers at all, and use_bp off
SWEEP = [(4096, 6, 1, 1, 1), (512, 4, 1, 0, 1), (16384, 1, 7, 7, 1), (520, 3, 2, 1, 0), (4096, 0, 0, 2, 1),
         (16384, 7, 1, 1, 1), (1024, 5, 0, 0, 1), (512, 2, 3, 2, 0), (2048, 6, 7, 7, 0), (512, 7, 2, 2, 1)]


@pytest.fixture(scope="module")
def dev():
    from cascaded_device import CascadedDevice
    return CascadedDevice()


def codec(opts=(4096, 4, 2, 1, 1)):
    from nvcomp_b200._lib import CascadedOpts
    from nvcomp_b200.batched import Codec
    return Codec("Cascaded", opts=CascadedOpts(*opts))


def oracle_compress(oracle, raw, opts):
    p, t, r, d, bp = opts
    return oracle.compress_typed("cascaded", raw, chunk_size=p, type=t, num_RLEs=r, num_deltas=d, use_bp=bp)


def _inputs(opts):
    """(name, bytes): the edge chunks of the type and partition size, a 64 KB slice of every bench dataset, and those
    slices cut to lengths that are not a multiple of the element size."""
    from nvcomp_b200 import datagen
    part, type_id = opts[0], opts[1]
    ts = tm.TYPE_SIZE[type_id]
    out = list(tm.edge_chunks(type_id, part))
    for k, fn in sorted(datagen.DATASETS.items()):
        raw = fn(1)[0].tobytes()[:65536]
        out.append((f"bench_{k}", raw))
        if ts > 1:
            out.append((f"bench_{k}_ragged", raw[:65536 - ts + 1 + len(k) % (ts - 1)]))
    return out


def dev_compress(dev, raws, opts, misalign=0):
    """compress_warp every chunk (inputs at 16-byte aligned addresses + misalign) into guarded outputs of
    max_compressed_bytes(n).  Returns (streams, status, out batch)."""
    from gpu_util import _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    inp = make_batch(raws, misalign=misalign)
    bounds = [dev.max_compressed_bytes(len(r), opts) for r in raws]
    out, allowed = _guarded_batch(bounds)
    status = torch.full((max(len(raws), 1),), -1, dtype=torch.int32, device="cuda")
    dev.compress_async(inp, out, status, opts)
    torch.cuda.synchronize()
    sizes = out.sizes.cpu().numpy()
    assert all(s <= b for s, b in zip(sizes, bounds)), "compressed size above max_compressed_bytes(n)"
    _check_canaries(out.slab.cpu().numpy(), allowed, out.offsets, "compress_warp")
    return out.to_host(sizes), status.cpu().numpy()[:len(raws)], out


def dev_decompress(dev, streams, caps, region, in_misalign=0, out_misalign=0):
    """decompress_warp into guarded outputs (gpu_util.guarded_decompress): (outputs of `actual` bytes, actual, status,
    out batch)."""
    from gpu_util import guarded_decompress

    def launch(comp, out, _max_chunk):
        actual = torch.full((max(len(caps), 1),), -1, dtype=torch.int64, device="cuda")
        status = torch.full((max(len(caps), 1),), -1, dtype=torch.int32, device="cuda")
        dev.decompress_async(comp, out, actual, status, region)
        return actual, status
    return guarded_decompress(launch, "decompress_warp", streams, caps, in_misalign, out_misalign)


def assert_verdicts(dev, oracle, streams, caps, names, in_misalign=0, out_misalign=0, use_oracle=True):
    """decompress_warp (in the largest region any stream needs) agrees with the batched decoder (and, for aligned
    pointers, the oracle) on every chunk: status, actual, and the bytes of a success."""
    from gpu_util import gpu_decompress
    outs, a, s, _ = dev_decompress(dev, streams, caps, dev.max_decompress_smem_bytes(), in_misalign, out_misalign)
    louts, la, ls, _ = gpu_decompress(codec(), streams, caps, in_misalign=in_misalign, out_misalign=out_misalign)
    bad = []
    for i in range(len(streams)):
        ok = (s[i], a[i]) == (ls[i], la[i]) and s[i] in (0, 12) and (s[i] == 0 or a[i] == 0)
        ok = ok and (s[i] != 0 or outs[i] == louts[i])
        if ok and use_oracle:
            w = oracle.decompress("cascaded", streams[i], caps[i])
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


def expected_visit(data: bytes, type_id: int, part: int):
    """(sum, hash, visits) of the visit kernel for a chunk of `part`-byte partitions that decodes to `data` (see
    cascaded_device_kernels.cu): blocks of 128 elements, restarted at every partition boundary."""
    w = _widen(data, type_id)
    n = len(w)
    if n == 0:
        return 0, 0, 0
    per = part // tm.TYPE_SIZE[type_id]
    starts = np.concatenate([np.arange(p, min(p + per, n), 128) for p in range(0, n, per)])
    idx = np.arange(n, dtype=np.uint64)
    m = _mix64(w ^ (idx * np.uint64(0x9E3779B97F4A7C15)))
    h = 0
    for d in np.add.reduceat(m, starts):
        h = ((h ^ int(d)) * 0x100000001B3) & M64
    return int(w.sum(dtype=np.uint64)), h, len(starts)


def dev_visit(dev, streams, elem_type, region=None, misalign=0):
    from nvcomp_b200.batched import make_batch
    n = max(len(streams), 1)
    sums, hashes, visits = (torch.full((n,), -1, dtype=torch.int64, device="cuda") for _ in range(3))
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    region = dev.max_decompress_smem_bytes() if region is None else region
    dev.visit_async(make_batch(streams, misalign=misalign), elem_type, sums, hashes, visits, status, region)
    torch.cuda.synchronize()
    u = [t.cpu().numpy()[:len(streams)].view(np.uint64) for t in (sums, hashes, visits)]
    return u[0], u[1], u[2], status.cpu().numpy()[:len(streams)]


def _header(b: bytes):
    """(type, uncompressed bytes, partition bytes) of a stream header, or (None, 0, 0) for a short stream."""
    if len(b) < 20:
        return None, 0, 0
    return b[4], int.from_bytes(b[8:12], "little"), int.from_bytes(b[12:16], "little")


def assert_visits(dev, oracle, streams, names):
    """for_each_block over every stream, with the element type the stream declares: a stream the oracle decodes (with
    room for all of it) gives the numpy sum, hash and block count of the oracle's elements; any other gives
    CannotDecompress and no visit."""
    by_type = {}
    for s, name in zip(streams, names):
        t, n, part = _header(s)
        if n > 1 << 25:                             # a corrupted size no stream here can back: left to the other tests
            continue
        by_type.setdefault(t if t in NP_TYPE else 1, []).append((name, s, n, part))
    seen = {0: 0, 12: 0}
    for t, cases in sorted(by_type.items()):
        sums, hashes, visits, st = dev_visit(dev, [c[1] for c in cases], t)
        for i, (name, s, n, part) in enumerate(cases):
            w = oracle.decompress("cascaded", s, n)
            if w is None:
                assert (st[i], visits[i]) == (12, 0), (name, int(st[i]), int(visits[i]))
            else:
                assert st[i] == 0, (name, int(st[i]))
                assert (int(sums[i]), int(hashes[i]), int(visits[i])) == expected_visit(w, t, part), name
            seen[int(st[i])] += 1
    return seen


# ------------------------------------------------------------------------------------------------------ constants
def test_constants_match_the_batched_api(dev):
    layers = (0, 1, 2, 7)
    for t in TYPES:
        for r in layers:
            for d in layers:
                for bp in (0, 1):
                    for part in (512, 520, 4096, 16384):
                        opts = (part, t, r, d, bp)
                        c = codec(opts)
                        for n in (0, 1, 7, 511, 4097, 65536, 1 << 24):
                            assert dev.max_compressed_bytes(n, opts) == c.compress_get_max_output_chunk_size(n), \
                                (opts, n)
                        assert dev.max_compressed_bytes((1 << 24) + 1, opts) == 0, opts
    for bad in ((504, 6, 1, 1, 1), (513, 6, 1, 1, 1), (16392, 6, 1, 1, 1), (4096, 8, 1, 1, 1), (4096, 6, 8, 1, 1),
                (4096, 6, 1, 8, 1), (4096, 6, -1, 1, 1)):
        assert dev.max_compressed_bytes(100, bad) == 0, bad
        assert dev.compress_smem_bytes(bad) == 0 and dev.decompress_smem_bytes(bad) == 0, bad
    assert dev.max_chunk_bytes() == 1 << 24 and dev.smem_alignment() == 16
    assert dev.compress_smem_bytes(BENCH_OPTS) == 24704
    assert dev.decompress_smem_bytes(BENCH_OPTS) == 5136
    assert dev.max_decompress_smem_bytes() == 65552
    assert dev.decompress_smem_bytes((16384, 0, 2, 0, 1)) == 65552
    for t in TYPES:
        for part in (512, 520, 4096, 16384):
            for r, d in ((0, 0), (1, 1), (2, 1), (7, 7)):
                opts = (part, t, r, d, 1)
                for v in (dev.compress_smem_bytes(opts), dev.decompress_smem_bytes(opts)):
                    assert v > 0 and v % 16 == 0, (opts, v)
                assert dev.decompress_smem_bytes(opts) <= dev.max_decompress_smem_bytes()


# -------------------------------------------------------------------------------------------------------- streams
@pytest.mark.parametrize("opts", SWEEP, ids=lambda o: "p{}_t{}_r{}_d{}_bp{}".format(*o))
def test_streams_match_llif_and_oracle(dev, oracle, opts):
    from gpu_util import gpu_compress
    ts = tm.TYPE_SIZE[opts[1]]
    items = _inputs(opts)
    names, raws = [k for k, _ in items], [v for _, v in items]
    lstreams, _ = gpu_compress(codec(opts), raws)
    for misalign in sorted({0, ts, 8}):
        streams, st, _ = dev_compress(dev, raws, opts, misalign)
        assert (st == 0).all(), misalign
        for name, raw, s, ls in zip(names, raws, streams, lstreams):
            assert s == ls, (misalign, name, len(raw), len(s), len(ls))
    for name, raw, ls in zip(names, raws, lstreams):
        assert ls == oracle_compress(oracle, raw, opts), name


def test_invalid_opts_and_chunk_too_large(dev):
    """Invalid options: InvalidValue; n > kMaxChunkBytes: ChunkSizeTooLarge; both with comp_bytes 0 and nothing
    written."""
    from gpu_util import FILL, _check_canaries, _guarded_batch
    from nvcomp_b200.batched import make_batch
    for opts, n, want in (((4096, 8, 1, 1, 1), 100, 10), ((504, 6, 1, 1, 1), 100, 10), ((4096, 6, 8, 0, 1), 100, 10),
                          ((4096, 6, 1, -1, 1), 100, 10), ((4096, 7, 1, 1, 1), (1 << 24) + 8, 18)):
        inp = make_batch([bytes(n)])
        out, allowed = _guarded_batch([4096])
        status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        dev.compress_async(inp, out, status, opts)
        torch.cuda.synchronize()
        assert (int(status[0]), int(out.sizes[0])) == (want, 0), (opts, n)
        host = out.slab.cpu().numpy()
        _check_canaries(host, allowed, out.offsets, "compress_warp")
        assert (host[int(out.offsets[0]):int(out.offsets[0]) + 4096] == FILL).all()


# ------------------------------------------------------------------------------------------------ decode verdicts
def _writer_cases():
    chunks, caps, names = [], [], []
    for name, c in list(W.VALID.items()) + list(W.INVALID.items()):
        if c.codec == "cascaded":
            for cap in sorted({c.cap, max(c.cap - 1, 0), 0}):
                chunks.append(c.comp); caps.append(cap); names.append(name)
    return chunks, caps, names


@pytest.fixture(scope="module")
def campaign():
    camp = W.corruption_campaign(W.campaign_sources(), "cascaded")
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
    """Outputs 1 to 15 bytes past 16-byte alignment: a stream whose output is not aligned to its element is rejected
    as the batched decoder rejects it; the rest decode to the batched decoder's bytes."""
    from gpu_util import gpu_compress
    cases = [c for c in W.VALID.values() if c.codec == "cascaded"]
    raws = [r for _, r in _inputs(BENCH_OPTS)[:12]]
    streams = ([c.comp for c in cases] + gpu_compress(codec(BENCH_OPTS), raws)[0]
               + gpu_compress(codec((512, 1, 2, 1, 1)), raws)[0])
    caps = [c.cap for c in cases] + [len(r) for r in raws] * 2
    names = [f"s{i}" for i in range(len(streams))]
    for m in range(1, 16):
        _, _, s = assert_verdicts(dev, oracle, streams, caps, names, out_misalign=m, use_oracle=False)
        for i, b in enumerate(streams):
            ts = tm.TYPE_SIZE[b[4]]
            assert (s[i] == 0) == (m % ts == 0), (m, i, ts, int(s[i]))


def test_misaligned_streams_and_size_query(dev, oracle, campaign):
    """Streams 1 to 7 bytes off their 8-byte alignment: CannotDecompress, actual 0, a size of 0, no visit.  Aligned:
    the size query gives the batched query's answer on every writer and campaign stream."""
    from nvcomp_b200.batched import make_batch
    cases = [c for c in W.VALID.values() if c.codec == "cascaded"]
    chunks, caps = [c.comp for c in cases], [c.cap for c in cases]
    for m in range(1, 8):
        _, a, s, _ = dev_decompress(dev, chunks, caps, dev.max_decompress_smem_bytes(), in_misalign=m)
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


# ------------------------------------------------------------------------------------------------------ region size
@pytest.mark.parametrize("opts", SWEEP, ids=lambda o: "p{}_t{}_r{}_d{}_bp{}".format(*o))
def test_region_size(dev, oracle, opts):
    """A region of decompress_smem_bytes(opts) decodes and visits streams written with opts; one 16 bytes smaller
    gives InvalidValue, actual 0, no byte written and no visit."""
    from gpu_util import FILL, gpu_compress
    items = [(k, v) for k, v in _inputs(opts) if len(v) >= tm.TYPE_SIZE[opts[1]]]
    raws = [v for _, v in items]
    streams, _ = gpu_compress(codec(opts), raws)
    need = dev.decompress_smem_bytes(opts)
    outs, a, s, _ = dev_decompress(dev, streams, [len(r) for r in raws], need)
    assert (s == 0).all() and outs == raws
    sums, hashes, visits, st = dev_visit(dev, streams, opts[1], region=need)
    assert (st == 0).all()
    for i, r in enumerate(raws):
        assert (int(sums[i]), int(hashes[i]), int(visits[i])) == expected_visit(r, opts[1], opts[0]), items[i][0]
    _, a, s, out = dev_decompress(dev, streams, [len(r) for r in raws], need - 16)
    assert (s == 10).all() and (a == 0).all()
    host = out.slab.cpu().numpy()
    for o, r in zip(out.offsets, raws):
        assert (host[o:o + len(r)] == FILL).all()
    _, _, visits, st = dev_visit(dev, streams, opts[1], region=need - 16)
    assert (st == 10).all() and (visits == 0).all()


# ------------------------------------------------------------------------------------------------- for_each_block
def test_for_each_block_writer_and_campaign(dev, oracle, campaign):
    names = [n for n, c in list(W.VALID.items()) + list(W.INVALID.items()) if c.codec == "cascaded"]
    streams = [c.comp for c in list(W.VALID.values()) + list(W.INVALID.values()) if c.codec == "cascaded"]
    seen = assert_visits(dev, oracle, streams + campaign[0], names + campaign[2])
    assert seen[0] >= 100 and seen[12] >= 300, seen



def test_check_walk_alone_matches_for_each_block(dev, campaign):
    """The benchmark's checking-walk kernel (tools/cascaded_device_bench.py times it on its own) accepts exactly the
    8-byte streams for_each_block visits."""
    from nvcomp_b200.batched import make_batch
    streams = [c.comp for c in list(W.VALID.values()) + list(W.INVALID.values()) if c.codec == "cascaded"]
    streams = [s for s in streams + campaign[0] if _header(s)[0] in (6, 7) and _header(s)[1] <= 1 << 25]
    region = dev.max_decompress_smem_bytes()
    _, _, _, st = dev_visit(dev, streams, 6, region=region)
    ok = torch.full((len(streams),), -1, dtype=torch.int32, device="cuda")
    dev.check_async(make_batch(streams), ok, region)
    torch.cuda.synchronize()
    ok = ok.cpu().numpy()
    assert ((ok == 1) == (st == 0)).all() and (ok >= 0).all()
    assert (st == 0).sum() >= 10 and (st == 12).sum() >= 10, ((st == 0).sum(), (st == 12).sum())


@pytest.mark.parametrize("opts", SWEEP, ids=lambda o: "p{}_t{}_r{}_d{}_bp{}".format(*o))
def test_for_each_block_encoder_streams(dev, oracle, opts):
    """The streams of every input, visited with the stream's type; with a type of another size the visit returns
    InvalidValue and calls nothing."""
    from gpu_util import gpu_compress
    items = _inputs(opts)
    streams = gpu_compress(codec(opts), [v for _, v in items])[0]
    seen = assert_visits(dev, oracle, streams, [k for k, _ in items])
    assert seen[12] == 0
    other = {1: 6, 2: 0, 4: 2, 8: 5}[tm.TYPE_SIZE[opts[1]]]
    _, _, visits, st = dev_visit(dev, streams, other)
    assert (st == 10).all() and (visits == 0).all()


# ------------------------------------------------------------------------------------------ concurrency and size
def test_mixed_warps_in_one_cta(dev, oracle):
    """Warps of the same CTAs compress one batch, decompress another and visit a third at once."""
    from gpu_util import gpu_compress
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import empty_batch, make_batch
    copts, dopts, vopts = (4096, 7, 1, 1, 1), (2048, 4, 2, 1, 1), BENCH_OPTS
    craws = [r.tobytes() for r in datagen.sorted_i64(150, seed=31)] + [v for _, v in _inputs(copts)]
    draws = [r.tobytes() for r in datagen.runlength_i32(200, seed=32)]
    vraws = [r.tobytes() for r in datagen.sorted_i64(250, seed=33)] + [v for _, v in _inputs(vopts)]
    lstreams, _ = gpu_compress(codec(copts), craws)
    dstreams, _ = gpu_compress(codec(dopts), draws)
    vstreams, _ = gpu_compress(codec(vopts), vraws)
    inp = make_batch(craws)
    cout = empty_batch(len(craws), dev.max_compressed_bytes(max(len(r) for r in craws), copts))
    comp, vcomp = make_batch(dstreams), make_batch(vstreams)
    dout = make_batch([bytes(len(r)) for r in draws])
    cst = torch.full((len(craws),), -1, dtype=torch.int32, device="cuda")
    actual = torch.full((len(draws),), -1, dtype=torch.int64, device="cuda")
    dst = torch.full((len(draws),), -1, dtype=torch.int32, device="cuda")
    sums, hashes, visits = (torch.full((len(vraws),), -1, dtype=torch.int64, device="cuda") for _ in range(3))
    vst = torch.full((len(vraws),), -1, dtype=torch.int32, device="cuda")
    region = max(dev.decompress_smem_bytes(dopts), dev.decompress_smem_bytes(vopts))
    dev.mixed_async(inp, cout, cst, copts, comp, dout, actual, dst, vcomp, sums, hashes, visits, vst, region)
    torch.cuda.synchronize()
    assert (cst.cpu().numpy() == 0).all() and (dst.cpu().numpy() == 0).all() and (vst.cpu().numpy() == 0).all()
    assert cout.to_host() == lstreams
    assert actual.cpu().tolist() == [len(r) for r in draws]
    assert dout.to_host() == draws
    u = [t.cpu().numpy().view(np.uint64) for t in (sums, hashes, visits)]
    for i, r in enumerate(vraws):
        assert (int(u[0][i]), int(u[1][i]), int(u[2][i])) == expected_visit(r, 6, 4096), i


def test_16mb_chunk(dev, oracle):
    """A 16 MB sorted int64 chunk (the largest allowed) at P = 16384: compress_warp's stream is the batched encoder's
    and the oracle's, and it round-trips through decompress_warp and for_each_block."""
    from gpu_util import gpu_compress
    opts = (16384, 6, 1, 1, 1)
    rng = np.random.default_rng(78)
    n = 1 << 24
    raw = np.cumsum(rng.integers(0, 3, n // 8) * (rng.random(n // 8) < 0.3)).astype(np.int64).tobytes()
    ls = gpu_compress(codec(opts), [raw])[0][0]
    assert ls == oracle_compress(oracle, raw, opts)
    streams, st, _ = dev_compress(dev, [raw], opts)
    assert st[0] == 0 and streams[0] == ls
    outs, a, s, _ = dev_decompress(dev, [ls], [n], dev.decompress_smem_bytes(opts), out_misalign=8)
    assert (s[0], a[0]) == (0, n) and outs[0] == raw
    assert oracle.decompress("cascaded", ls, n) == raw
    sums, hashes, visits, vst = dev_visit(dev, [ls], 6, region=dev.decompress_smem_bytes(opts))
    assert vst[0] == 0 and (int(sums[0]), int(hashes[0]), int(visits[0])) == expected_visit(raw, 6, 16384)
