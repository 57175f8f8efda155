"""-m gpu: LZ4 and Snappy decoding held to the oracle through the C ABI -- hand-built streams (tests/lz_writer.py) and a
seeded corruption corpus in large mixed batches, at capacities that send one stream through both decode kernels, with
independent input and output misalignments; the scheduler's edges (batch sizes around the persistent grids' warp
counts, cost buckets, workspaces, permutations); and stream order without a device-wide synchronize (the light kernel
runs on a side stream that must join the caller's), including a CUDA graph capture.

Every stream here runs in the host emulator, which has guard pages, before it runs on the GPU: the writer streams and
the CPU corpus in tests/test_lz_writer.py, the GPU-compressed corpus, the scheduler pools, the 16 MB run-length chunks and
the graph-capture batches here (_emu_check)."""
import numpy as np
import pytest
import torch

import lz_writer as W
from gpu_util import CANARY, FILL, _check_canaries, _guarded_batch
from test_lz_writer import (INVALID, VALID, SeqEmu, _dense_lz4, _dense_snappy, bucket, corpus_inputs, cpu_producers,
                            is_light)

pytestmark = pytest.mark.gpu
FMT = {"lz4": "LZ4", "snappy": "Snappy"}


_EMU = []


def _emu():
    if not _EMU:
        _EMU.append(SeqEmu())
    return _EMU[0]


def _emu_check(kind, chunks, caps, want):
    """Decode the streams in the host emulator first, each with the decoder its kernel runs (the direct loop for a
    light chunk, the block decoder for a dense one), and require the oracle's result."""
    for mode, light in (("direct", True), ("block", False)):
        idx = [i for i, (c, cap) in enumerate(zip(chunks, caps)) if is_light(cap, len(c)) == light]
        for k in range(0, len(idx), 64):
            part = idx[k:k + 64]
            got = _emu().decode_seq(kind, [chunks[i] for i in part], [caps[i] for i in part], mode)
            assert got == [want[i] for i in part], (kind, mode)


def _mix(chunks, caps, light=0, dense=0, buckets=()):
    """Minimum numbers of chunks per kernel and per cost bucket in one launched batch."""
    b = np.bincount([bucket(cap, len(c)) for c, cap in zip(chunks, caps)], minlength=6)
    assert b[:2].sum() >= light and b[2:].sum() >= dense, b
    for k in buckets:
        assert b[k] >= 1, (k, b)


def _codec(kind):
    from nvcomp_b200.batched import Codec
    return Codec(FMT[kind])


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launch(kind, chunks, caps, in_mis=0, out_mis=0, temp="exact", stream=None, codec=None):
    """Enqueue one DecompressAsync.  temp: "exact" | "none" | "short" (one byte short) | "big" (oversized, 0xFF) |
    a tensor (used as is, its full size).  Returns the pieces _verify needs; nothing is synchronized."""
    from nvcomp_b200.batched import make_batch
    codec = codec or _codec(kind)
    caps = [int(c) for c in caps]
    comp = make_batch(chunks, misalign=in_mis)
    out, allowed = _guarded_batch(caps, out_mis)
    n = len(chunks)
    tb = codec.decompress_get_temp_size(n, max(caps + [1]))
    if isinstance(temp, torch.Tensor):
        assert temp.numel() >= tb, "a workspace below DecompressGetTempSize silently takes the static stride"
        ws, wb = temp, temp.numel()
    elif temp == "none":
        ws, wb = None, 0
    elif temp == "short":
        ws = torch.zeros(tb, dtype=torch.uint8, device="cuda"); wb = tb - 1
    elif temp == "big":
        ws = torch.full((2 * tb + 4096,), 0xFF, dtype=torch.uint8, device="cuda"); wb = ws.numel()
    else:
        ws = torch.full((tb,), 0xFF, dtype=torch.uint8, device="cuda"); wb = tb
    actual = torch.full((n,), 0x7777, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    s = stream or torch.cuda.current_stream()
    s.wait_stream(torch.cuda.current_stream())                      # the uploads and fills above
    codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(), actual.data_ptr(), n,
                           None if ws is None else ws.data_ptr(), wb, out.ptrs.data_ptr(), status.data_ptr(),
                           s.cuda_stream)
    return dict(kind=kind, chunks=chunks, caps=caps, comp=comp, out=out, allowed=allowed, actual=actual,
                status=status, ws=ws)


def _want(oracle, kind, chunks, caps):
    return [oracle.decompress(kind, c, cap) for c, cap in zip(chunks, caps)]


def _verify(r, want, host=None, actual=None, status=None, what=""):
    """Per chunk: status 0 iff the oracle accepts, actual = the oracle's length (0 on failure), the oracle's bytes,
    FILL behind them, canaries intact.  host/actual/status: copies taken elsewhere (default: read r's buffers)."""
    out = r["out"]
    host = out.slab.cpu().numpy() if host is None else host
    a = r["actual"].cpu().numpy() if actual is None else actual
    s = r["status"].cpu().numpy() if status is None else status
    _check_canaries(host, r["allowed"], out.offsets, f"{r['kind']} {what}")
    for i, (o, cap, w) in enumerate(zip(out.offsets, r["caps"], want)):
        if w is None:
            assert s[i] == 12 and a[i] == 0, (what, i, int(s[i]), int(a[i]), cap)
            continue
        assert s[i] == 0 and a[i] == len(w), (what, i, int(s[i]), int(a[i]), len(w), cap)
        assert host[o:o + len(w)].tobytes() == w, (what, i, cap)
        assert (host[o + len(w):o + cap] == FILL).all(), (what, i, "wrote past actual")


def _caps_for(c):
    n = len(c.out)
    return sorted({n, max(n - 1, 0), n + 1, max(n, 4 * len(c.comp)), 65536})


# ---------------------------------------------------------------------------------------------------------------------
# writer streams and the corruption corpus
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_writer_streams_gpu(kind, oracle):
    """Every valid writer stream at capacities {exact, exact - 1, exact + 1, max(len, 4 comp), 65 536} and every invalid
    one at its capacity and 65 536, in one mixed batch per misalignment pair.  A stream with a ratio between 1.02 and 4
    goes through the dense kernel at exact capacity and the light kernel at 4 comp."""
    chunks, caps, both = [], [], 0
    for name, c in VALID.items():
        if c.codec != kind:
            continue
        n, m = len(c.out), len(c.comp)
        if 1.02 < n / max(m, 1) < 4:
            assert not is_light(n, m) and is_light(4 * m, m), name
            both += 1
        for cap in _caps_for(c):
            chunks.append(c.comp); caps.append(cap)
    for name, c in INVALID.items():
        if c.codec == kind:
            chunks += [c.comp, c.comp]; caps += [c.cap, 65536]
    assert both >= (40 if kind == "lz4" else 4), both
    want = _want(oracle, kind, chunks, caps)
    # the 1-16 MB streams in batches of their own: the small ones run as one large mixed batch.  Minimum chunks per
    # kernel (light, dense) and the buckets each batch must populate:
    groups = {(0, 1 << 17): (100, 100 if kind == "lz4" else 10, (0, 1, 5)),
              (1 << 17, 1 << 22): (4, 1 if kind == "lz4" else 0, (0,)),
              (1 << 22, 1 << 40): (2 if kind == "lz4" else 0, 0, (0,) if kind == "lz4" else ())}
    for in_mis, out_mis in [(0, 0), (1, 14), (9, 3)]:
        for (lo, hi), (nl, nd, bl) in groups.items():
            idx = [i for i, c in enumerate(caps) if lo <= c < hi]
            if not idx:
                continue
            _mix([chunks[i] for i in idx], [caps[i] for i in idx], nl, nd, bl)
            r = _launch(kind, [chunks[i] for i in idx], [caps[i] for i in idx], in_mis, out_mis)
            _verify(r, [want[i] for i in idx], what=f"mis {in_mis}/{out_mis}")


def _gpu_corpus(oracle):
    """Corrupted streams of this library's GPU compressor (on dataset slices), checked in the emulator first."""
    from gpu_util import gpu_compress
    rng = np.random.default_rng(11)
    ins = corpus_inputs()
    raws = []
    for _ in range(150):
        raw = ins[int(rng.integers(0, len(ins)))]
        a = int(rng.integers(0, max(len(raw), 1)))
        raws.append(raw[a:a + int(rng.integers(1, 16384))] or b"x")
    out = []
    for kind in ("lz4", "snappy"):
        streams, _ = gpu_compress(_codec(kind), raws)
        for raw, comp in zip(raws, streams):
            assert oracle.decompress(kind, comp, len(raw)) == raw
            for j in range(2):
                kd, bad = W.mutate(rng, kind, comp)
                cap = W.corpus_cap(len(out) + j, bad, len(raw))
                mode = "direct" if is_light(cap, len(bad)) else "block"      # the decoder its kernel runs
                assert _emu().decode(kind, bad, cap, mode, 0, 0) == oracle.decompress(kind, bad, cap)
                out.append((kind, "gpu", kd, bad, len(raw), cap))
    return out


def test_corruption_corpus_gpu(oracle, liblz4):
    """The 4000-stream seeded corpus of the CPU producers plus corrupted GPU-compressed streams, in large mixed
    batches (warps decode many chunks in a row): the oracle's verdict, size and bytes for every chunk, and the size
    query's answer."""
    corpus = [(c, p, k, s, n, W.corpus_cap(i, s, n))
              for i, (c, p, k, s, n) in enumerate(W.corruption_corpus(cpu_producers(oracle, liblz4), corpus_inputs()))]
    corpus += _gpu_corpus(oracle)
    for kind in ("lz4", "snappy"):
        items = [x for x in corpus if x[0] == kind]
        chunks, caps = [x[3] for x in items], [x[5] for x in items]
        want = _want(oracle, kind, chunks, caps)
        assert sum(w is None for w in want) > 300 and sum(w is not None for w in want) > 50
        half = len(chunks) // 2
        for sl, (im, om) in ((slice(0, half), (0, 7)), (slice(half, None), (13, 2))):
            _mix(chunks[sl], caps[sl], light=300, dense=100, buckets=(0, 1, 5))
            r = _launch(kind, chunks[sl], caps[sl], im, om)
            _verify(r, want[sl], what=f"corpus {im}/{om}")
        _check_sizes(kind, chunks, oracle)


def _check_sizes(kind, chunks, oracle):
    from nvcomp_b200.batched import make_batch
    got = _codec(kind).get_decompress_size(make_batch(chunks, misalign=3)).cpu().tolist()
    for i, c in enumerate(chunks):
        o = oracle.size(kind, c)
        assert got[i] == (o if o >= 0 else 0), (kind, i, got[i], o)


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_size_query_writer_streams(kind, oracle):
    _check_sizes(kind, [c.comp for c in {**VALID, **INVALID}.values() if c.codec == kind], oracle)


# ---------------------------------------------------------------------------------------------------------------------
# scheduler
# ---------------------------------------------------------------------------------------------------------------------
_POOLS = {}


def _pool(kind, oracle):
    """Small streams by class: dense (exact capacity), light run-length, light incompressible, and dense ones of every
    compressed-size bucket."""
    if kind not in _POOLS:
        _POOLS[kind] = _make_pool(kind, oracle)
    return _POOLS[kind]


def _make_pool(kind, oracle):
    rng = np.random.default_rng(23)
    mk = (lambda n: _dense_lz4(rng, n)) if kind == "lz4" else (lambda n: _dense_snappy(rng, n))
    dense = [mk(int(rng.integers(300, 3000))) for _ in range(12)]
    runs = []
    for _ in range(6):
        per = int(rng.choice([1, 2, 4, 8]))
        raw = rng.integers(0, 256, per, dtype=np.uint8).tobytes() * int(rng.integers(200, 2000))
        runs.append((oracle.compress(kind, raw), raw))
    incomp = []
    for _ in range(6):
        raw = rng.integers(0, 256, int(rng.integers(100, 3000)), dtype=np.uint8).tobytes()
        incomp.append((oracle.compress(kind, raw), raw))
    by_bucket = {b: [] for b in range(6)}
    for c in dense:
        by_bucket[bucket(len(c.out), len(c.comp))].append((c.comp, c.out))
    for comp, raw in runs:
        by_bucket[bucket(len(raw), len(comp))].append((comp, raw))
    for comp, raw in incomp:
        by_bucket[bucket(len(raw), len(comp))].append((comp, raw))
    for target in (20000, 36000, 52000):                           # dense buckets 4, 3, 2 (16 KB steps of input)
        for _ in range(2):
            c = mk(target * 2)
            while len(c.comp) < target:
                c = mk(int(len(c.out) * 1.2))
            by_bucket[bucket(len(c.out), len(c.comp))].append((c.comp, c.out))
    assert all(by_bucket[b] for b in range(6)), {b: len(v) for b, v in by_bucket.items()}
    items = [x for v in by_bucket.values() for x in v]
    _emu_check(kind, [c for c, _ in items], [len(r) for _, r in items], [r for _, r in items])
    return by_bucket


def _batch_from(by_bucket, buckets, n, rng):
    items = []
    for i in range(n):
        b = buckets[i % len(buckets)]
        items.append(by_bucket[b][int(rng.integers(0, len(by_bucket[b])))])
    return [c for c, _ in items], [len(r) for _, r in items], [r for _, r in items]


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_batch_sizes_around_the_grid(kind, oracle):
    """Batch sizes SMs * 4 * k + {-1, 0, +1}, k = 1..10: every CTAs-per-SM setting of both persistent grids has a
    batch whose chunk count is one below, at and one above its warp count (where the static first chunk hands over to
    ticket + static_stride).  All-light, all-dense and mixed batches."""
    rng = np.random.default_rng(31)
    pool = _pool(kind, oracle)
    sms = _sms()
    mixes = {"light": [0, 1], "dense": [5], "mixed": [0, 1, 5]}     # small chunks: the costly buckets are below
    for k in range(1, 11):
        for d in (-1, 0, 1):
            n = sms * 4 * k + d
            for mix, bl in mixes.items():
                chunks, caps, want = _batch_from(pool, bl, n, rng)
                assert {bucket(c, len(x)) for x, c in zip(chunks, caps)} == set(bl)
                r = _launch(kind, chunks, caps, int(rng.integers(0, 16)), int(rng.integers(0, 16)))
                _verify(r, want, what=f"n={n} {mix}")


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_cost_buckets(kind, oracle):
    """All six buckets populated, and batches with empty buckets between populated ones."""
    rng = np.random.default_rng(37)
    pool = _pool(kind, oracle)
    for bl in ([0, 1, 2, 3, 4, 5], [0, 5], [1, 3], [2, 5], [0, 2, 4], [1, 2, 5], [3], [5, 0, 3]):
        chunks, caps, want = _batch_from(pool, bl, 700, rng)
        counts = np.bincount([bucket(c, len(x)) for x, c in zip(chunks, caps)], minlength=6)
        assert all(counts[b] >= 100 for b in bl) and counts.sum() == counts[bl].sum(), counts
        _verify(_launch(kind, chunks, caps), want, what=f"buckets {bl}")


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_workspaces(kind, oracle):
    """No workspace (static stride), one byte short (static stride), exact, and oversized and pre-filled with 0xFF;
    one workspace reused by two back-to-back calls; a random permutation of a batch gives the same per-chunk
    results."""
    rng = np.random.default_rng(41)
    pool = _pool(kind, oracle)
    chunks, caps, want = _batch_from(pool, [0, 1, 2, 3, 4, 5], 3000, rng)
    for t in ("none", "short", "exact", "big"):
        _verify(_launch(kind, chunks, caps, 2, 5, temp=t), want, what=f"temp {t}")
    codec = _codec(kind)
    tb = codec.decompress_get_temp_size(len(chunks), 65536)
    ws = torch.full((tb,), 0xFF, dtype=torch.uint8, device="cuda")
    c2, caps2, want2 = _batch_from(pool, [5, 1, 3], 2500, rng)
    r1 = _launch(kind, chunks, caps, temp=ws, codec=codec)
    r2 = _launch(kind, c2, caps2, temp=ws, codec=codec)
    _verify(r1, want, what="reuse 1")
    _verify(r2, want2, what="reuse 2")
    perm = rng.permutation(len(chunks))
    rp = _launch(kind, [chunks[i] for i in perm], [caps[i] for i in perm], 7, 7)
    _verify(rp, [want[i] for i in perm], what="permutation")


# ---------------------------------------------------------------------------------------------------------------------
# stream order: nothing below synchronizes the device before it looks at the outputs
# ---------------------------------------------------------------------------------------------------------------------
def _runlength_16mb(kind, rng):
    """A 16 MB chunk of runs (periods 1-8 bytes, up to 60 KB long) -- light-kernel work that takes a while."""
    if kind == "lz4":
        w = W.Lz4()
        while len(w.out) < (16 << 20) - 70000:
            per = int(rng.choice([1, 2, 4, 8, 3]))
            w.seq(rng.integers(0, 256, per, dtype=np.uint8).tobytes(), per, int(rng.integers(1000, 60000)))
        return w.end(b"end").case()
    s = W.Snappy()
    while len(s.out) < (16 << 20) - 70000:
        per = int(rng.choice([1, 2, 4, 8, 3]))
        s.lit(rng.integers(0, 256, per, dtype=np.uint8).tobytes())
        for _ in range(int(rng.integers(10, 300))):
            s.copy2(per, 64)
    return s.case()


def _snapshot(r, s):
    """Device-to-device copies of the outputs, sizes and statuses, enqueued on stream s."""
    with torch.cuda.stream(s):
        return r["out"].slab.clone(), r["actual"].clone(), r["status"].clone()


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_stream_order(kind, oracle):
    rng = np.random.default_rng(43)
    pool = _pool(kind, oracle)
    big = [_runlength_16mb(kind, rng) for _ in range(2)]
    _emu_check(kind, [c.comp for c in big], [len(c.out) for c in big], [c.out for c in big])
    heavy = [big[i % 2].comp for i in range(16)]
    heavy_out = [big[i % 2].out for i in range(16)]
    d_chunks, d_caps, d_want = _batch_from(pool, [2, 3, 4, 5], 64, rng)
    chunks, caps, want = heavy + d_chunks, [len(o) for o in heavy_out] + d_caps, heavy_out + d_want
    assert sum(is_light(c, len(x)) for x, c in zip(chunks, caps)) == 16

    # 1. the light list carries almost all the work; a copy enqueued right behind the call on the same stream
    s = torch.cuda.Stream()
    r = _launch(kind, chunks, caps, stream=s)
    snap = _snapshot(r, s)
    s.synchronize()
    _verify(r, want, host=snap[0].cpu().numpy(), actual=snap[1].cpu().numpy(), status=snap[2].cpu().numpy(),
            what="copy behind the call")

    # 2. two back-to-back calls on one stream sharing one workspace (the second call's counter reset must wait for
    # the first call's light kernel)
    codec = _codec(kind)
    c2, caps2, want2 = _batch_from(pool, [0, 1, 5], 4000, rng)
    # sized for the larger batch: both calls use the ticket lists (a short workspace would fall back to the static
    # stride and never reset the shared counters; _launch asserts it is large enough)
    ws = torch.empty(codec.decompress_get_temp_size(max(len(chunks), len(c2)), 1 << 24), dtype=torch.uint8,
                     device="cuda")
    s = torch.cuda.Stream()
    r1 = _launch(kind, chunks, caps, temp=ws, stream=s, codec=codec)
    r2 = _launch(kind, c2, caps2, temp=ws, stream=s, codec=codec)
    snap1, snap2 = _snapshot(r1, s), _snapshot(r2, s)
    s.synchronize()
    _verify(r1, want, *(x.cpu().numpy() for x in snap1), what="back-to-back 1")
    _verify(r2, want2, *(x.cpu().numpy() for x in snap2), what="back-to-back 2")

    # 3. two streams decoding different batches at the same time (they share the device's side stream)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ra = _launch(kind, chunks, caps, stream=sa)
    rb = _launch(kind, c2, caps2, stream=sb, in_mis=4, out_mis=12)
    snapa, snapb = _snapshot(ra, sa), _snapshot(rb, sb)
    sb.synchronize()
    _verify(rb, want2, *(x.cpu().numpy() for x in snapb), what="stream b")
    sa.synchronize()
    _verify(ra, want, *(x.cpu().numpy() for x in snapa), what="stream a")
    torch.cuda.synchronize()


def _twins(kind, rng, n):
    """Two batches of valid streams with equal compressed sizes and different bytes (same structure, other
    literals)."""
    out = ([], [])
    for i in range(n):
        seed = int(rng.integers(0, 1 << 30))
        for t in (0, 1):
            r1, r2 = np.random.default_rng(seed), np.random.default_rng(seed * 7 + t + 1)
            if kind == "lz4":
                w = W.Lz4().seq(r2.integers(0, 256, 64, dtype=np.uint8).tobytes(), 8, 8)
                for _ in range(int(r1.integers(1, 400))):
                    lits = r2.integers(0, 256, int(r1.integers(0, 6)), dtype=np.uint8).tobytes()
                    w.seq(lits, int(r1.integers(1, 64)), int(r1.integers(4, 3000 if i % 3 == 0 else 12)))
                c = w.end(r2.integers(0, 256, 5, dtype=np.uint8).tobytes()).case()
            else:
                s = W.Snappy().lit(r2.integers(0, 256, 64, dtype=np.uint8).tobytes())
                for _ in range(int(r1.integers(1, 400))):
                    s.lit(r2.integers(0, 256, int(r1.integers(1, 6)), dtype=np.uint8).tobytes())
                    s.copy2(int(r1.integers(1, 64)), int(r1.integers(1, 65 if i % 3 == 0 else 12)))
                c = s.case()
            out[t].append(c)
    for a, b in zip(*out):
        assert len(a.comp) == len(b.comp) and len(a.out) == len(b.out)
    return out


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_graph_capture(kind, oracle):
    """decompress_async captured in a CUDA graph (the fork onto the side stream and the join are captured with it),
    replayed twice with new input bytes copied into the same buffers in between."""
    from nvcomp_b200.batched import make_batch
    rng = np.random.default_rng(47)
    a, b = _twins(kind, rng, 600)
    for t in (a, b):
        _emu_check(kind, [c.comp for c in t], [len(c.out) for c in t], [c.out for c in t])
    codec = _codec(kind)
    caps = [len(c.out) for c in a]
    comp = make_batch([c.comp for c in a], misalign=3)
    out, allowed = _guarded_batch(caps, 11)
    n = len(a)
    tb = codec.decompress_get_temp_size(n, max(caps))
    ws = torch.empty(tb, dtype=torch.uint8, device="cuda")
    actual = torch.zeros(n, dtype=torch.int64, device="cuda")
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    call = lambda: codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(),
                                          actual.data_ptr(), n, ws.data_ptr(), tb, out.ptrs.data_ptr(),
                                          status.data_ptr(), torch.cuda.current_stream().cuda_stream)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()                                                    # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    fill = torch.from_numpy(np.where(allowed, FILL, CANARY).astype(np.uint8)).cuda()
    r = dict(kind=kind, caps=caps, out=out, allowed=allowed, actual=actual, status=status)
    for batch in (a, b, a):
        comp.slab.copy_(make_batch([c.comp for c in batch], misalign=3).slab)
        out.slab.copy_(fill)
        actual.fill_(0x7777)
        status.fill_(-1)
        g.replay()
        snap = _snapshot(r, torch.cuda.current_stream())
        torch.cuda.current_stream().synchronize()
        _verify(r, [c.out for c in batch], *(x.cpu().numpy() for x in snap), what="graph replay")
    torch.cuda.synchronize()
