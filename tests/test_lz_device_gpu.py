"""-m gpu: the warp-level LZ4 and Snappy device APIs (include/nvcomp/device/lz4.cuh, snappy.cuh) through the kernels of
tests/cpp/lz_device_kernels.cu (built by `make` into build/tests/liblz_device.so, compiled with -Iinclude only and
linked against nothing of this library).

compress_warp must write the batched encoder's streams byte for byte; decompress_warp must return the oracle's and the
batched call's status, size and bytes for every chunk and capacity, through both decode bodies; the size queries must
agree with GetDecompressSizeAsync.  Every output sits in a guarded buffer (tests/gpu_util.py).  A warp must be able to
reuse its region for anything between calls, and warps of one CTA must be able to mix the four operations."""
import glob
import os

import numpy as np
import pytest
import torch

import lz_writer as W
from gpu_util import FILL, _check_canaries, _guarded_batch, gpu_compress, gpu_decompress, guarded_decompress
from test_lz_oracle_gpu import _caps_for, _runlength_16mb
from test_lz_writer import INVALID, VALID, SeqEmu, _dense_lz4, _dense_snappy, corpus_inputs, cpu_producers, is_light

pytestmark = pytest.mark.gpu
FMT = {"lz4": "LZ4", "snappy": "Snappy"}
KINDS = ["lz4", "snappy"]
OK, INVALID_VALUE, CANNOT_DECOMPRESS, TOO_LARGE = 0, 10, 12, 18
LZ4_TYPES = {"CHAR": 0, "UCHAR": 1, "SHORT": 2, "USHORT": 3, "INT": 4, "UINT": 5, "BITS": 0xFF}
LZ4_BAD_TYPES = [6, 7, 8, 9, 100, -1]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_DEV = []


def _dev():
    if not _DEV:
        from lz_device import LzDevice
        _DEV.append(LzDevice())
    return _DEV[0]


def _codec(kind, data_type=None):
    from nvcomp_b200._lib import LZ4Opts
    from nvcomp_b200.batched import Codec
    return Codec(FMT[kind], LZ4Opts(data_type) if data_type is not None else None)


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def dev_compress(kind, raws, data_type=0, in_mis=0, out_mis=0):
    """compress_warp on every chunk into guarded outputs of max_compressed_bytes(n) bytes.  Returns (streams, sizes,
    statuses, out batch, host slab)."""
    from nvcomp_b200.batched import make_batch
    inp = make_batch(raws, misalign=in_mis)
    lens = [_dev().max_compressed_bytes(kind, len(r)) for r in raws]
    out, allowed = _guarded_batch(lens, out_mis)
    out.sizes.fill_(-1)
    status = torch.full((max(len(raws), 1),), -1, dtype=torch.int32, device="cuda")
    _dev().compress_async(kind, inp, out, status, data_type)
    torch.cuda.synchronize()
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, f"{kind} compress_warp")
    sizes = out.sizes.cpu().numpy()
    st = status.cpu().numpy()[:len(raws)]
    streams = [host[o:o + int(n)].tobytes() if s == OK else None for o, n, s in zip(out.offsets, sizes, st)]
    for i, (o, n, cap) in enumerate(zip(out.offsets, sizes, lens)):
        if st[i] == OK:
            assert 0 <= n <= cap, (kind, i, int(n), cap)
    return streams, sizes, st, out, host


def dev_decompress(kind, chunks, caps, in_mis=0, out_mis=0):
    """decompress_warp on every chunk into guarded outputs.  Returns (outputs, actual, status)."""
    def launch(comp, out, _):
        n = len(comp)
        actual = torch.full((max(n, 1),), 0x7777, dtype=torch.int64, device="cuda")
        status = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
        _dev().decompress_async(kind, comp, out, actual, status)
        return actual, status
    outs, a, s, _ = guarded_decompress(launch, f"{kind} decompress_warp", chunks, caps, in_mis, out_mis)
    return outs, a, s


def check_verdicts(kind, chunks, caps, want, in_mis=0, out_mis=0, what=""):
    """decompress_warp against the oracle's verdicts `want` and against the batched call, chunk by chunk."""
    outs, a, s = dev_decompress(kind, chunks, caps, in_mis, out_mis)
    bouts, ba, bs, _ = gpu_decompress(_codec(kind), chunks, caps, in_misalign=in_mis, out_misalign=out_mis)
    for i, w in enumerate(want):
        tag = (kind, what, i, in_mis, out_mis, caps[i], len(chunks[i]))
        assert int(s[i]) == int(bs[i]) and int(a[i]) == int(ba[i]), tag + (int(s[i]), int(bs[i]), int(a[i]), int(ba[i]))
        if w is None:
            assert s[i] == CANNOT_DECOMPRESS and a[i] == 0, tag
        else:
            assert s[i] == OK and a[i] == len(w), tag + (int(s[i]), int(a[i]), len(w))
            assert outs[i] == w and bouts[i] == w, tag


def routes(chunks, caps):
    """(light, dense): how many chunks each decode body gets (lz_chunk_is_light, restated in test_lz_writer.py)."""
    light = sum(is_light(cap, len(c)) for c, cap in zip(chunks, caps))
    return light, len(chunks) - light


def slices64k():
    """64 KB slices of every datagen dataset and the golden .raw inputs."""
    from nvcomp_b200 import datagen
    out = []
    for name, gen in datagen.DATASETS.items():
        rows = gen(2)
        out.append(b"".join(r.tobytes() for r in rows)[:65536])
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*.raw"))):
        with open(p, "rb") as f:
            out.append(f.read()[:65536])
    return out


def edge_lengths(rng):
    """Chunks of 0, 1, 4, 5, 11, 12, 13, 16, 65 535 and 65 536 bytes (compressible and random)."""
    base = slices64k()[0]
    out = []
    for n in (0, 1, 4, 5, 11, 12, 13, 16, 65535, 65536):
        out.append(base[:n])
        out.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    return out


def golden_streams():
    """(kind, stream, raw): liblz4 default and HC-12, pyarrow Snappy."""
    out = []
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*.raw"))):
        stem = p[:-4]
        with open(p, "rb") as f:
            raw = f.read()
        for ext, kind in ((".lz4", "lz4"), (".lz4hc", "lz4"), (".snappy", "snappy")):
            if os.path.exists(stem + ext):
                with open(stem + ext, "rb") as f:
                    out.append((kind, f.read(), raw))
    return out


def big_raws(rng):
    """1 and 16 MB chunks: far matches (a random 65 535-byte block repeated) and runs of periods 1-8 bytes."""
    block = rng.integers(0, 256, 65535, dtype=np.uint8).tobytes()
    out = []
    for size in (1 << 20, 16 << 20):
        out.append((block * (size // len(block) + 1))[:size])
        parts, n = [], 0
        while n < size:
            per = int(rng.choice([1, 2, 4, 8, 3]))
            run = rng.integers(0, 256, per, dtype=np.uint8).tobytes() * int(rng.integers(100, 15000))
            parts.append(run)
            n += len(run)
        out.append(b"".join(parts)[:size])
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. constants
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_constants(kind):
    """max_compressed_bytes equals CompressGetMaxOutputChunkSize for 0..65 536 and 2^24, and is 0 where that call
    refuses (2^24 + 1); the shared-memory constants are the ones the test kernels size their regions with."""
    from nvcomp_b200.batched import NvcompError
    codec = _codec(kind)
    for n in list(range(0, 65537)) + [1 << 24]:
        assert _dev().max_compressed_bytes(kind, n) == codec.compress_get_max_output_chunk_size(n), (kind, n)
    with pytest.raises(NvcompError) as e:
        codec.compress_get_max_output_chunk_size((1 << 24) + 1)
    assert e.value.status == TOO_LARGE
    assert _dev().max_compressed_bytes(kind, (1 << 24) + 1) == 0
    c = _dev().constants(kind)
    assert c == dict(max_chunk=1 << 24, alignment=16, decompress_smem=7248, compress_smem=8192), c
    assert c["decompress_smem"] % c["alignment"] == 0 and c["compress_smem"] % c["alignment"] == 0
    assert _dev().region_bytes() == max(c["decompress_smem"], c["compress_smem"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. streams
# ---------------------------------------------------------------------------------------------------------------------
def _decodes_everywhere(kind, streams, raws, oracle, liblz4):
    import pyarrow as pa
    snap = pa.Codec("snappy")
    for i, (s, raw) in enumerate(zip(streams, raws)):
        assert oracle.decompress(kind, s, len(raw)) == raw, (kind, i)
        if kind == "lz4":
            assert liblz4.decompress(s, len(raw)) == raw, i
        elif raw:
            assert snap.decompress(s, decompressed_size=len(raw)).to_pybytes() == raw, i


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("in_mis,out_mis", [(0, 0), (3, 5), (1, 15)])
def test_streams_equal_batched(kind, in_mis, out_mis, oracle, liblz4):
    """compress_warp writes the batched encoder's stream byte for byte on dataset and golden slices and the edge
    lengths, at input and output misalignments; the streams decode with the oracle, liblz4 and pyarrow."""
    rng = np.random.default_rng(5)
    raws = slices64k() + edge_lengths(rng)
    streams, sizes, st, _, _ = dev_compress(kind, raws, in_mis=in_mis, out_mis=out_mis)
    assert (st == OK).all(), st
    want, _ = gpu_compress(_codec(kind), raws, misalign=in_mis, out_misalign=out_mis)
    for i, (s, w) in enumerate(zip(streams, want)):
        assert s == w, (kind, i, len(raws[i]), len(s), len(w))
    _decodes_everywhere(kind, streams, raws, oracle, liblz4)


@pytest.mark.parametrize("kind", KINDS)
def test_streams_16mb(kind, oracle, liblz4):
    """A 16 MB chunk equals the batched stream; 2^24 + 1 bytes return ChunkSizeTooLarge with size 0 and nothing
    written."""
    rng = np.random.default_rng(9)
    raw16 = b"".join(slices64k())
    raw16 = (raw16 * ((16 << 20) // len(raw16) + 1))[:16 << 20]
    raw16 = bytearray(raw16)
    raw16[::4097] = rng.integers(0, 256, len(raw16[::4097]), dtype=np.uint8).tobytes()
    raw16 = bytes(raw16)
    streams, _, st, _, _ = dev_compress(kind, [raw16])
    assert st[0] == OK
    want, _ = gpu_compress(_codec(kind), [raw16])
    assert streams[0] == want[0]
    _decodes_everywhere(kind, streams, [raw16], oracle, liblz4)
    too = raw16 + b"x"
    from nvcomp_b200.batched import make_batch
    inp = make_batch([too])
    out, allowed = _guarded_batch([64], 0)
    out.sizes.fill_(123)
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    _dev().compress_async(kind, inp, out, status)
    torch.cuda.synchronize()
    assert int(status.item()) == TOO_LARGE and int(out.sizes.item()) == 0
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, "too large")
    assert (host[out.offsets[0]:out.offsets[0] + 64] == FILL).all()


@pytest.mark.parametrize("in_mis", [0, 2])
def test_lz4_data_types(in_mis, oracle, liblz4):
    """Every LZ4 data_type gives the batched stream for that type; invalid types return InvalidValue, size 0 and
    write nothing."""
    rng = np.random.default_rng(3)
    raws = slices64k() + edge_lengths(rng)
    for name, t in LZ4_TYPES.items():
        streams, _, st, _, _ = dev_compress("lz4", raws, data_type=t, in_mis=in_mis)
        assert (st == OK).all(), name
        want, _ = gpu_compress(_codec("lz4", t), raws, misalign=in_mis)
        assert streams == want, name
        _decodes_everywhere("lz4", streams, raws, oracle, liblz4)
    for t in LZ4_BAD_TYPES:
        _, sizes, st, out, host = dev_compress("lz4", raws[:4], data_type=t, in_mis=in_mis)
        assert (st == INVALID_VALUE).all() and (sizes == 0).all(), (t, st, sizes)
        for o, r in zip(out.offsets, raws[:4]):
            n = _dev().max_compressed_bytes("lz4", len(r))
            assert (host[o:o + n] == FILL).all(), t


# ---------------------------------------------------------------------------------------------------------------------
# 3. verdicts
# ---------------------------------------------------------------------------------------------------------------------
def _writer_batch(kind):
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
    return chunks, caps


@pytest.mark.parametrize("kind", KINDS)
def test_writer_streams(kind, oracle):
    """The hand-built valid and invalid streams at the capacities of test_lz_oracle_gpu (exact, exact +- 1,
    4 x compressed, 64 KB), so every stream with a ratio between 1.02 and 4 runs through both decode bodies; input and
    output misalignments 0-15."""
    chunks, caps = _writer_batch(kind)
    light, dense = routes(chunks, caps)
    assert light > 50 and dense > 10, (light, dense)
    want = [oracle.decompress(kind, c, cap) for c, cap in zip(chunks, caps)]
    for k in range(16):
        check_verdicts(kind, chunks, caps, want, k, (7 * k + 3) % 16, "writer")


def _caps_of(n, m):
    return sorted({n, max(n - 1, 0), n + 1, max(n, 4 * m), 65536})


def test_corpus_golden_and_gpu_streams(oracle, liblz4):
    """The 4 000-stream seeded corruption corpus, the golden vectors (liblz4 default and HC-12, pyarrow Snappy) and
    this library's GPU-compressed streams at the oracle test's capacities: oracle and batched verdicts, sizes and
    bytes."""
    corpus = [(c, s, W.corpus_cap(i, s, n))
              for i, (c, p, k, s, n) in enumerate(W.corruption_corpus(cpu_producers(oracle, liblz4), corpus_inputs()))]
    assert len(corpus) == 4000
    for kind, s, raw in golden_streams():
        for cap in _caps_of(len(raw), len(s)):
            corpus.append((kind, s, cap))
    rng = np.random.default_rng(12)
    raws = [r[:int(rng.integers(1, len(r) + 1))] for r in slices64k() if r]
    for kind in KINDS:
        streams, _ = gpu_compress(_codec(kind), raws)
        for s, raw in zip(streams, raws):
            for cap in _caps_of(len(raw), len(s)):
                corpus.append((kind, s, cap))
    for kind in KINDS:
        items = [x for x in corpus if x[0] == kind]
        chunks, caps = [x[1] for x in items], [x[2] for x in items]
        light, dense = routes(chunks, caps)
        assert light > 300 and dense > 100, (kind, light, dense)
        want = [oracle.decompress(kind, c, cap) for c, cap in zip(chunks, caps)]
        assert sum(w is None for w in want) > 300 and sum(w is not None for w in want) > 50
        half = len(chunks) // 2
        check_verdicts(kind, chunks[:half], caps[:half], want[:half], 0, 7, "corpus a")
        check_verdicts(kind, chunks[half:], caps[half:], want[half:], 13, 2, "corpus b")


@pytest.mark.parametrize("kind", KINDS)
def test_big_chunks(kind, oracle):
    """1 and 16 MB chunks of far matches and of runs (the oracle's streams and the writer's 16 MB run-length chunk),
    at exact capacity and one byte short."""
    rng = np.random.default_rng(21)
    chunks, caps = [], []
    for raw in big_raws(rng):
        s = oracle.compress(kind, raw)
        chunks += [s, s]; caps += [len(raw), len(raw) - 1]
    c = _runlength_16mb(kind, rng)
    chunks += [c.comp, c.comp]; caps += [len(c.out), len(c.out) - 1]
    want = [oracle.decompress(kind, ch, cap) for ch, cap in zip(chunks, caps)]
    check_verdicts(kind, chunks, caps, want, 0, 0, "big")
    check_verdicts(kind, chunks, caps, want, 5, 11, "big")


# ---------------------------------------------------------------------------------------------------------------------
# 4. size queries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_decompressed_size(kind, oracle, liblz4):
    """lz4::decompressed_size_warp and snappy::decompressed_size against GetDecompressSizeAsync (and the oracle) on
    the writer streams, the corruption corpus and the golden vectors."""
    from nvcomp_b200.batched import make_batch
    chunks = [c.comp for c in {**VALID, **INVALID}.values() if c.codec == kind]
    chunks += [s for (c, p, k, s, n) in W.corruption_corpus(cpu_producers(oracle, liblz4), corpus_inputs())
               if c == kind]
    chunks += [s for k, s, raw in golden_streams() if k == kind]
    for mis in (0, 3):
        comp = make_batch(chunks, misalign=mis)
        got = _dev().decompressed_size(kind, comp).cpu().tolist()
        want = _codec(kind).get_decompress_size(comp).cpu().tolist()
        assert got == want, kind
    for i, c in enumerate(chunks):
        o = oracle.size(kind, c)
        assert got[i] == (o if o >= 0 else 0), (kind, i)


# ---------------------------------------------------------------------------------------------------------------------
# 5. region hygiene
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_region_hygiene(kind, oracle):
    """One warp decodes light, dense and failing chunks -- some fail with a staged-block copy in flight -- with one
    region, and overwrites and reads back the whole region after every call.  No byte may read back wrong (no copy
    landed late, the invalidated mbarrier is plain memory again), the next call must still give the oracle's verdict
    (its mbarrier was initialized afresh over the pattern), and the neighbouring warps' regions keep their canary."""
    from nvcomp_b200.batched import make_batch
    rng = np.random.default_rng(31)
    make = _dense_lz4 if kind == "lz4" else _dense_snappy
    chunks, caps = [], []
    for k in range(10):
        good = make(rng)
        bad = make(rng, bad_at=int(rng.integers(3000, 15000)))
        per = int(rng.choice([1, 2, 4, 8]))
        raw = rng.integers(0, 256, per, dtype=np.uint8).tobytes() * int(rng.integers(2000, 20000))
        run = oracle.compress(kind, raw)
        chunks += [good.comp, bad.comp, run, good.comp, good.comp]
        caps += [len(good.out), len(good.out) * 2, len(raw), len(good.out) - int(rng.integers(1, 9000)),
                 len(good.out)]
    want = [oracle.decompress(kind, c, cap) for c, cap in zip(chunks, caps)]
    light, dense = routes(chunks, caps)
    assert light >= 10 and dense >= 30, (light, dense)
    emu = SeqEmu()
    in_flight = [emu.fails_in_flight(kind, c, cap) for c, cap, w in zip(chunks, caps, want)
                 if w is None and not is_light(cap, len(c))]
    assert in_flight.count(1) >= 4, in_flight
    n = len(chunks)
    comp = make_batch(chunks, misalign=3)
    out, allowed = _guarded_batch(caps, 5)
    actual = torch.full((n,), 0x7777, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    mismatch = torch.full((n,), 0xFFFF, dtype=torch.int32, device="cuda")
    canary = torch.full((2,), 0xFFFF, dtype=torch.int32, device="cuda")
    _dev().hygiene_async(kind, comp, out, actual, status, mismatch, canary)
    torch.cuda.synchronize()
    assert mismatch.cpu().tolist() == [0] * n
    assert canary.cpu().tolist() == [0, 0]
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, f"{kind} hygiene")
    a, s = actual.cpu().numpy(), status.cpu().numpy()
    for i, (o, w) in enumerate(zip(out.offsets, want)):
        if w is None:
            assert s[i] == CANNOT_DECOMPRESS and a[i] == 0, i
        else:
            assert s[i] == OK and a[i] == len(w) and host[o:o + len(w)].tobytes() == w, i


# ---------------------------------------------------------------------------------------------------------------------
# 6. mixed CTA
# ---------------------------------------------------------------------------------------------------------------------
def test_mixed_cta(oracle):
    """Four warps of one CTA run LZ4 compress, Snappy compress, LZ4 decompress and Snappy decompress at once; each
    gets what it gets alone."""
    from nvcomp_b200.batched import make_batch
    rng = np.random.default_rng(41)
    raws = [r[:int(rng.integers(1000, len(r) + 1))] for r in slices64k() if len(r) > 1000]
    raws = (raws * 4)[:60]
    lz, _, _, _, _ = dev_compress("lz4", raws, data_type=LZ4_TYPES["INT"])
    sn, _, _, _, _ = dev_compress("snappy", raws)
    caps = [len(r) for r in raws]
    roles, keep = [], []
    for kind in KINDS:
        inp = make_batch(raws, misalign=1)
        lens = [_dev().max_compressed_bytes(kind, len(r)) for r in raws]
        out, allowed = _guarded_batch(lens, 0)
        st = torch.full((len(raws),), -1, dtype=torch.int32, device="cuda")
        roles.append((inp, out, st)); keep.append(allowed)
    for kind, streams in (("lz4", lz), ("snappy", sn)):
        comp = make_batch(streams, misalign=2)
        out, allowed = _guarded_batch(caps, 9)
        actual = torch.full((len(raws),), 0x7777, dtype=torch.int64, device="cuda")
        st = torch.full((len(raws),), -1, dtype=torch.int32, device="cuda")
        roles.append((comp, out, actual, st)); keep.append(allowed)
    _dev().mixed_async(roles, data_type=LZ4_TYPES["INT"])
    torch.cuda.synchronize()
    for k, (kind, want) in enumerate((("lz4", lz), ("snappy", sn))):
        inp, out, st = roles[k]
        host = out.slab.cpu().numpy()
        _check_canaries(host, keep[k], out.offsets, f"mixed {kind} compress")
        assert (st.cpu().numpy() == OK).all()
        sizes = out.sizes.cpu().numpy()
        assert [host[o:o + int(n)].tobytes() for o, n in zip(out.offsets, sizes)] == want, kind
    for k, kind in ((2, "lz4"), (3, "snappy")):
        comp, out, actual, st = roles[k]
        host = out.slab.cpu().numpy()
        _check_canaries(host, keep[k], out.offsets, f"mixed {kind} decompress")
        assert (st.cpu().numpy() == OK).all() and actual.cpu().tolist() == caps
        assert [host[o:o + n].tobytes() for o, n in zip(out.offsets, caps)] == raws, kind
