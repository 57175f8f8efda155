"""-m gpu: the warp-level Deflate and Gzip device APIs (include/nvcomp/device/deflate.cuh, gzip.cuh) through the kernels
of tests/cpp/deflate_zstd_device_kernels.cu (built by `make` into build/tests/libdeflate_zstd_device.so, compiled with
-Iinclude only and linked against nothing of this library).

decompress_warp must return the batched call's status, size and bytes for every chunk and capacity, exactly, and
zlib's verdict; decompressed_size_warp must agree with GetDecompressSizeAsync; compress_warp must write the batched
encoder's streams byte for byte.  Every output sits in a guarded buffer (tests/gpu_util.py).  A warp must be able to
reuse its region for anything between calls, and warps of one CTA must be able to mix Deflate compression with
Deflate, Gzip and Zstd decoding.  The helpers here are shared with tests/test_zstd_device_gpu.py."""
import glob
import json
import os
import zlib

import numpy as np
import pytest
import torch

import deflate_writer as W
from conftest import sample_inputs
from gpu_util import FILL, _check_canaries, _guarded_batch, gpu_compress, gpu_decompress, guarded_decompress

pytestmark = pytest.mark.gpu
OK, INVALID_VALUE, CANNOT_DECOMPRESS, BAD_CHECKSUM, TOO_LARGE = 0, 10, 12, 13, 18
FMT = {"deflate": "Deflate", "gzip": "Gzip", "zstd": "Zstd"}
GZ = {"deflate": False, "gzip": True}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INPUTS = sample_inputs()

_DEV = []


def _dev():
    if not _DEV:
        from deflate_zstd_device import DeflateZstdDevice
        _DEV.append(DeflateZstdDevice())
    return _DEV[0]


def _codec(kind, algo=None):
    from nvcomp_b200._lib import DeflateOpts
    from nvcomp_b200.batched import Codec
    return Codec(FMT[kind], DeflateOpts(algo) if algo is not None else None)


# ---------------------------------------------------------------------------------------------------------------------
# helpers (shared with test_zstd_device_gpu.py)
# ---------------------------------------------------------------------------------------------------------------------
def dev_decompress(kind, chunks, caps, in_mis=0, out_mis=0, want_actual=True):
    """decompress_warp on every chunk into guarded outputs.  Returns (outputs, actual, status)."""
    def launch(comp, out, _):
        n = len(comp)
        actual = torch.full((max(n, 1),), 0x7777, dtype=torch.int64, device="cuda") if want_actual else None
        status = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
        _dev().decompress_async(kind, comp, out, actual, status)
        return actual, status
    outs, a, s, _ = guarded_decompress(launch, f"{kind} decompress_warp", chunks, caps, in_mis, out_mis)
    return outs, a, s


def match_batched(kind, chunks, caps, in_mis=0, out_mis=0, what=""):
    """decompress_warp and the batched call on the same chunks: status, actual and bytes equal, chunk by chunk.
    Returns (outputs, actual, status)."""
    outs, a, s = dev_decompress(kind, chunks, caps, in_mis, out_mis)
    bouts, ba, bs, _ = gpu_decompress(_codec(kind), chunks, caps, in_misalign=in_mis, out_misalign=out_mis)
    for i in range(len(chunks)):
        tag = (kind, what, i, in_mis, out_mis, caps[i], len(chunks[i]))
        assert int(s[i]) == int(bs[i]) and int(a[i]) == int(ba[i]), tag + (int(s[i]), int(bs[i]), int(a[i]), int(ba[i]))
        assert s[i] in (OK, CANNOT_DECOMPRESS, BAD_CHECKSUM), tag
        if s[i] == OK:
            assert outs[i] == bouts[i], tag
        else:
            assert a[i] == 0, tag
    return outs, a, s


def batched_sizes(kind, chunks):
    from nvcomp_b200.batched import make_batch
    comp = make_batch(chunks)
    n = len(chunks)
    sizes = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda")
    _codec(kind).get_decompress_size_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), sizes.data_ptr(), n,
                                           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return sizes.cpu().tolist()[:n]


def match_batched_sizes(kind, chunks, in_mis=0):
    from nvcomp_b200.batched import make_batch
    got = _dev().decompressed_size(kind, make_batch(chunks, misalign=in_mis))
    torch.cuda.synchronize()
    got = got.cpu().tolist()
    want = batched_sizes(kind, chunks)
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:10]
    return got


def edge_caps(chunks, sizes):
    """Every chunk at capacities 0, n - 1, n and n + 1 (n: its decoded size)."""
    cc, caps = [], []
    for c, n in zip(chunks, sizes):
        for cap in sorted({0, max(n - 1, 0), n, n + 1}):
            cc.append(c)
            caps.append(cap)
    return cc, caps


def run_reuse(kind, chunks, caps):
    """One warp decodes `chunks` in order with one region, overwriting it with 0xA5 after every call.  The neighbouring
    warps' regions sit right before and after it, at the codec's kDecompressSmemBytes, and must keep their canaries.
    Returns (outputs, actual, status)."""
    from nvcomp_b200.batched import make_batch
    n = len(chunks)
    comp = make_batch(chunks, misalign=3)
    out, allowed = _guarded_batch(caps, 5)
    actual = torch.full((n,), 0x7777, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    mismatch = torch.full((n,), 0xFFFF, dtype=torch.int32, device="cuda")
    canary = torch.full((2,), 0xFFFF, dtype=torch.int32, device="cuda")
    _dev().reuse_async(kind, comp, out, actual, status, mismatch, canary)
    torch.cuda.synchronize()
    assert mismatch.cpu().tolist() == [0] * n
    assert canary.cpu().tolist() == [0, 0]
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, f"{kind} reuse")
    a, s = actual.cpu().numpy(), status.cpu().numpy()
    return [host[o:o + int(x)].tobytes() for o, x in zip(out.offsets, a)], a, s


def run_huge_sizes(kind, chunks, caps):
    """A comp_bytes or capacity of 2^32 or more: decompress_warp and the batched call both return CannotDecompress
    with actual = 0 and write nothing, and decompressed_size_warp and the batched size query both return 0.  Only the
    size arrays carry the large values: the decoders reject such a chunk before reading or writing it."""
    from nvcomp_b200.batched import make_batch
    cases = []                                    # (chunk, comp_bytes, capacity)
    for c, cap in zip(chunks, caps):
        for big in (1 << 32, (1 << 32) + len(c), 1 << 40):
            cases += [(c, big, cap), (c, len(c), big)]
    n = len(cases)
    comp = make_batch([c for c, _, _ in cases])
    comp.sizes.copy_(torch.tensor([b for _, b, _ in cases], dtype=torch.int64))
    alloc = [cap if cap < 1 << 32 else len(c) + 64 for c, _, cap in cases]
    for who in ("device", "batched"):
        out, allowed = _guarded_batch(alloc, 0)
        out.sizes.copy_(torch.tensor([cap for _, _, cap in cases], dtype=torch.int64))
        actual = torch.full((n,), 0x7777, dtype=torch.int64, device="cuda")
        status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        if who == "device":
            _dev().decompress_async(kind, comp, out, actual, status)
        else:
            actual, status = _codec(kind).decompress(comp, out, max_chunk=max(alloc))
        torch.cuda.synchronize()
        host = out.slab.cpu().numpy()
        _check_canaries(host, allowed, out.offsets, f"{kind} {who} huge sizes")
        assert (host[allowed] == FILL).all(), (kind, who, "a rejected chunk wrote output")
        assert status.cpu().tolist()[:n] == [CANNOT_DECOMPRESS] * n, (kind, who)
        assert actual.cpu().tolist()[:n] == [0] * n, (kind, who)
    sizes = _dev().decompressed_size(kind, comp)
    bsizes = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    _codec(kind).get_decompress_size_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), bsizes.data_ptr(), n,
                                           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    small = [i for i, (c, b, _) in enumerate(cases) if b == len(c)]        # the size query takes no capacity
    assert [v for i, v in enumerate(sizes.cpu().tolist()) if i not in small] == [0] * (n - len(small)), kind
    assert sizes.cpu().tolist() == bsizes.cpu().tolist(), kind


def run_fused_sum(kind, chunks, raws):
    """decompress_warp + a sum by the same warp: every chunk decodes and its u64 sum of 32-bit words equals numpy's."""
    from nvcomp_b200.batched import empty_batch, make_batch
    n = len(chunks)
    comp = make_batch(chunks, misalign=1)
    out = empty_batch(n, max(len(r) for r in raws))
    out.sizes.copy_(torch.tensor([len(r) for r in raws], dtype=torch.int64))
    sums = torch.zeros(n, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    _dev().decompress_sum_async(kind, comp, out, sums, status)
    torch.cuda.synchronize()
    assert (status.cpu().numpy() == OK).all(), kind
    for i, r in enumerate(raws):
        pad = r + bytes(-len(r) % 4)
        want = int(np.frombuffer(pad, dtype="<u4").astype(np.uint64).sum(dtype=np.uint64))
        assert int(sums[i].item()) & ((1 << 64) - 1) == want, (kind, i)


def zstd_golden():
    """(raw, stream) of the committed libzstd vectors (tests/golden/zstd_manifest.json)."""
    gdir = os.path.join(ROOT, "tests", "golden")
    with open(os.path.join(gdir, "zstd_manifest.json")) as f:
        vecs = json.load(f)["vectors"]
    out = []
    for v in vecs:
        with open(os.path.join(gdir, v["raw"]), "rb") as f:
            raw = f.read()
        with open(os.path.join(gdir, v["comp"]), "rb") as f:
            out.append((raw, f.read()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# corpora
# ---------------------------------------------------------------------------------------------------------------------
def zlib_streams(gz):
    """(stream, raw): every sample input at zlib levels 0, 1, 6 and 9 under every strategy, flush-point streams and
    the hand-built streams of deflate_writer."""
    out = []
    for name in sorted(INPUTS):
        data = INPUTS[name]
        for level in (0, 1, 6, 9):
            for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
                out.append((W.compress(data, gz, level, strategy), data))
        n = len(data)
        out.append((W.compress(data, gz, 6, flushes=[(0, zlib.Z_SYNC_FLUSH), (n // 3, zlib.Z_FULL_FLUSH)]), data))
    if gz:
        out += [(s, want) for _, s, want in W.gzip_streams()]
        out += [(W.gzip_member(s, want, name=b"e", hcrc=True), want) for _, s, want in W.valid_streams()]
    else:
        out += [(s, want) for _, s, want in W.valid_streams()] + [W.code284_extra31()]
    return out


def invalid(gz):
    """(stream, zlib verdict) of deflate_writer's invalid streams."""
    if gz:
        return [(s, v) for _, s, v in W.invalid_gzip()]
    return [(s, "bad") for _, s in W.invalid_streams()]


def corruptions(gz, count=3000):
    """`count` seeded corruptions of one format from deflate_writer.corruption_corpus: (stream, cap)."""
    items = [(s, cap) for g, s, cap in W.corruption_corpus(2024, int(count * 2.3)) if g == gz]
    assert len(items) >= count, len(items)
    return items[:count]


def big_raws():
    """1 MB and 16 MB chunks."""
    from nvcomp_b200 import datagen
    big = datagen.tabular_f32(256).tobytes()                          # 16 MB
    noise = np.random.default_rng(5).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    return [big[: 1 << 20], noise, big]


def slices64k():
    """64 KB slices of every datagen dataset and the golden .raw inputs."""
    from nvcomp_b200 import datagen
    out = []
    for name, gen in datagen.DATASETS.items():
        out.append(b"".join(r.tobytes() for r in gen(2))[:65536])
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*.raw"))):
        with open(p, "rb") as f:
            out.append(f.read()[:65536])
    return out


def compress_inputs():
    rng = np.random.default_rng(17)
    base = slices64k()
    out = list(base)
    for n in (0, 1, 4, 5, 65535, 65536):
        out.append(base[0][:n])
        out.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. constants
# ---------------------------------------------------------------------------------------------------------------------
def test_constants():
    c = _dev().constants()
    assert c == {"deflate_decompress_smem": 10368, "deflate_compress_smem_0": 11152, "deflate_compress_smem_1": 68496,
                 "deflate_compress_smem_2": 11152, "deflate_compress_smem_3": 0, "deflate_compress_smem_neg1": 0,
                 "deflate_max_compress_chunk": 65536, "deflate_alignment": 16, "gzip_decompress_smem": 10368 + 1152,
                 "gzip_alignment": 16, "zstd_decompress_smem": 15872 + 1024, "zstd_alignment": 16}
    assert _dev().region_bytes() == 16896
    for n in (0, 1, 65534, 65535, 65536):
        max_out = _codec("deflate", 0).compress_get_max_output_chunk_size(n)
        assert _dev().max_compressed_bytes(n) == max_out == n + 5 * (n // 65535 + 1), n
    assert _dev().max_compressed_bytes(65537) == 0


# ---------------------------------------------------------------------------------------------------------------------
# 2. decompress_warp against the batched call and zlib
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(GZ))
def test_corpus_matches_batched_and_zlib(kind):
    gz = GZ[kind]
    items = zlib_streams(gz)
    chunks = [s for s, _ in items] + [s for s, _ in invalid(gz)]
    caps = [len(d) for _, d in items] + [1 << 16] * len(invalid(gz))
    outs, a, s = match_batched(kind, chunks, caps, what="corpus")
    for i, (c, cap) in enumerate(zip(chunks, caps)):
        verdict, want = W.zlib_expect(c, gz, cap)
        if verdict == "ok":
            assert s[i] == OK and outs[i] == want, (kind, i)
        else:
            assert s[i] == (BAD_CHECKSUM if verdict == "checksum" else CANNOT_DECOMPRESS), (kind, i, verdict, s[i])


@pytest.mark.parametrize("kind", list(GZ))
def test_corruptions_match_batched_and_zlib(kind):
    """3000 seeded corruptions of the format."""
    gz = GZ[kind]
    items = corruptions(gz)
    chunks, caps = [s for s, _ in items], [c for _, c in items]
    outs, a, s = match_batched(kind, chunks, caps, in_mis=5, out_mis=11, what="corruptions")
    for i, (c, cap) in enumerate(items):
        verdict, want = W.zlib_expect(c, gz, cap)
        if verdict == "ok":
            assert s[i] == OK and outs[i] == want, (kind, i)
        else:
            assert s[i] == (BAD_CHECKSUM if verdict == "checksum" else CANNOT_DECOMPRESS), (kind, i, verdict, s[i])


@pytest.mark.parametrize("kind", list(GZ))
def test_capacity_edges(kind):
    items = zlib_streams(GZ[kind])[::3]
    chunks, caps = edge_caps([s for s, _ in items], [len(d) for _, d in items])
    match_batched(kind, chunks, caps, what="caps")


@pytest.mark.parametrize("kind", list(GZ))
def test_misalignment(kind):
    """Input and output misalignments 0-15 (each input offset with a different output offset)."""
    items = zlib_streams(GZ[kind])[::7]
    chunks, caps = [s for s, _ in items], [len(d) for _, d in items]
    for m in range(16):
        outs, a, s = match_batched(kind, chunks, caps, in_mis=m, out_mis=(7 * m + 3) % 16, what="misalign")
        assert (s == OK).all() and outs == [d for _, d in items], (kind, m)


@pytest.mark.parametrize("kind", list(GZ))
def test_big_chunks(kind):
    raws = big_raws()
    chunks = [W.compress(r, GZ[kind], level=6) for r in raws]
    outs, a, s = match_batched(kind, chunks, [len(r) for r in raws], what="big")
    assert (s == OK).all() and outs == raws
    assert match_batched_sizes(kind, chunks) == [len(r) for r in raws]


@pytest.mark.parametrize("kind", list(GZ))
def test_null_actual(kind):
    items = zlib_streams(GZ[kind])[::5] + [(s, b"") for s, _ in invalid(GZ[kind])]
    chunks, caps = [s for s, _ in items], [max(len(d), 1) for _, d in items]
    _, _, s = dev_decompress(kind, chunks, caps, want_actual=False)
    _, _, bs, _ = gpu_decompress(_codec(kind), chunks, caps)
    assert s.tolist() == bs.tolist()


@pytest.mark.parametrize("kind", list(GZ))
def test_sizes_of_2_32_or_more(kind):
    items = zlib_streams(GZ[kind])[:6]
    run_huge_sizes(kind, [s for s, _ in items], [len(d) for _, d in items])


# ---------------------------------------------------------------------------------------------------------------------
# 3. decompressed_size_warp
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(GZ))
def test_decompressed_size(kind):
    gz = GZ[kind]
    chunks = [s for s, _ in zlib_streams(gz)] + [s for s, _ in invalid(gz)] + [s for s, _ in corruptions(gz)]
    match_batched_sizes(kind, chunks)
    match_batched_sizes(kind, chunks[::9], in_mis=13)


# ---------------------------------------------------------------------------------------------------------------------
# 4. compress_warp
# ---------------------------------------------------------------------------------------------------------------------
def dev_compress(raws, algo, in_mis=0, out_mis=0):
    """compress_warp on every chunk into guarded outputs of max_compressed_bytes(n) bytes.  Returns (streams, sizes,
    statuses, host slab, out batch)."""
    from nvcomp_b200.batched import make_batch
    inp = make_batch(raws, misalign=in_mis)
    lens = [_dev().max_compressed_bytes(len(r)) for r in raws]
    out, allowed = _guarded_batch(lens, out_mis)
    out.sizes.fill_(-1)
    status = torch.full((max(len(raws), 1),), -1, dtype=torch.int32, device="cuda")
    _dev().compress_async(inp, out, status, algo)
    torch.cuda.synchronize()
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, f"compress_warp algo {algo}")
    sizes = out.sizes.cpu().numpy()
    st = status.cpu().numpy()[:len(raws)]
    streams = [host[o:o + int(n)].tobytes() if s == OK else None for o, n, s in zip(out.offsets, sizes, st)]
    for i, (n, cap) in enumerate(zip(sizes, lens)):
        if st[i] == OK:
            assert 0 <= n <= cap, (algo, i, int(n), cap)
    return streams, sizes, st, host, out


@pytest.mark.parametrize("algo", [0, 1, 2])
def test_compress_equals_batched(algo):
    raws = compress_inputs()
    for m in range(16):
        streams, _, st, _, _ = dev_compress(raws, algo, in_mis=m, out_mis=(5 * m + 1) % 16)
        assert (st == OK).all(), (algo, m)
        want, _ = gpu_compress(_codec("deflate", algo), raws, misalign=m)
        assert streams == want, (algo, m, [i for i, (a, b) in enumerate(zip(streams, want)) if a != b][:5])
        if m == 0:
            for s, r in zip(streams, raws):
                z = zlib.decompressobj(-15)
                assert z.decompress(s) == r and z.eof, algo


@pytest.mark.parametrize("algo", [0, 1, 2])
def test_compress_argument_errors(algo):
    """n > 64 KB returns ChunkSizeTooLarge; an algo outside 0-2 returns InvalidValue; both with size 0 and nothing
    written (the guarded output of max_compressed_bytes(n) bytes is empty for n > 64 KB, and the canaries of the
    bad-algo slots are checked against an untouched FILL)."""
    raws = [bytes(65537), INPUTS["text"]]
    _, sizes, st, _, _ = dev_compress(raws, algo)
    assert st[0] == TOO_LARGE and sizes[0] == 0
    assert st[1] == OK
    for bad in (3, -1, 100):
        streams, sizes, st, host, out = dev_compress([INPUTS["text"], b""], bad)
        assert st.tolist() == [INVALID_VALUE] * 2 and sizes.tolist() == [0, 0], bad
        n = _dev().max_compressed_bytes(len(INPUTS["text"]))
        assert (host[out.offsets[0]:out.offsets[0] + n] == 0xA5).all(), bad


# ---------------------------------------------------------------------------------------------------------------------
# 5. region reuse, mixed CTA, fused sums
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(GZ))
def test_region_reuse(kind):
    """Valid, fixed-code, corrupted and short-capacity chunks through one region overwritten with 0xA5 after every
    call: every result equals the plain decode's (which equals the batched call's)."""
    gz = GZ[kind]
    items = zlib_streams(gz)[::4]
    chunks = [s for s, _ in items] + [s for s, _ in corruptions(gz, 200)]
    caps = [len(d) for _, d in items] + [c for _, c in corruptions(gz, 200)]
    chunks, caps = chunks + chunks[:20], caps + [max(c - 1, 0) for c in caps[:20]]
    outs, a, s = run_reuse(kind, chunks, caps)
    wouts, wa, ws = match_batched(kind, chunks, caps, in_mis=3, out_mis=5, what="reuse")
    assert s.tolist() == ws.tolist() and a.tolist() == wa.tolist()
    assert [o if st == OK else b"" for o, st in zip(outs, s)] == [o if st == OK else b"" for o, st in zip(wouts, ws)]
    assert (s == OK).sum() >= len(items) and (s != OK).sum() >= 20


@pytest.mark.parametrize("algo", [0, 2])
def test_mixed_cta(algo):
    """Four warps of one CTA run Deflate compression, inflate, gunzip and Zstd decode at once with one region size;
    each gets what it gets alone."""
    from nvcomp_b200.batched import make_batch
    rng = np.random.default_rng(41)
    raws = [r[:int(rng.integers(1000, len(r) + 1))] for r in slices64k() if len(r) > 1000]
    raws = (raws * 4)[:60]
    want_c, _ = gpu_compress(_codec("deflate", algo), raws)
    gzs = [W.compress(r, True, level=6) for r in raws]
    zg = zstd_golden()
    zraws, zstreams = [r for r, _ in zg], [s for _, s in zg]
    roles, keep = [], []
    inp = make_batch(raws, misalign=1)
    out, allowed = _guarded_batch([_dev().max_compressed_bytes(len(r)) for r in raws], 0)
    st = torch.full((len(raws),), -1, dtype=torch.int32, device="cuda")
    roles.append((inp, out, st)); keep.append(allowed)
    for streams, caps in ((want_c, [len(r) for r in raws]), (gzs, [len(r) for r in raws]),
                          (zstreams, [len(r) for r in zraws])):
        comp = make_batch(streams, misalign=2)
        out, allowed = _guarded_batch(caps, 9)
        actual = torch.full((len(streams),), 0x7777, dtype=torch.int64, device="cuda")
        st = torch.full((len(streams),), -1, dtype=torch.int32, device="cuda")
        roles.append((comp, out, actual, st)); keep.append(allowed)
    _dev().mixed_async(roles, algo=algo)
    torch.cuda.synchronize()
    inp, out, st = roles[0]
    host = out.slab.cpu().numpy()
    _check_canaries(host, keep[0], out.offsets, "mixed compress")
    assert (st.cpu().numpy() == OK).all()
    assert [host[o:o + int(n)].tobytes() for o, n in zip(out.offsets, out.sizes.cpu().numpy())] == want_c
    for k, want in ((1, raws), (2, raws), (3, zraws)):
        comp, out, actual, st = roles[k]
        host = out.slab.cpu().numpy()
        _check_canaries(host, keep[k], out.offsets, f"mixed role {k}")
        assert (st.cpu().numpy() == OK).all() and actual.cpu().tolist() == [len(w) for w in want], k
        assert [host[o:o + len(w)].tobytes() for o, w in zip(out.offsets, want)] == want, k


@pytest.mark.parametrize("kind", list(GZ))
def test_fused_sum(kind):
    raws = slices64k() + [INPUTS["ragged_40001"], INPUTS["short13"]]
    run_fused_sum(kind, [W.compress(r, GZ[kind], level=6) for r in raws], raws)
