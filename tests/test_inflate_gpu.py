"""-m gpu: batched Deflate / Gzip decompression through the C ABI (nvcomp_b200.batched over libnvcomp.so), with zlib
as the oracle.  Every output buffer is guarded (gpu_util): canaries around each chunk, and nothing written in
[actual, cap) of a chunk that decodes.  The corrupted streams check that malformed input is rejected with a status."""
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch

import deflate_writer as W
from conftest import ROOT, sample_inputs

pytestmark = pytest.mark.gpu
INPUTS = sample_inputs()
FORMATS = {"Deflate": False, "Gzip": True}


def _codec(fmt):
    from nvcomp_b200.batched import Codec
    return Codec(fmt)


def _zlib_streams(gz):
    """(stream, expected bytes) of every sample input x level x strategy x memLevel, and flush-point streams."""
    out = []
    for name in sorted(INPUTS):
        data = INPUTS[name]
        for level in (0, 1, 6, 9):
            for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
                for mem_level in (1, 9):
                    out.append((W.compress(data, gz, level, strategy, mem_level), data))
        n = len(data)
        for mode in (zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
            out.append((W.compress(data, gz, 6, flushes=[(0, mode), (n // 3, mode), (n // 2, mode), (n, mode)]), data))
    return out


def _edge_streams(gz):
    if gz:
        return [(s, want) for _, s, want in W.gzip_streams()] + \
            [(W.gzip_member(s, want, name=b"e"), want) for _, s, want in W.valid_streams()]
    return [(s, want) for _, s, want in W.valid_streams()] + [W.code284_extra31()]


@pytest.fixture(scope="module")
def streams():
    return {fmt: _zlib_streams(gz) + _edge_streams(gz) for fmt, gz in FORMATS.items()}


@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("mis", [0, 1, 7])
def test_streams_decode_bit_exact(fmt, mis, streams):
    from gpu_util import gpu_decompress
    comp = [s for s, _ in streams[fmt]]
    want = [d for _, d in streams[fmt]]
    outs, actual, status, _ = gpu_decompress(_codec(fmt), comp, [len(d) for d in want], misalign=mis)
    assert (status == 0).all(), np.flatnonzero(status)[:10]
    assert [int(a) for a in actual] == [len(d) for d in want]
    bad = [i for i, (o, d) in enumerate(zip(outs, want)) if o != d]
    assert not bad, bad[:10]


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_optional_outputs_and_workspace(fmt, streams):
    """actual and/or statuses may be null; actual may alias the capacities; the workspace may be null."""
    from gpu_util import gpu_decompress
    from nvcomp_b200.batched import make_batch, empty_batch
    codec = _codec(fmt)
    items = streams[fmt][::7]
    comp = [s for s, _ in items]
    want = [d for _, d in items]
    caps = [len(d) for d in want]
    for wa, ws in ((False, True), (True, False), (False, False)):
        outs, actual, status, _ = gpu_decompress(codec, comp, caps, want_actual=wa, want_status=ws)
        assert outs == want, (wa, ws)
        if status is not None:
            assert (status == 0).all()
        if actual is not None:
            assert [int(a) for a in actual] == caps
    cb = make_batch(comp)
    stream = torch.cuda.current_stream().cuda_stream
    # actual aliases caps, no workspace
    out = empty_batch(len(comp), max(caps + [1]), fill=0)
    out.sizes.copy_(torch.tensor(caps, dtype=torch.int64))
    codec.decompress_async(cb.ptrs.data_ptr(), cb.sizes.data_ptr(), out.sizes.data_ptr(), out.sizes.data_ptr(),
                           len(comp), None, 0, out.ptrs.data_ptr(), None, stream)
    torch.cuda.synchronize()
    assert out.sizes.cpu().tolist() == caps
    assert out.to_host() == want
    # an empty batch is a no-op, whatever the pointers
    codec.decompress_async(None, None, None, None, 0, None, 0, None, None, stream)
    codec.get_decompress_size_async(None, None, None, 0, stream)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_size_query(fmt, streams):
    from nvcomp_b200.batched import make_batch
    items = [(s, len(d)) for s, d in streams[fmt][::3]]
    if FORMATS[fmt]:   # the size query cannot see a CRC-32 mismatch (it produces no bytes); it does check ISIZE
        items += [(s, 3000 if rule == "bad_crc" else 0) for rule, s, _ in W.invalid_gzip()]
    else:
        items += [(s, 0) for _, s in W.invalid_streams()]
    sizes = _codec(fmt).get_decompress_size(make_batch([s for s, _ in items]))
    torch.cuda.synchronize()
    assert sizes.cpu().tolist() == [w for _, w in items]


@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("dataset", ["tabular_f32", "runlength_i32", "sorted_i64", "lowentropy_bytes", "snappy_synth"])
def test_large_batches(fmt, dataset):
    """2000 chunks of 64 KB: many more chunks than warps, so the ticket scheduler hands them out."""
    from gpu_util import gpu_decompress
    from nvcomp_b200 import datagen
    arr = getattr(datagen, dataset)(2000)
    raw = [arr[i].tobytes() for i in range(len(arr))]
    comp = [W.compress(r, FORMATS[fmt], level=(1, 6, 9)[i % 3]) for i, r in enumerate(raw)]
    outs, actual, status, _ = gpu_decompress(_codec(fmt), comp, [len(r) for r in raw])
    assert (status == 0).all() and (actual == 65536).all()
    assert outs == raw


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_large_chunks(fmt):
    from gpu_util import gpu_decompress
    from nvcomp_b200 import datagen
    big = datagen.tabular_f32(256).tobytes()                          # 16 MB
    noise = np.random.default_rng(5).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    raw = [big[: 1 << 20], big, big[: 4 << 20] + noise]
    comp = [W.compress(r, FORMATS[fmt], level=6) for r in raw]
    outs, actual, status, _ = gpu_decompress(_codec(fmt), comp, [len(r) for r in raw])
    assert (status == 0).all() and [int(a) for a in actual] == [len(r) for r in raw]
    assert outs == raw


def test_corruption_corpus():
    """The 3000 seeded corruptions of the CPU campaign: zlib's verdict, status in {0, 12, 13}, actual 0 on failure,
    canaries intact (gpu_decompress)."""
    from gpu_util import gpu_decompress
    corpus = W.corruption_corpus(2024, 3000)
    for fmt, gz in FORMATS.items():
        items = [(s, cap) for g, s, cap in corpus if g == gz]
        outs, actual, status, _ = gpu_decompress(_codec(fmt), [s for s, _ in items], [c for _, c in items])
        for i, (s, cap) in enumerate(items):
            verdict, want = W.zlib_expect(s, gz, cap)
            assert status[i] in (0, 12, 13), (fmt, i, status[i])
            if verdict == "ok":
                assert status[i] == 0 and outs[i] == want, (fmt, i)
            else:
                assert status[i] == (13 if verdict == "checksum" else 12), (fmt, i, verdict, status[i])
                assert actual[i] == 0, (fmt, i)


def test_rejections_and_checksums():
    from gpu_util import gpu_decompress
    for fmt, gz in FORMATS.items():
        if gz:
            items = [(s, 13 if v == "checksum" else 12) for _, s, v in W.invalid_gzip()]
        else:
            items = [(s, 12) for _, s in W.invalid_streams()]
        _, actual, status, _ = gpu_decompress(_codec(fmt), [s for s, _ in items], [1 << 16] * len(items))
        assert status.tolist() == [w for _, w in items], fmt
        assert (actual == 0).all()
    # capacity one byte short
    data = INPUTS["text"]
    for fmt, gz in FORMATS.items():
        comp = W.compress(data, gz)
        outs, actual, status, _ = gpu_decompress(_codec(fmt), [comp, comp], [len(data), len(data) - 1])
        assert status.tolist() == [0, 12] and actual.tolist() == [len(data), 0] and outs[0] == data


def test_reference_gzip_example(tmp_path):
    """The reference's examples/gzip_gpu_decompression.cu, compiled unchanged (oracle/build_gzip_example.sh, run by build()):
    zlib compresses 64 KB chunks on the host, this library decodes them.  The example gives zlib an output buffer of
    one chunk, so the file must compress well (tabular_f32)."""
    from nvcomp_b200 import datagen
    exe = os.path.join(ROOT, "oracle", "_ref", "bin", "gzip_gpu_decompression")
    if not os.path.exists(exe):
        pytest.skip("gzip_gpu_decompression not built (oracle/build_gzip_example.sh needs the nvCOMP tree)")
    p = tmp_path / "f32.bin"
    datagen.tabular_f32(64).reshape(-1)[: 64 * 16384 - 777].tofile(str(p))
    r = subprocess.run([exe, "-f", str(p)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    assert "decompression validated :)" in r.stdout
