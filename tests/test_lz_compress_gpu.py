"""-m gpu: the LZ4 and Snappy encoders on the GPU -- nvcompBatched{LZ4,Snappy}CompressAsync at every LZ4 data_type
and the warp-level compress_warp of include/nvcomp/device/{lz4,snappy}.cuh -- held byte for byte to the same
encoder run in the host warp emulator (tests/emu/emu_lz_encode.cpp), and to the stream-rules model of
tests/lz_encode_model.py where the emulator would be too slow.

The matcher's hash inserts are deterministic, so a chunk's stream depends on its bytes alone: not on its batch
position, its alignment, the temp buffer, the call or the hardware's choice among same-bucket stores.  Every output
sits in a guarded buffer (tests/gpu_util.py)."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import lz_encode_model as M
from gpu_util import FILL, _check_canaries, _guarded_batch
from nvcomp_b200 import datagen
from test_lz_device_gpu import LZ4_TYPES, OK, _codec, dev_compress

pytestmark = pytest.mark.gpu
STEP = {"CHAR": 1, "UCHAR": 1, "BITS": 1, "SHORT": 2, "USHORT": 2, "INT": 4, "UINT": 4}
# (kind, data_type name or None for Snappy)
CALLS = [("lz4", t) for t in LZ4_TYPES] + [("snappy", None)]

INPUTS = M.corpus()
NAMES = sorted(INPUTS)


@pytest.fixture(scope="module")
def enc():
    return M.EmuLzEncoder()


def _emulate(enc, kind, raws, step=1):
    """The emulator's streams; ctypes drops the GIL, so the chunks run on every host core."""
    with ThreadPoolExecutor(os.cpu_count() or 4) as pool:
        return list(pool.map(lambda r: enc.compress(kind, r, step), raws))


def batched(kind, raws, data_type=None, in_mis=0, out_mis=0, temp=True, max_chunk=None):
    """nvcompBatched<Codec>CompressAsync into guarded output slots of GetMaxOutputChunkSize(max_chunk) bytes.
    Returns (streams, sizes, out batch, host slab, slot bytes)."""
    from nvcomp_b200.batched import make_batch
    codec = _codec(kind, LZ4_TYPES[data_type] if data_type else None)
    inp = make_batch(raws, misalign=in_mis)
    n = len(raws)
    if max_chunk is None:
        max_chunk = max([len(r) for r in raws] + [1])
    max_out = codec.compress_get_max_output_chunk_size(max_chunk)
    tb = codec.compress_get_temp_size(n, max_chunk) if temp else 0
    tbuf = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
    out, allowed = _guarded_batch([max_out] * n, out_mis)
    out.sizes.fill_(-1)
    codec.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), max_chunk, n, tbuf.data_ptr() if temp else 0,
                         tb, out.ptrs.data_ptr(), out.sizes.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, f"{kind} {data_type} compress")
    sizes = out.sizes.cpu().numpy()
    assert ((sizes >= 0) & (sizes <= max_out)).all(), (kind, data_type, sizes.min(), sizes.max(), max_out)
    for o, s in zip(out.offsets, sizes):
        assert (host[o + int(s):o + max_out] == FILL).all(), f"{kind} {data_type}: a chunk wrote past its size {s}"
    return [host[o:o + int(s)].tobytes() for o, s in zip(out.offsets, sizes)], sizes, out, host, max_out


# ---------------------------------------------------------------------------------------------------------------------
# the corpus, byte for byte
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,data_type", CALLS)
def test_batched_equals_emulator(kind, data_type, enc):
    raws = [INPUTS[k] for k in NAMES]
    step = STEP[data_type] if data_type else 1
    want = _emulate(enc, kind, raws, step)
    got, *_ = batched(kind, raws, data_type)
    for name, g, w in zip(NAMES, got, want):
        assert g == w, (kind, data_type, name, len(g), len(w))


@pytest.mark.parametrize("kind,data_type", CALLS)
def test_compress_warp_equals_emulator(kind, data_type, enc):
    raws = [INPUTS[k] for k in NAMES]
    step = STEP[data_type] if data_type else 1
    want = _emulate(enc, kind, raws, step)
    got, _, st, _, _ = dev_compress(kind, raws, data_type=LZ4_TYPES[data_type] if data_type else 0)
    assert (st == OK).all(), st
    for name, g, w in zip(NAMES, got, want):
        assert g == w, (kind, data_type, name, len(g), len(w))


# ---------------------------------------------------------------------------------------------------------------------
# 2 000 x 64 KB per dataset
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lz4", "snappy"])
@pytest.mark.parametrize("dataset", sorted(datagen.DATASETS))
def test_datasets_decode_and_sample_equals_emulator(dataset, kind, enc, liblz4):
    import pyarrow as pa
    snap = pa.Codec("snappy")
    data = datagen.DATASETS[dataset](2000)
    raws = [r.tobytes() for r in data]
    got, *_ = batched(kind, raws)
    for i, (g, r) in enumerate(zip(got, raws)):
        if kind == "lz4":
            assert liblz4.decompress(g, len(r)) == r, (dataset, i)
        else:
            assert snap.decompress(g, decompressed_size=len(r)).to_pybytes() == r, (dataset, i)
    pick = np.random.default_rng(len(dataset)).choice(len(raws), 64, replace=False)
    want = _emulate(enc, kind, [raws[i] for i in pick])
    for i, w in zip(pick, want):
        assert got[i] == w, (dataset, kind, int(i))


# ---------------------------------------------------------------------------------------------------------------------
# a stream depends on its input alone
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,data_type", [("lz4", "CHAR"), ("lz4", "INT"), ("snappy", None)])
def test_same_bytes_everywhere(kind, data_type, enc):
    """One chunk at every position of a batch of others, at input and output misalignments 0-15, with and without
    a temp buffer (the work ticket or a static stride), and across two calls, gives the emulator's stream."""
    step = STEP[data_type] if data_type else 1
    probe = INPUTS["slice:lz4_mixed"]
    want = enc.compress(kind, probe, step)
    others = [r.tobytes() for r in datagen.tabular_f32(40, seed=21)]
    for pos in (0, 1, 17, 40):
        raws = others[:pos] + [probe] + others[pos:]
        for temp in (True, False):
            got, *_ = batched(kind, raws, data_type, temp=temp)
            assert got[pos] == want, (pos, temp)
    for k in range(16):
        got, *_ = batched(kind, [probe, INPUTS["sample:price_walk"], probe], data_type, in_mis=k, out_mis=15 - k)
        assert got[0] == want and got[2] == want, k
    first, *_ = batched(kind, others + [probe] * 8, data_type)
    second, *_ = batched(kind, others + [probe] * 8, data_type)
    assert first == second and first[-8:] == [want] * 8


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_16mb_chunk_passes_model(kind, liblz4):
    """A 16 MB chunk from both APIs: the same stream, which passes the stream-rules model and decodes."""
    rng = np.random.default_rng(16)
    raw = b"".join(INPUTS[f"slice:{d}"] for d in sorted(datagen.DATASETS))
    raw = bytearray((raw * ((16 << 20) // len(raw) + 1))[:16 << 20])
    raw[::4099] = rng.integers(0, 256, len(raw[::4099]), dtype=np.uint8).tobytes()
    raw = bytes(raw)
    got, *_ = batched(kind, [raw])
    warp, _, st, _, _ = dev_compress(kind, [raw])
    assert st[0] == OK and warp[0] == got[0]
    M.check(kind, got[0], raw)
    if kind == "lz4":
        assert liblz4.decompress(got[0], len(raw)) == raw


@pytest.mark.parametrize("kind,data_type", CALLS)
def test_empty_chunk(kind, data_type):
    """A 0-byte chunk in a batch: LZ4 writes the one empty token 0x00, Snappy the preamble varint 0."""
    raws = [INPUTS["sample:text"], b"", INPUTS["size:13"]]
    step = STEP[data_type] if data_type else 1
    got, *_ = batched(kind, raws, data_type)
    warp, _, st, _, _ = dev_compress(kind, raws, data_type=LZ4_TYPES[data_type] if data_type else 0)
    assert (st == OK).all() and warp == got
    assert got[1] == b"\x00"
    for g, r in zip(got, raws):
        M.check(kind, g, r, step)


@pytest.mark.parametrize("kind", ["lz4", "snappy"])
def test_chunk_over_max_chunk_writes_nothing(kind, enc):
    """A chunk longer than the call's max_chunk gets size 0 and writes nothing into its slot, which was sized for
    max_chunk; the chunks around it are compressed as usual."""
    small = [INPUTS["size:4097"], INPUTS["sample:text"][:4000]]
    for big in (INPUTS["slice:random_bytes"], INPUTS["size:4097"] + b"\x00"):
        raws = [small[0], big, small[1]]
        got, sizes, out, host, slot = batched(kind, raws, max_chunk=4097)
        assert int(sizes[1]) == 0
        assert (host[out.offsets[1]:out.offsets[1] + slot] == FILL).all()
        assert got[0] == enc.compress(kind, small[0]) and got[2] == enc.compress(kind, small[1])
