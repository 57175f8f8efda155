"""GPU: zstd::compress_warp (include/nvcomp/device/zstd.cuh) through the kernels of
tests/cpp/zstd_compress_device_kernels.cu.  The frames must equal the host warp emulator's byte for byte, decode
through nvcompBatchedZstdDecompressAsync, zstd::decompress_warp and libzstd, stay inside max_compressed_bytes(n), and
come out the same at every misalignment, in a CTA whose other warps decode, and in a region the decoder has just
used."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import zstd_writer as W
from conftest import ROOT
from nvcomp_b200 import datagen
from nvcomp_b200.batched import Codec, empty_batch, make_batch
from zstd_encode_corpus import EmuZstdEncoder, corpus

pytestmark = pytest.mark.gpu

OK, INVALID_VALUE, CHUNK_TOO_LARGE = 0, 10, 18
GUARD = 0xEE
LIB_PATH = os.path.join(ROOT, "build", "tests", "libzstd_compress_device.so")
_P, _Z, _I, _U = C.c_void_p, C.c_size_t, C.c_int, C.c_uint


class Role(C.Structure):
    _fields_ = [("src", _P), ("src_bytes", _P), ("dst", _P), ("dst_bytes", _P), ("actual", _P), ("status", _P),
                ("n", _Z)]


class Lib:
    def __init__(self):
        lib = C.CDLL(LIB_PATH)
        lib.zc_dev_constants.argtypes = [_P]
        lib.zc_dev_max_compressed_bytes.argtypes = [_Z]
        lib.zc_dev_max_compressed_bytes.restype = _Z
        lib.zc_dev_compress.argtypes = [_P] * 5 + [_Z, _I, _P, _P]
        lib.zc_dev_mixed.argtypes = [_P, _U, _P]
        lib.zc_dev_reuse.argtypes = [_P] * 9 + [_Z, _P]
        self.lib = lib

    def constants(self):
        out = (C.c_size_t * 4)()
        self.lib.zc_dev_constants(out)
        return list(out)

    def bound(self, n):
        return self.lib.zc_dev_max_compressed_bytes(n)

    def compress(self, inp, out, status, algo=0, ticket=None, comp_bytes=True):
        err = self.lib.zc_dev_compress(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), out.ptrs.data_ptr(),
                                       out.sizes.data_ptr() if comp_bytes else None, status.data_ptr(), len(inp),
                                       algo, None if ticket is None else ticket.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream)
        assert err == 0, err


@pytest.fixture(scope="module")
def lib():
    return Lib()


@pytest.fixture(scope="module")
def emu():
    return EmuZstdEncoder()


@pytest.fixture(scope="module")
def zs():
    z = W.libzstd_or_none()
    if z is None:
        pytest.skip("libzstd 1.5.5 (libzstd.so.1) not available")
    return z


INPUTS = corpus()
NAMES = sorted(INPUTS)


def run(lib, chunks, in_mis=0, out_mis=0, algo=0, ticket=True, comp_bytes=True):
    """compress_warp on every chunk into guarded outputs; returns (frames, statuses, the raw output slots)."""
    inp = make_batch(chunks, misalign=in_mis)
    stride = max(lib.bound(min(len(c), 65536)) for c in chunks) + 64
    out = empty_batch(len(chunks), stride, misalign=out_mis, fill=GUARD)
    if not comp_bytes:
        out.sizes.fill_(-1)
    st = torch.full((len(chunks),), -1, dtype=torch.int32, device="cuda")
    t = torch.zeros(1, dtype=torch.int64, device="cuda") if ticket else None
    lib.compress(inp, out, st, algo=algo, ticket=t, comp_bytes=comp_bytes)
    torch.cuda.synchronize()
    sizes = out.sizes.cpu().numpy()
    slots = out.to_host([stride] * len(chunks))
    frames = [s[:max(int(n), 0)] for s, n in zip(slots, sizes)]
    return frames, st.cpu().numpy(), slots, sizes


def test_constants(lib, emu, zs):
    smem, max_chunk, align, dsmem = lib.constants()
    assert smem == emu.lib.emu_zstd_enc_smem() and smem % align == 0 and smem <= 49152
    assert max_chunk == 65536 and align == 16 and dsmem == 16896
    for n in (0, 1, 255, 256, 16384, 16385, 40001, 65535, 65536):
        assert lib.bound(n) == emu.bound(n) <= zs.lib.ZSTD_compressBound(n)
    assert lib.bound(65537) == 0


def test_gpu_equals_emulator(lib, emu):
    chunks = [INPUTS[k] for k in NAMES]
    frames, st, slots, sizes = run(lib, chunks)
    assert (st == OK).all()
    for k, c, f, s in zip(NAMES, chunks, frames, slots):
        assert f == emu.compress(c), k
        assert set(s[len(f):]) <= {GUARD}, k       # nothing past the frame, up to the guard band


@pytest.mark.parametrize("mis", [(1, 0), (0, 7), (3, 13), (15, 15)])
def test_misaligned(lib, emu, mis):
    names = ["edge:len256", "sample:price_walk", "edge:rle_literals", "sample:random_777", "edge:len0"]
    chunks = [INPUTS[k] for k in names]
    frames, st, _, _ = run(lib, chunks, in_mis=mis[0], out_mis=mis[1], ticket=False)
    assert (st == OK).all()
    assert frames == [emu.compress(c) for c in chunks]


def test_null_comp_bytes(lib, emu):
    chunks = [INPUTS["sample:gen_data3"], INPUTS["edge:len1"]]
    _, st, slots, sizes = run(lib, chunks, comp_bytes=False)
    assert (st == OK).all() and (sizes == -1).all()
    for c, s in zip(chunks, slots):
        f = emu.compress(c)
        assert s[:len(f)] == f


@pytest.mark.parametrize("algo,n,want", [(1, 1000, INVALID_VALUE), (-1, 1000, INVALID_VALUE),
                                         (0, 65537, CHUNK_TOO_LARGE), (2, 70000, INVALID_VALUE)])
def test_argument_errors(lib, algo, n, want):
    chunks = [bytes(range(256)) * (n // 256) + bytes(n % 256)]
    _, st, slots, sizes = run(lib, chunks, algo=algo)
    assert st[0] == want and sizes[0] == 0
    assert set(slots[0]) == {GUARD}


def _same_chunks(a, b, n=65536):
    """The first n bytes of every chunk of two batches are equal (compared on the device)."""
    return all(torch.equal(a.slab[int(x):int(x) + n], b.slab[int(y):int(y) + n]) for x, y in zip(a.offsets, b.offsets))


def _roundtrip(lib, zs, chunks, kind):
    from deflate_zstd_device import DeflateZstdDevice
    inp = make_batch(chunks)
    out = empty_batch(len(chunks), lib.bound(65536))
    st = torch.full((len(chunks),), -1, dtype=torch.int32, device="cuda")
    lib.compress(inp, out, st, ticket=torch.zeros(1, dtype=torch.int64, device="cuda"))
    assert (st == OK).all()
    # batched decode
    dec = empty_batch(len(chunks), 65536, fill=0)
    actual, dst = Codec("Zstd").decompress(out, dec)
    torch.cuda.synchronize()
    assert (dst == OK).all() and (actual.cpu().numpy() == [len(c) for c in chunks]).all()
    assert _same_chunks(dec, inp)
    # decompress_warp
    dec2 = empty_batch(len(chunks), 65536, fill=0)
    act2 = torch.zeros(len(chunks), dtype=torch.int64, device="cuda")
    st2 = torch.full((len(chunks),), -1, dtype=torch.int32, device="cuda")
    DeflateZstdDevice().decompress_async("zstd", out, dec2, act2, st2)
    torch.cuda.synchronize()
    assert (st2 == OK).all() and _same_chunks(dec2, inp)
    # libzstd on a sample
    frames = out.to_host()
    for i in np.random.default_rng(1).choice(len(chunks), 40, replace=False):
        assert zs.expect(frames[i], 65536) == ("ok", chunks[i]), (kind, i)
    return sum(len(f) for f in frames)


@pytest.mark.parametrize("kind", ["tabular_f32", "runlength_i32"])
def test_roundtrip_10000_chunks(lib, zs, kind):
    raw = (datagen.tabular_f32(10000) if kind == "tabular_f32" else datagen.runlength_i32(10000)).tobytes()
    chunks = [raw[i:i + 65536] for i in range(0, len(raw), 65536)]
    assert len(chunks) == 10000
    comp = _roundtrip(lib, zs, chunks, kind)
    assert comp < len(raw) / (2.3 if kind == "tabular_f32" else 60)


def test_mixed_cta(lib, emu):
    import zlib
    a = [INPUTS[k] for k in NAMES[:40]]
    d = [INPUTS[k] for k in NAMES[40:]]
    zframes = [emu.compress(c) for c in a]
    b_in = make_batch(zframes)
    b_out = empty_batch(len(a), 65536, fill=0)
    raws = [INPUTS[k] for k in NAMES[:30]]
    zc = [zlib.compressobj(6, zlib.DEFLATED, -15) for _ in raws]
    c_in = make_batch([z.compress(r) + z.flush() for z, r in zip(zc, raws)])
    c_out = empty_batch(len(raws), 65536, fill=0)
    a_in, d_in = make_batch(a), make_batch(d)
    a_out = empty_batch(len(a), lib.bound(65536), fill=GUARD)
    d_out = empty_batch(len(d), lib.bound(65536), fill=GUARD)
    dev = "cuda"
    sts = [torch.full((x,), -1, dtype=torch.int32, device=dev) for x in (len(a), len(a), len(raws), len(d))]
    acts = [torch.zeros(x, dtype=torch.int64, device=dev) for x in (len(a), len(raws))]
    roles = (Role * 4)(
        Role(a_in.ptrs.data_ptr(), a_in.sizes.data_ptr(), a_out.ptrs.data_ptr(), a_out.sizes.data_ptr(), None,
             sts[0].data_ptr(), len(a)),
        Role(b_in.ptrs.data_ptr(), b_in.sizes.data_ptr(), b_out.ptrs.data_ptr(), b_out.sizes.data_ptr(),
             acts[0].data_ptr(), sts[1].data_ptr(), len(a)),
        Role(c_in.ptrs.data_ptr(), c_in.sizes.data_ptr(), c_out.ptrs.data_ptr(), c_out.sizes.data_ptr(),
             acts[1].data_ptr(), sts[2].data_ptr(), len(raws)),
        Role(d_in.ptrs.data_ptr(), d_in.sizes.data_ptr(), d_out.ptrs.data_ptr(), d_out.sizes.data_ptr(), None,
             sts[3].data_ptr(), len(d)))
    assert lib.lib.zc_dev_mixed(roles, 7, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert all((s == OK).all() for s in sts)
    assert a_out.to_host() == zframes
    assert d_out.to_host() == [emu.compress(c) for c in d]
    assert b_out.to_host(acts[0].cpu().numpy()) == a
    assert c_out.to_host(acts[1].cpu().numpy()) == raws


def test_region_reuse(lib, emu):
    chunks = [INPUTS[k] for k in NAMES] * 2
    inp = make_batch(chunks)
    comp = empty_batch(len(chunks), lib.bound(65536), fill=GUARD)
    dec = empty_batch(len(chunks), 65536, fill=0)
    act = torch.zeros(len(chunks), dtype=torch.int64, device="cuda")
    cst = torch.full((len(chunks),), -1, dtype=torch.int32, device="cuda")
    dst = torch.full((len(chunks),), -1, dtype=torch.int32, device="cuda")
    assert lib.lib.zc_dev_reuse(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), comp.ptrs.data_ptr(),
                                comp.sizes.data_ptr(), dec.ptrs.data_ptr(), dec.sizes.data_ptr(), act.data_ptr(),
                                cst.data_ptr(), dst.data_ptr(), len(chunks),
                                torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert (cst == OK).all() and (dst == OK).all()
    assert comp.to_host() == [emu.compress(c) for c in chunks]
    assert dec.to_host(act.cpu().numpy()) == chunks
