"""GPU: the warp-level LZ4 frame device API (include/nvcomp/device/lz4frame.cuh) through the kernels of
tests/cpp/lz4frame_device_kernels.cu.  decompress_warp and decompressed_size_warp must return what the batched
nvcompBatchedLZ4Frame* calls return for every chunk and capacity -- with garbage written into each warp's region between
calls, in CTAs whose warps mix lz4::decompress_warp and lz4frame::decompress_warp, and from the library built once more
with -rdc=true."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from nvcomp_b200.batched import Codec, make_batch
from test_lz4frame_gpu import CANARY, PAD, cases, lz4f  # noqa: F401  (module fixtures)

pytestmark = pytest.mark.gpu
_P, _Z, _I = C.c_void_p, C.c_size_t, C.c_int
LIBS = {"plain": "liblz4frame_device.so", "rdc": "liblz4frame_device_rdc.so"}


def load(kind):
    path = os.path.join(ROOT, "build", "tests", LIBS[kind])
    assert os.path.exists(path), f"{path} is missing: build it with `make`"
    lib = C.CDLL(path)
    lib.lz4f_dev_decompress.argtypes = [_P] * 6 + [_Z, _I, _P]
    lib.lz4f_dev_decompressed_size.argtypes = [_P] * 3 + [_Z, _P]
    lib.lz4f_dev_mixed.argtypes = ([_P] * 6 + [_Z]) * 2 + [_P]
    return lib


def batched(cases):
    codec = Codec("LZ4Frame")
    comp = make_batch([c[1] for c in cases])
    out = make_batch([bytes([CANARY]) * (c[2] + PAD) for c in cases])
    caps = torch.tensor([c[2] for c in cases], dtype=torch.int64, device="cuda")
    out.sizes = caps
    actual, status = codec.decompress(comp, out)
    sizes = codec.get_decompress_size(comp)
    torch.cuda.synchronize()
    return out.slab.cpu().numpy(), actual.cpu().tolist(), status.cpu().tolist(), sizes.cpu().tolist()


@pytest.mark.parametrize("kind", ["plain", "rdc"])
@pytest.mark.parametrize("scribble", [0, 1])
def test_device_api_equals_batched(cases, kind, scribble):
    lib = load(kind)
    ref_slab, ref_act, ref_st, ref_sz = batched(cases)
    n = len(cases)
    comp = make_batch([c[1] for c in cases])
    out = make_batch([bytes([CANARY]) * (c[2] + PAD) for c in cases])
    caps = torch.tensor([c[2] for c in cases], dtype=torch.int64, device="cuda")
    actual = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    sizes = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    sh = torch.cuda.current_stream().cuda_stream
    assert lib.lz4f_dev_decompress(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.ptrs.data_ptr(), caps.data_ptr(),
                                   actual.data_ptr(), status.data_ptr(), n, scribble, sh) == 0
    assert lib.lz4f_dev_decompressed_size(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), sizes.data_ptr(), n, sh) == 0
    torch.cuda.synchronize()
    assert status.cpu().tolist() == ref_st
    assert actual.cpu().tolist() == ref_act
    assert sizes.cpu().tolist() == ref_sz
    assert np.array_equal(out.slab.cpu().numpy(), ref_slab)


def test_mixed_cta(cases, lz4f):
    """Even warps decode LZ4 frames, odd warps the raw LZ4 blocks of single-block frames, in the same CTAs."""
    lib = load("plain")
    frames = [c for c in cases if c[3] == 0]
    ref_slab, ref_act, ref_st, _ = batched(frames)
    from nvcomp_b200 import datagen
    data = datagen.tabular_f32(64, seed=51)
    blocks = [lz4f.compress_block(r.tobytes()) for r in data]
    fc = make_batch([c[1] for c in frames])
    fo = make_batch([bytes([CANARY]) * (c[2] + PAD) for c in frames])
    fcap = torch.tensor([c[2] for c in frames], dtype=torch.int64, device="cuda")
    fact = torch.zeros(len(frames), dtype=torch.int64, device="cuda")
    fst = torch.full((len(frames),), -1, dtype=torch.int32, device="cuda")
    bc = make_batch(blocks)
    bo = make_batch([bytes(65536)] * len(blocks))
    bcap = torch.full((len(blocks),), 65536, dtype=torch.int64, device="cuda")
    bact = torch.zeros(len(blocks), dtype=torch.int64, device="cuda")
    bst = torch.full((len(blocks),), -1, dtype=torch.int32, device="cuda")
    assert lib.lz4f_dev_mixed(fc.ptrs.data_ptr(), fc.sizes.data_ptr(), fo.ptrs.data_ptr(), fcap.data_ptr(),
                              fact.data_ptr(), fst.data_ptr(), len(frames), bc.ptrs.data_ptr(), bc.sizes.data_ptr(),
                              bo.ptrs.data_ptr(), bcap.data_ptr(), bact.data_ptr(), bst.data_ptr(), len(blocks),
                              torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert fst.cpu().tolist() == ref_st and fact.cpu().tolist() == ref_act
    assert np.array_equal(fo.slab.cpu().numpy(), ref_slab)
    assert (bst == 0).all().item() and (bact == 65536).all().item()
    slab = bo.slab.cpu().numpy()
    assert all(slab[o:o + 65536].tobytes() == data[i].tobytes() for i, o in enumerate(bo.offsets))
