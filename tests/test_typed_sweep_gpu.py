"""-m gpu: the Cascaded, Bitcomp and ANS encoders are pinned to the oracle byte for byte over their whole option space
on the edge inputs of typed_model.py.  For every configuration, one batch of edge chunks is compressed on the GPU into
guarded buffers pre-filled with a non-zero pattern (gpu_util), and:
  (a) every GPU stream equals the oracle's stream byte for byte;
  (b) the fields parsed out of it equal the plain model's prediction (a subset of configurations: the model is
      Python, and test_typed_model.py checks it against the oracle on the same inputs for every type);
  (c) it fits in CompressGetMaxOutputChunkSize (gpu_compress checks it);
  (d) the GPU decodes the GPU streams and the oracle streams back to the input, statuses 0 and sizes exact, writing
      exactly `actual` bytes (gpu_decompress checks it);
  (e) GetDecompressSizeAsync returns the input length."""
import functools

import pytest
import torch

import typed_model as tm
from test_typed_model import oracle_compress

pytestmark = pytest.mark.gpu

TYPES = sorted(tm.TYPE_SIZE)
MODEL_LAYERS = {(0, 0), (1, 0), (0, 1), (1, 1), (2, 1), (7, 7)}


@functools.lru_cache(maxsize=None)
def _cascaded_chunks(type_id, part):
    return tuple(tm.edge_chunks(type_id, part))


def _first_diff(a: bytes, b: bytes) -> int:
    return next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))


def _sweep(oracle, codec, kind, chunks, okw, model=None, parse=None, misalign=0):
    from gpu_util import gpu_compress, gpu_decompress
    from nvcomp_b200.batched import make_batch
    names = [n for n, _ in chunks]
    raws = [c for _, c in chunks]
    comps, _ = gpu_compress(codec, raws, out_misalign=misalign)                      # (c)
    ocomps = [oracle_compress(oracle, kind, r, **okw) for r in raws]
    diff = [(n, len(c), len(o), _first_diff(c, o)) for n, c, o in zip(names, comps, ocomps) if c != o]
    assert not diff, (kind, okw, "GPU != oracle (name, gpu bytes, oracle bytes, first differing byte)", diff)  # (a)
    if model is not None:
        for n, c, r in zip(names, comps, raws):
            assert parse(c) == model(r), (kind, okw, n)                             # (b)
    lens = [len(r) for r in raws]
    outs, actual, status, _ = gpu_decompress(codec, comps + ocomps, lens * 2, misalign=misalign)   # (d)
    assert (status == 0).all(), (kind, okw, [names[i % len(names)] for i in range(len(status)) if status[i]])
    assert actual.tolist() == lens * 2, (kind, okw)
    bad = [names[i % len(names)] for i, (o, r) in enumerate(zip(outs, raws * 2)) if o != r]
    assert not bad, (kind, okw, bad)
    sizes = codec.get_decompress_size(make_batch(comps))                             # (e)
    torch.cuda.synchronize()
    assert sizes.cpu().tolist() == lens, (kind, okw)


def _cascaded(oracle, type_id, part, r, d, bp, with_model):
    from nvcomp_b200._lib import CascadedOpts
    from nvcomp_b200.batched import Codec
    codec = Codec("Cascaded", opts=CascadedOpts(part, type_id, r, d, bp))
    model = (lambda raw: tm.cascaded_model(raw, type_id, part, r, d, bp)) if with_model else None
    _sweep(oracle, codec, "cascaded", _cascaded_chunks(type_id, part),
           dict(chunk_size=part, type=type_id, num_RLEs=r, num_deltas=d, use_bp=bp), model, tm.parse_cascaded)


@pytest.mark.parametrize("bp", [0, 1])
@pytest.mark.parametrize("d", range(8))
@pytest.mark.parametrize("r", range(8))
@pytest.mark.parametrize("type_id", TYPES)
def test_cascaded_grid(oracle, type_id, r, d, bp):
    """Every legal layer stack (0..7 run-length x 0..7 delta layers), both use_bp, all 8 types, 4 KB partitions."""
    _cascaded(oracle, type_id, 4096, r, d, bp, (r, d) in MODEL_LAYERS)


@pytest.mark.parametrize("layers", [(0, 0), (1, 0), (1, 1), (2, 1), (0, 7), (7, 0), (7, 7)])
@pytest.mark.parametrize("part", [512, 520, 1000, 8192, 16384])
@pytest.mark.parametrize("type_id", TYPES)
def test_cascaded_partition_sizes_sweep(oracle, type_id, part, layers):
    """Partition sizes from 512 bytes (16 decode warps) to 16 KB (1 warp for 1-byte elements with two buffers),
    including element counts that are not a multiple of 4."""
    for bp in (0, 1):
        _cascaded(oracle, type_id, part, *layers, bp, layers == (1, 1) and bp == 1)


@pytest.mark.parametrize("misalign", [0, 8])
@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("type_id", TYPES)
def test_bitcomp_sweep(oracle, type_id, algo, misalign):
    """Both algorithms, all types; stream pointers 16-byte aligned and 8- but not 16-byte aligned."""
    from nvcomp_b200._lib import BitcompOpts
    from nvcomp_b200.batched import Codec
    codec = Codec("Bitcomp", opts=BitcompOpts(algo, type_id))
    _sweep(oracle, codec, "bitcomp", tm.bitcomp_edge_chunks(type_id), dict(algo=algo, type=type_id),
           lambda raw: tm.bitcomp_model(raw, algo, type_id), tm.parse_bitcomp, misalign=misalign)


def test_ans_sweep(oracle):
    from nvcomp_b200.batched import Codec
    chunks = tm.ans_edge_chunks()
    big = [c for c in chunks if len(c[1]) > 1 << 20]          # alone: its 16 MB slot would be every chunk's
    _sweep(oracle, Codec("ANS"), "ans", [c for c in chunks if c not in big], {}, tm.ans_model, tm.parse_ans)
    _sweep(oracle, Codec("ANS"), "ans", big, {}, tm.ans_model, tm.parse_ans)
