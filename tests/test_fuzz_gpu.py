"""-m gpu: robustness.  Random garbage and bit-flipped valid streams must never fault or hang; every chunk
ends with status Success (and then the exact size) or CannotDecompress with size 0 (reference
CHANGELOG.md:160-164: undecodable input yields size 0 + an error status, never an illegal access).  For Cascaded,
Bitcomp and ANS the verdict, size and bytes must be the oracle's.
tools: run this file under `compute-sanitizer --tool memcheck` to check for out-of-bounds accesses."""
import numpy as np
import pytest
import torch

from conftest import sample_inputs

pytestmark = pytest.mark.gpu
INPUTS = sample_inputs()


def _codec(kind):
    from nvcomp_b200._lib import BitcompOpts, CascadedOpts
    from nvcomp_b200.batched import Codec
    opts = {"Cascaded": CascadedOpts(4096, 4, 2, 1, 1), "Bitcomp": BitcompOpts(0, 5)}.get(kind)
    return Codec(kind, opts=opts)


@pytest.mark.parametrize("kind", ["LZ4", "Snappy", "Cascaded", "Bitcomp", "ANS"])
def test_garbage_and_bitflips(kind, oracle):
    from gpu_util import gpu_compress, gpu_decompress
    rng = np.random.default_rng(2024)
    codec = _codec(kind)
    names = ["text", "runlength_i32", "price_walk", "lowentropy", "sorted_i64", "period7"]
    raws = [INPUTS[n][: len(INPUTS[n]) // 8 * 8] for n in names]
    goods, _ = gpu_compress(codec, raws)
    chunks, caps, expect = [], [], []
    # 1. pure garbage of assorted lengths (8-byte aligned starts via make_batch)
    for n in [1, 2, 3, 7, 16, 64, 257, 1000, 4096, 20000]:
        chunks.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes()); caps.append(65536); expect.append(None)
    # 2. valid streams with random bit flips / truncations / extensions
    for g, r in zip(goods, raws):
        for _ in range(6):
            b = bytearray(g)
            for pos in rng.integers(0, len(b), rng.integers(1, 8)):
                b[pos] ^= 1 << rng.integers(0, 8)
            chunks.append(bytes(b)); caps.append(len(r)); expect.append(None)
        chunks.append(g[: rng.integers(1, len(g))]); caps.append(len(r)); expect.append(None)
        chunks.append(g + b"\x00" * 5); caps.append(len(r)); expect.append(None)
        chunks.append(g); caps.append(len(r)); expect.append(r)           # untouched control
    outs, actual, status, _ = gpu_decompress(codec, chunks, caps)
    for i, (c, cap, e) in enumerate(zip(chunks, caps, expect)):
        assert status[i] in (0, 12), (kind, i, status[i])
        if status[i] == 12:
            assert actual[i] == 0
        else:
            assert actual[i] <= cap
        if e is not None:
            assert status[i] == 0 and outs[i] == e, (kind, i)
        if kind in ("Cascaded", "Bitcomp", "ANS"):
            # the typed formats: the oracle's verdict and bytes on every chunk
            w = oracle.decompress(kind.lower(), c, cap)
            assert (int(status[i]), int(actual[i])) == ((12, 0) if w is None else (0, len(w))), (kind, i)
            assert w is None or outs[i] == w, (kind, i)
