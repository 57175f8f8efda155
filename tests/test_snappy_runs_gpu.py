"""GPU: run-length Snappy streams through nvcompBatchedSnappyDecompressAsync at capacities that send them to the light
kernel (whose direct loop decodes run elements 32 at a time), alone and alternating with dense chunks.  Status,
actual bytes and output equal the oracle's; nothing outside a chunk's output is written."""
import numpy as np
import pytest

import lz_writer as W
from test_lz_oracle_gpu import _launch, _mix, _verify, _want
from test_lz_writer import is_light
from test_snappy_runs_emu import _clustered, _run_soup

pytestmark = pytest.mark.gpu


def _run_streams(oracle):
    """Run-element soups (valid, with serial elements, and corrupted) and clustered-column streams from both producers,
    each with a capacity that makes it a light chunk."""
    import pyarrow as pa
    snap = pa.Codec("snappy")
    rng = np.random.default_rng(21)
    chunks = []
    for i in range(200):
        s = _run_soup(rng, int(rng.integers(1, 400)), stop_rate=float(rng.choice([0.0, 0.0, 0.05, 0.3])),
                      start=int(rng.integers(1, 9)))
        comp = s.case().comp
        if i % 4 == 3:
            comp = W.mutate(rng, "snappy", comp)[1]
        chunks.append(comp)
    for raw in _clustered(4):
        chunks += [oracle.compress("snappy", raw), snap.compress(raw).to_pybytes()]
    caps = []
    for c in chunks:
        n = min(max(oracle.size("snappy", c), 0), 1 << 18)    # a corrupted preamble may claim gigabytes
        caps.append(max(n, 4 * len(c)))
    assert all(is_light(cap, len(c)) for c, cap in zip(chunks, caps))
    return chunks, caps


def test_run_streams_light_kernel(oracle):
    chunks, caps = _run_streams(oracle)
    want = _want(oracle, "snappy", chunks, caps)
    assert sum(w is not None for w in want) > len(want) // 2
    for in_mis, out_mis in ((0, 0), (3, 11), (13, 6)):
        r = _launch("snappy", chunks, caps, in_mis=in_mis, out_mis=out_mis)
        _verify(r, want, what=("light", in_mis, out_mis))


def test_run_streams_alternating_with_dense(oracle):
    """Run-length and dense chunks alternate in one batch: both kernels run side by side on neighbouring chunks."""
    from nvcomp_b200 import datagen
    light, lcaps = _run_streams(oracle)
    dense_raw = [r.tobytes() for r in datagen.tabular_f32(len(light), column=0)]
    chunks, caps = [], []
    for i, (c, cap) in enumerate(zip(light, lcaps)):
        d = oracle.compress("snappy", dense_raw[i])
        chunks += [c, d]
        caps += [cap, len(dense_raw[i])]
    _mix(chunks, caps, light=len(light), dense=len(light))
    want = _want(oracle, "snappy", chunks, caps)
    r = _launch("snappy", chunks, caps, in_mis=5, out_mis=9)
    _verify(r, want, what="mixed")
