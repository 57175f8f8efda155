"""-m gpu: every codec writes only inside its output chunks.  Capacities are exact (cap == len: the chunk decodes and
fills its buffer to the last byte, nothing beyond) or one byte short (cap == len - 1: the chunk fails and writes
nothing past cap).  gpu_util surrounds every chunk with canaries and checks them, and [actual, cap) after a success."""
import pytest

from conftest import sample_inputs

pytestmark = pytest.mark.gpu

INPUTS = sample_inputs()
NAMES = ["one", "short13", "zeros_1000", "random_777", "text", "ragged_40001", "runlength_i32", "sorted_i64",
         "lowentropy", "random_64k"]


def _codec(kind):
    from nvcomp_b200._lib import BitcompOpts, CascadedOpts
    from nvcomp_b200.batched import Codec
    opts = {"Cascaded": CascadedOpts(4096, 4, 1, 1, 1), "Bitcomp": BitcompOpts(1, 5)}.get(kind)
    return Codec(kind, opts=opts)


# LZ4 / Snappy streams and outputs take any address; the typed streams need 8-byte aligned ones (8 but not 16 is the
# case that takes the scalar store paths)
@pytest.mark.parametrize("kind,misalign", [("LZ4", 0), ("LZ4", 3), ("Snappy", 0), ("Snappy", 1), ("Cascaded", 0),
                                           ("Cascaded", 8), ("Bitcomp", 0), ("Bitcomp", 8), ("ANS", 0), ("ANS", 8)])
def test_exact_and_short_capacities(kind, misalign):
    from gpu_util import gpu_compress, gpu_decompress
    codec = _codec(kind)
    raws = [INPUTS[n] for n in NAMES]
    # compressed outputs: the typed encoders store whole words, so they are offset only by multiples of 8
    comps, _ = gpu_compress(codec, raws, misalign=misalign, out_misalign=misalign if misalign % 8 == 0 else 0)
    lens = [len(r) for r in raws]
    outs, actual, status, _ = gpu_decompress(codec, comps, lens, misalign=misalign)
    assert (status == 0).all(), (kind, status)
    assert actual.tolist() == lens and outs == raws
    outs, actual, status, _ = gpu_decompress(codec, comps, [n - 1 for n in lens], misalign=misalign)
    assert (status == 12).all() and (actual == 0).all(), (kind, status, actual)
