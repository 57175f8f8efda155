"""-m gpu: Cascaded, Bitcomp and ANS batched codecs (CUDA, through the C ABI).  The reference bitstreams
are undocumented (parity unpinned at the stream level), so the checks are: GPU round trip is bit-exact;
GPU streams decode with the independent CPU oracle; oracle-encoded streams decode on the GPU; malformed
streams fail cleanly."""
import numpy as np
import pytest
import torch

from conftest import sample_inputs

pytestmark = pytest.mark.gpu

INPUTS = sample_inputs()
NAMES = [n for n in sorted(INPUTS)]
TS = {0: 1, 1: 1, 2: 2, 3: 2, 4: 4, 5: 4, 6: 8, 7: 8}


def _raws(ts):
    return [INPUTS[n][: len(INPUTS[n]) // ts * ts] for n in NAMES]


def _roundtrip(codec, kind, raws, oracle, okw):
    from gpu_util import gpu_compress, gpu_decompress
    comps, cb = gpu_compress(codec, raws)
    max_out = codec.compress_get_max_output_chunk_size(max(len(r) for r in raws))
    assert max(len(c) for c in comps) <= max_out
    # GPU stream -> CPU oracle
    for n, c, r in zip(NAMES, comps, raws):
        assert oracle.decompress(kind, c, len(r)) == r, (kind, n, okw)
    # GPU stream -> GPU
    outs, actual, status, _ = gpu_decompress(codec, comps, [len(r) for r in raws])
    assert (status == 0).all(), (kind, okw, status)
    assert actual.tolist() == [len(r) for r in raws]
    assert outs == raws
    # CPU oracle stream -> GPU
    ocomps = [oracle.compress_typed(kind, r, **okw) for r in raws]
    outs, actual, status, _ = gpu_decompress(codec, ocomps, [len(r) for r in raws])
    assert (status == 0).all(), (kind, okw, status)
    assert outs == raws
    # size query
    from nvcomp_b200.batched import make_batch
    sizes = codec.get_decompress_size(make_batch(comps))
    torch.cuda.synchronize()
    assert sizes.cpu().tolist() == [len(r) for r in raws]
    return comps


@pytest.mark.parametrize("type_id", sorted(TS))
@pytest.mark.parametrize("layers", [(0, 0, 1), (1, 0, 1), (1, 1, 1), (2, 1, 1), (2, 2, 0), (0, 1, 1), (3, 2, 1), (1, 1, 0), (1, 0, 0)])
def test_cascaded(oracle, type_id, layers):
    from nvcomp_b200._lib import CascadedOpts
    from nvcomp_b200.batched import Codec
    r, d, bp = layers
    codec = Codec("Cascaded", opts=CascadedOpts(4096, type_id, r, d, bp))
    _roundtrip(codec, "cascaded", _raws(8), oracle, dict(type=type_id, num_RLEs=r, num_deltas=d, use_bp=bp))


@pytest.mark.parametrize("part", [512, 520, 1000, 1024, 8192, 16384])     # 520, 1000: element counts not divisible by 4
def test_cascaded_partition_sizes(oracle, part):
    from nvcomp_b200._lib import CascadedOpts
    from nvcomp_b200.batched import Codec
    for type_id in (1, 4, 6):
        codec = Codec("Cascaded", opts=CascadedOpts(part, type_id, 2, 1, 1))
        _roundtrip(codec, "cascaded", _raws(8), oracle,
                   dict(chunk_size=part, type=type_id, num_RLEs=2, num_deltas=1, use_bp=1))


def test_cascaded_compresses_sorted_int64(oracle):
    """cfg3: sorted int64 with {4096, LONGLONG, 1, 1, 1} must actually compress (delta + RLE + bit-pack)."""
    from gpu_util import gpu_compress
    from nvcomp_b200._lib import CascadedOpts
    from nvcomp_b200.batched import Codec
    codec = Codec("Cascaded", opts=CascadedOpts(4096, 6, 1, 1, 1))
    comps, _ = gpu_compress(codec, [INPUTS["sorted_i64"]])
    assert len(comps[0]) < 65536 / 8


@pytest.mark.parametrize("type_id", sorted(TS))
@pytest.mark.parametrize("algo", [0, 1])
def test_bitcomp(oracle, type_id, algo):
    from nvcomp_b200._lib import BitcompOpts
    from nvcomp_b200.batched import Codec
    codec = Codec("Bitcomp", opts=BitcompOpts(algo, type_id))
    _roundtrip(codec, "bitcomp", _raws(8), oracle, dict(algo=algo, type=type_id))


@pytest.mark.parametrize("kind", ["cascaded", "bitcomp"])
def test_chunk_length_not_a_multiple_of_the_element_size(oracle, kind):
    """Trailing bytes (length % sizeof(type)) are carried verbatim: every length round-trips, through the LLIF and
    against the oracle in both directions (ADVICE r1: they used to be dropped silently)."""
    from gpu_util import gpu_compress, gpu_decompress
    from nvcomp_b200._lib import BitcompOpts, CascadedOpts
    from nvcomp_b200.batched import Codec
    base = INPUTS["sorted_i64"]
    raws = [base[:n] for n in (1, 3, 7, 9, 1001, 4099, 40001, 65535, 65533)] + [b""]
    for type_id in (2, 4, 6):
        if kind == "cascaded":
            codec, okw = Codec("Cascaded", opts=CascadedOpts(4096, type_id, 1, 1, 1)), dict(type=type_id, num_RLEs=1, num_deltas=1, use_bp=1)
        else:
            codec, okw = Codec("Bitcomp", opts=BitcompOpts(0, type_id)), dict(algo=0, type=type_id)
        comps, _ = gpu_compress(codec, raws)
        for c, r in zip(comps, raws):
            assert oracle.decompress(kind, c, len(r)) == r, (kind, type_id, len(r))
        outs, actual, status, _ = gpu_decompress(codec, comps, [len(r) for r in raws])
        assert (status == 0).all() and actual.tolist() == [len(r) for r in raws] and outs == raws, (kind, type_id)
        ocomps = [oracle.compress_typed(kind, r, **okw) for r in raws]
        outs, actual, status, _ = gpu_decompress(codec, ocomps, [len(r) for r in raws])
        assert (status == 0).all() and outs == raws, (kind, type_id)


def test_ans(oracle):
    from nvcomp_b200.batched import Codec
    codec = Codec("ANS")
    raws = [INPUTS[n] for n in NAMES]
    comps = _roundtrip(codec, "ans", raws, oracle, {})
    i = NAMES.index("gen_data3")
    assert len(comps[i]) < 0.27 * len(raws[i])      # ~2 bits/byte


@pytest.mark.parametrize("kind", ["Cascaded", "Bitcomp", "ANS"])
def test_typed_malformed(kind, oracle):
    from gpu_util import gpu_compress, gpu_decompress
    from nvcomp_b200.batched import Codec
    codec = Codec(kind)
    raw = INPUTS["lowentropy"]
    comps, _ = gpu_compress(codec, [raw])
    good = comps[0]
    rng = np.random.default_rng(3)
    corrupt = bytearray(good)
    for pos in rng.integers(16, len(good), 64):
        corrupt[pos] ^= 0xFF
    bad = [good[: len(good) // 2], good[:24], bytes(64), b"", good, bytes(corrupt)]
    caps = [len(raw)] * 4 + [len(raw) - 8, len(raw)]
    outs, actual, status, _ = gpu_decompress(codec, bad + [good], caps + [len(raw)])
    for i in range(5):
        assert status[i] == 12 and actual[i] == 0, (kind, i, status[i], actual[i])
    # corrupted payload: the oracle's verdict, and its bytes when it decodes
    want = oracle.decompress(kind.lower(), bytes(corrupt), len(raw))
    if want is None:
        assert status[5] == 12 and actual[5] == 0, (kind, status[5], actual[5])
    else:
        assert status[5] == 0 and outs[5] == want, (kind, status[5], actual[5])
    assert status[6] == 0 and outs[6] == raw


@pytest.mark.parametrize("kind,dataset", [("Cascaded", "sorted_i64"), ("Bitcomp", "sorted_i64"),
                                          ("Bitcomp", "runlength_i32"), ("ANS", "lowentropy_bytes"),
                                          ("ANS", "snappy_synth"), ("ANS", "random_bytes"),
                                          ("Cascaded", "runlength_i32")])
def test_typed_batch_roundtrip_property(kind, dataset):
    """decompress(compress(x)) == x over 2000 x 64 KB chunks, compared on the device."""
    from nvcomp_b200 import datagen
    from nvcomp_b200._lib import BitcompOpts, CascadedOpts
    from nvcomp_b200.batched import Batch, Codec, empty_batch
    n = 2000
    data = datagen.DATASETS[dataset](n)
    t64 = "i64" in dataset
    opts = None
    if kind == "Cascaded":
        opts = CascadedOpts(4096, 6 if t64 else 4, 1, 1, 1)
    if kind == "Bitcomp":
        opts = BitcompOpts(0, 7 if t64 else 5)
    codec = Codec(kind, opts=opts)
    slab = torch.from_numpy(data.reshape(-1)).cuda()
    offsets = np.arange(n, dtype=np.int64) * 65536
    inp = Batch(slab, torch.from_numpy(offsets + slab.data_ptr()).cuda(),
                torch.full((n,), 65536, dtype=torch.int64, device="cuda"), offsets)
    comp = codec.compress(inp, max_chunk=65536)
    out = empty_batch(n, 65536, fill=0x5A)
    actual, status = codec.decompress(comp, out, max_chunk=65536)
    torch.cuda.synchronize()
    assert (status == 0).all().item()
    assert (actual == 65536).all().item()
    assert torch.equal(out.slab[: n * 65536], slab)


@pytest.mark.parametrize("kind", ["LZ4", "Snappy", "Cascaded", "Bitcomp", "ANS"])
def test_maximum_chunk_size(kind, oracle):
    """Chunks up to nvcomp<Fmt>CompressionMaxAllowedChunkSize (16 MB): round trip bit-exact, GPU stream decodes
    with the CPU oracle; one byte more is rejected with nvcompErrorChunkSizeTooLarge."""
    from gpu_util import gpu_compress, gpu_decompress
    from nvcomp_b200 import datagen
    from nvcomp_b200._lib import BitcompOpts, CascadedOpts
    from nvcomp_b200.batched import Codec, NvcompError
    opts = {"Cascaded": CascadedOpts(4096, 4, 1, 1, 1), "Bitcomp": BitcompOpts(0, 5)}.get(kind)
    codec = Codec(kind, opts=opts)
    big = np.concatenate([datagen.runlength_i32(64, seed=3).reshape(-1), datagen.tabular_f32(128, seed=4).reshape(-1),
                          datagen.lowentropy_bytes(64, seed=5).reshape(-1)])          # 16 MB
    assert big.size == 1 << 24
    raws = [big.tobytes(), big[: (1 << 20) + 8].tobytes()]
    comps, _ = gpu_compress(codec, raws)
    okind = {"LZ4": "lz4", "Snappy": "snappy", "Cascaded": "cascaded", "Bitcomp": "bitcomp", "ANS": "ans"}[kind]
    assert oracle.decompress(okind, comps[1], len(raws[1])) == raws[1]
    outs, actual, status, _ = gpu_decompress(codec, comps, [len(r) for r in raws])
    assert (status == 0).all() and outs == raws
    with pytest.raises(NvcompError):
        codec.compress_get_max_output_chunk_size((1 << 24) + 1)


@pytest.mark.parametrize("type_id", sorted(TS))
def test_bitcomp_delta_width_sweep(oracle, type_id):
    """Blocks whose zig-zag delta width runs from 0 to the full type width hit every decode path (<= 8 bits:
    32-bit funnel unpack; 9..16: 64-bit unpack with 32-bit prefix; > 16: 64-bit), with ragged last blocks and
    chunk pointers that are 8- but not 16-byte aligned (scalar instead of vector stores)."""
    from gpu_util import gpu_compress, gpu_decompress
    from nvcomp_b200._lib import BitcompOpts
    from nvcomp_b200.batched import Codec
    ts = TS[type_id]
    dt = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[ts]
    rng = np.random.default_rng(5 + type_id)
    raws = []
    for n in [1, 127, 128, 129, 1000, 8192]:
        parts = []
        for k in range(0, min(8 * ts, 62)):             # one 128-element block per delta magnitude 2^k
            step = rng.integers(-(1 << k), (1 << k) + 1, 128).astype(np.int64)
            parts.append(step)
        steps = np.concatenate(parts)[: max(n, 1)]
        if n > len(steps):
            steps = np.resize(steps, n)
        vals = (np.cumsum(steps) + int(rng.integers(0, 1 << 20))).astype(np.int64).astype(dt)
        raws.append(vals.tobytes())
    codec = Codec("Bitcomp", opts=BitcompOpts(0, type_id))
    for mis in (0, 8):
        comps, _ = gpu_compress(codec, raws, misalign=mis)
        for c, r in zip(comps, raws):
            assert oracle.decompress("bitcomp", c, len(r)) == r
        outs, actual, status, _ = gpu_decompress(codec, comps, [len(r) for r in raws], misalign=mis)
        assert (status == 0).all(), status
        assert outs == raws
        ocomps = [oracle.compress_typed("bitcomp", r, algo=0, type=type_id) for r in raws]
        outs, actual, status, _ = gpu_decompress(codec, ocomps, [len(r) for r in raws], misalign=mis)
        assert (status == 0).all() and outs == raws


def test_ans_entropy_and_segment_edges(oracle):
    """ANS streams from ~0.5 to ~7.5 bits/byte (few to many renormalisation words per round: the word ring
    is refilled one block every few groups up to several blocks per group) at sizes around the 32-symbol
    round and the 16384-symbol segment."""
    from gpu_util import gpu_compress, gpu_decompress
    from nvcomp_b200.batched import Codec
    rng = np.random.default_rng(77)
    raws = []
    for p in [0.9, 0.5, 0.2, 0.05, 0.02, 0.008]:                 # geometric symbol distributions
        for n in [1, 31, 32, 33, 1000, 16383, 16384, 16385, 50000, 65536]:
            raws.append(np.minimum(rng.geometric(p, n) - 1, 255).astype(np.uint8).tobytes())
    raws.append(bytes([7]) * 40000)                              # constant chunk
    codec = Codec("ANS")
    comps, _ = gpu_compress(codec, raws)
    for c, r in zip(comps, raws):
        assert oracle.decompress("ans", c, len(r)) == r
    outs, actual, status, _ = gpu_decompress(codec, comps, [len(r) for r in raws])
    assert (status == 0).all(), status
    assert outs == raws
    ocomps = [oracle.compress_typed("ans", r) for r in raws]
    outs, actual, status, _ = gpu_decompress(codec, ocomps, [len(r) for r in raws])
    assert (status == 0).all() and outs == raws
