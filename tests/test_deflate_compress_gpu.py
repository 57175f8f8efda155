"""-m gpu: batched Deflate compression through the C ABI (nvcomp_b200.batched over libnvcomp.so).  The GPU's streams
must equal the host warp emulator's byte for byte (tests/test_deflate_encode_emu.py pins those to the stream rules),
inflate under zlib and under this library's decoder, and stay inside their guarded output buffers."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch

import test_deflate_encode_emu as E
from conftest import ROOT
from gpu_util import gpu_compress, gpu_decompress
from nvcomp_b200 import datagen
from nvcomp_b200._lib import DeflateOpts, Status
from nvcomp_b200.batched import Codec, NvcompError, make_batch

pytestmark = pytest.mark.gpu
ALGOS = (0, 1, 2)
BIN = os.path.join(ROOT, "oracle", "_ref", "bin")


def codec(algo):
    return Codec("Deflate", opts=DeflateOpts(algo))


def inflate(stream: bytes) -> bytes:
    z = zlib.decompressobj(-15)
    out = z.decompress(stream)
    assert z.eof and not z.unused_data
    return out


@pytest.fixture(scope="module")
def emu():
    return E.Emu()


@pytest.mark.parametrize("algo", ALGOS)
def test_gpu_bytes_equal_emulator(emu, algo):
    """Every input of the CPU test, in one batch: the GPU stream is the emulator's, and a second run agrees."""
    names = sorted(E.INPUTS)
    chunks = [E.INPUTS[k] for k in names]
    first, _ = gpu_compress(codec(algo), chunks)
    second, _ = gpu_compress(codec(algo), chunks)
    assert first == second
    for name, data, got in zip(names, chunks, first):
        assert got == emu.compress(algo, data), (name, algo)


def _datasets(n):
    return {
        "tabular_f32": datagen.tabular_f32(n, seed=41),
        "runlength_i32": datagen.runlength_i32(n, seed=42),
        "sorted_i64": datagen.sorted_i64(n, seed=43),
        "lowentropy_bytes": datagen.lowentropy_bytes(n, seed=44),
        "snappy_synth": datagen.snappy_synth(n, 3, seed=45),
        "lz4_mixed": datagen.lz4_mixed(n, seed=46),
        "random_bytes": datagen.random_bytes(n, seed=47),
    }


def _roundtrip(algo, chunks, misalign=0):
    c = codec(algo)
    streams, _ = gpu_compress(c, chunks, misalign=misalign)
    for i, (s, data) in enumerate(zip(streams, chunks)):
        assert inflate(s) == data, (algo, i)
    outs, actual, status, _ = gpu_decompress(c, streams, [len(x) for x in chunks], misalign=misalign)
    assert (status == 0).all() and outs == chunks, algo
    return streams


@pytest.mark.parametrize("algo", ALGOS)
def test_roundtrip_datasets(algo):
    """2000-chunk batches of every dataset: zlib and the GPU decoder both return the input."""
    for name, arr in _datasets(2000).items():
        _roundtrip(algo, [arr[i].tobytes() for i in range(arr.shape[0])])


@pytest.mark.parametrize("misalign", [0, 1, 7])
@pytest.mark.parametrize("algo", ALGOS)
def test_roundtrip_ragged_misaligned(algo, misalign):
    """Ragged sizes from 0 to 65 536 bytes, inputs and outputs at 16-byte aligned addresses + misalign."""
    rng = np.random.default_rng(100 + algo)
    sizes = [0, 1, 2, 3, 4, 5, 65535, 65536] + list(rng.integers(0, 65537, 600))
    src = datagen.tabular_f32(8, seed=48).tobytes() + datagen.runlength_i32(8, seed=49).tobytes()
    starts = rng.integers(0, len(src) - 65536, len(sizes))
    chunks = [src[s:s + n] for s, n in zip(starts, sizes)]
    _roundtrip(algo, chunks, misalign)


def test_arguments():
    lib = codec(0).lib
    vp = C.c_void_p
    n, m = 64, 65536
    chunks = [datagen.tabular_f32(1, seed=50)[0].tobytes()[: 1000 * i] for i in range(n)]
    # temp == nullptr: the static schedule
    c = codec(0)
    inp = make_batch(chunks)
    max_out = c.compress_get_max_output_chunk_size(m)
    assert max_out == m + 5 * (m // 65535 + 1)
    out = make_batch([b"\0" * max_out] * n)
    c.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), m, n, None, 0, out.ptrs.data_ptr(),
                     out.sizes.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert [inflate(s) for s in out.to_host()] == chunks
    # a batch of 0 is a no-op, even with null pointers
    c.compress_async(None, None, m, 0, None, 0, None, None, torch.cuda.current_stream().cuda_stream)
    # algo outside 0..2: InvalidValue from all three entry points
    size = C.c_size_t(0)
    for bad in (3, -1):
        o = DeflateOpts(bad)
        assert lib.nvcompBatchedDeflateCompressGetTempSize(n, m, o, C.byref(size)) == Status.ErrorInvalidValue
        assert lib.nvcompBatchedDeflateCompressGetMaxOutputChunkSize(m, o, C.byref(size)) == Status.ErrorInvalidValue
        assert lib.nvcompBatchedDeflateCompressAsync(vp(inp.ptrs.data_ptr()), vp(inp.sizes.data_ptr()), m, n, None,
                                                     0, vp(out.ptrs.data_ptr()), vp(out.sizes.data_ptr()), o,
                                                     None) == Status.ErrorInvalidValue
    # chunks over 64 KB: ChunkSizeTooLarge
    o = DeflateOpts(0)
    assert lib.nvcompBatchedDeflateCompressGetTempSize(n, m + 1, o, C.byref(size)) == Status.ErrorChunkSizeTooLarge
    assert lib.nvcompBatchedDeflateCompressGetMaxOutputChunkSize(m + 1, o, C.byref(size)) == \
        Status.ErrorChunkSizeTooLarge
    assert lib.nvcompBatchedDeflateCompressAsync(vp(inp.ptrs.data_ptr()), vp(inp.sizes.data_ptr()), m + 1, n, None, 0,
                                                 vp(out.ptrs.data_ptr()), vp(out.sizes.data_ptr()), o,
                                                 None) == Status.ErrorChunkSizeTooLarge
    with pytest.raises(NvcompError):
        c.compress_get_max_output_chunk_size(m + 1)
    # the Ex temp sizes agree with the plain calls
    a, b = C.c_size_t(0), C.c_size_t(0)
    for algo in ALGOS:
        assert lib.nvcompBatchedDeflateCompressGetTempSize(n, m, DeflateOpts(algo), C.byref(a)) == 0
        assert lib.nvcompBatchedDeflateCompressGetTempSizeEx(n, m, DeflateOpts(algo), C.byref(b), n * m) == 0
        assert a.value == b.value
    assert lib.nvcompBatchedDeflateDecompressGetTempSize(n, m, C.byref(a)) == 0
    assert lib.nvcompBatchedDeflateDecompressGetTempSizeEx(n, m, C.byref(b), n * m) == 0
    assert a.value == b.value


def test_deflate_manager_cpp():
    exe = os.path.join(ROOT, "build", "tests", "deflate_hlif_test")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", ROOT, "build/tests/deflate_hlif_test"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-2000:])
    assert "deflate_hlif_test ok" in r.stdout


def _run_ref(name, *args, timeout=600):
    exe = os.path.join(BIN, name)
    if not os.path.exists(exe):
        pytest.skip(f"{name} not built (oracle/build_reference_harness.sh needs the nvCOMP source tree)")
    r = subprocess.run([exe, *args], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, (name, r.stdout[-2000:], r.stderr[-2000:])
    return r.stdout


@pytest.fixture(scope="module")
def data_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("deflate_refdata")
    files = {}
    for name, arr in (("f32", datagen.tabular_f32(64)), ("i32", datagen.runlength_i32(64)),
                      ("bytes", datagen.lowentropy_bytes(64))):
        p = str(d / f"{name}.bin")
        arr.reshape(-1)[: 64 * 65536 - 1234 if name == "bytes" else None].tofile(p)
        files[name] = p
    return files


@pytest.mark.parametrize("algo", ["0", "1", "2"])
@pytest.mark.parametrize("key", ["f32", "i32", "bytes"])
def test_reference_deflate_benchmark(algo, key, data_files):
    """benchmark_deflate_chunked -a algo -f file: compress -> decompress -> byte compare inside the reference harness."""
    out = _run_ref("benchmark_deflate_chunked", "-a", algo, "-f", data_files[key])
    assert "compressed ratio" in out and "decompression throughput (GB/s)" in out and "Mismatch" not in out, out


def test_reference_hlif_benchmark(data_files):
    out = _run_ref("benchmark_hlif", "deflate", "-f", data_files["f32"])
    assert "decompression throughput (GB/s)" in out
