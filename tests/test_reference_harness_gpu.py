"""-m gpu: the reference's OWN benchmarks and examples, compiled unchanged against include/ + libnvcomp.so
by oracle/build_reference_harness.sh (binaries in oracle/_ref/, built by build() where the nvCOMP tree exists), run as
the acceptance harness: every one of them self-verifies (status, sizes, bytes) and prints the reference's
4-line report (benchmarks/benchmark_template_chunked.cuh:553-617)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu
BIN = os.path.join(ROOT, "oracle", "_ref", "bin")


def _run(name, *args, timeout=600):
    exe = os.path.join(BIN, name)
    if not os.path.exists(exe):
        pytest.skip(f"{name} not built (oracle/build_reference_harness.sh needs the nvCOMP source tree)")
    r = subprocess.run([exe, *args], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, (name, r.stdout[-2000:], r.stderr[-2000:])
    return r.stdout


@pytest.fixture(scope="module")
def data_files(tmp_path_factory):
    from nvcomp_b200 import datagen
    d = tmp_path_factory.mktemp("refdata")
    files = {}
    for name, arr in (("i32", datagen.runlength_i32(64)), ("f32", datagen.tabular_f32(64)),
                      ("i64", datagen.sorted_i64(64)), ("bytes", datagen.lowentropy_bytes(64))):
        p = str(d / f"{name}.bin")
        arr.reshape(-1)[: 64 * 65536 - 1234 if name == "bytes" else None].tofile(p)
        files[name] = p
    return files


def _check_report(out):
    assert "compressed ratio" in out and "decompression throughput (GB/s)" in out, out


@pytest.mark.parametrize("fmt,key,extra", [
    ("lz4", "f32", []), ("lz4", "i32", ["-t", "int"]), ("snappy", "f32", []),
    ("cascaded", "i64", ["-t", "longlong", "-r", "1", "-d", "1", "-b", "1"]), ("cascaded", "i32", ["-t", "int"]),
    ("bitcomp", "i64", ["-t", "ulonglong"]), ("bitcomp", "i32", ["-t", "uint", "-a", "1"]), ("ans", "bytes", []),
])
def test_chunked_benchmarks(fmt, key, extra, data_files):
    """benchmark_<fmt>_chunked -f file: compress -> decompress -> byte compare inside the reference harness."""
    _check_report(_run(f"benchmark_{fmt}_chunked", "-f", data_files[key], *extra))


def test_snappy_synth():
    out = _run("benchmark_snappy_synth", "-b", "500", "-w", "2", "-i", "3")
    assert "decompression throughput (GB/s)" in out and "Mismatch" not in out and "failed" not in out


def test_lz4_synth_hlif():
    """benchmark_lz4_synth: LZ4Manager round trips of all-zero and all-random buffers, 64 KB ... 512 MB
    (reference benchmarks/benchmark_lz4_synth.cpp:64-72; BASELINE configs[0] names this path)."""
    out = _run("benchmark_lz4_synth", timeout=900)
    assert out.count("decompression throughput (GB/s)") == 28


@pytest.mark.parametrize("key", ["f32", "i32", "bytes"])
def test_lz4_cpu_interop_examples(key, data_files):
    """The reference's known-answer tests of the LZ4 wire format, compiled unchanged (tests/shim/lz4.h only declares
    liblz4's prototypes): liblz4-HC(12) streams decode on the GPU (examples/lz4_cpu_compression.cu:61-66,121-140) and
    GPU streams decode with LZ4_decompress_safe (examples/lz4_cpu_decompression.cu:143-157)."""
    out = _run("lz4_cpu_compression", "-f", data_files[key])
    assert "decompression validated :)" in out
    out = _run("lz4_cpu_decompression", "-f", data_files[key])
    assert "CPU decompression validated :)" in out


def test_quickstarts():
    _run("low_level_quickstart_example")
    _run("high_level_quickstart_example")


@pytest.mark.parametrize("fmt,key,extra", [("lz4", "f32", []), ("snappy", "i32", []), ("ans", "bytes", []),
                                           ("bitcomp", "i32", ["-t", "int"]),
                                           ("cascaded", "i32", ["-t", "int"])])
def test_hlif_benchmark(fmt, key, extra, data_files):
    out = _run("benchmark_hlif", fmt, "-f", data_files[key], *extra)
    assert "decompression throughput (GB/s)" in out


def test_unsupported_formats_report_not_supported(data_files):
    exe = os.path.join(BIN, "benchmark_zstd_chunked")
    if not os.path.exists(exe):
        pytest.skip("not built")
    r = subprocess.run([exe, "-f", data_files["bytes"]], capture_output=True, text=True, timeout=120)
    assert r.returncode != 0     # out-of-scope format: the harness' status assert fires, nothing crashes


def test_cmake_built_reference_binary_runs():
    """A binary produced by the reference's OWN CMake build against cmake/nvcomp-config.cmake
    (oracle/_ref/cmake, built by oracle/build_reference_harness.sh for sm_90a)."""
    exe = os.path.join(ROOT, "oracle", "_ref", "cmake", "bin", "low_level_quickstart_example")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/cmake not present")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    exe = os.path.join(ROOT, "oracle", "_ref", "cmake", "bin", "benchmark_snappy_synth")
    r = subprocess.run([exe, "-b", "200", "-w", "1", "-i", "2"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "decompression throughput (GB/s)" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
