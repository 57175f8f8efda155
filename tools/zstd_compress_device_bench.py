"""zstd::compress_warp (include/nvcomp/device/zstd.cuh) on 10 000 x 64 KB chunks of tabular float32, run-length int32
and low-entropy bytes, next to deflate::compress_warp algo 0 on the same chunks (tests/cpp/deflate_zstd_device_kernels.cu)
and host libzstd at levels 1 and 3 (one chunk per ZSTD_compress2 call, all host cores).  Prints one table with the
card's name and power limit read in the same run.  Usage: python tools/zstd_compress_device_bench.py [--chunks N]
[--steps K] [--warmup W]"""
import argparse
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from nvcomp_b200 import datagen  # noqa: E402
from nvcomp_b200.batched import empty_batch, make_batch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def host_libzstd(zs, chunks, level):
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        t = time.perf_counter()
        sizes = list(ex.map(lambda c: len(zs.compress(c, level=level)), chunks))
        return time.perf_counter() - t, sum(sizes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: compress_warp timings need an H100")
    from deflate_zstd_device import DeflateZstdDevice
    from test_zstd_compress_device_gpu import Lib
    import zstd_writer as W
    zl, dz, zs = Lib(), DeflateZstdDevice(), W.LibZstd()
    print(f"card: {card()}")
    print(f"{'data':<18} {'zstd ratio':>10} {'zstd GB/s':>10} {'deflate0 ratio':>14} {'deflate0 GB/s':>13} "
          f"{'libzstd-1 ratio':>15} {'GB/s':>6} {'libzstd-3 ratio':>15} {'GB/s':>6}")
    data = {"tabular_f32": datagen.tabular_f32, "runlength_i32": datagen.runlength_i32,
            "lowentropy_bytes": datagen.lowentropy_bytes}
    for name, gen in data.items():
        raw = gen(args.chunks).tobytes()
        chunks = [raw[i:i + 65536] for i in range(0, len(raw), 65536)]
        inp = make_batch(chunks)
        zout = empty_batch(len(chunks), zl.bound(65536))
        dout = empty_batch(len(chunks), dz.max_compressed_bytes(65536))
        st = torch.zeros(len(chunks), dtype=torch.int32, device="cuda")
        tz = timed(lambda: zl.compress(inp, zout, st), args.steps, args.warmup)
        assert (st == 0).all()
        zbytes = int(zout.sizes.sum())
        td = timed(lambda: dz.compress_async(inp, dout, st, 0), args.steps, args.warmup)
        assert (st == 0).all()
        dbytes = int(dout.sizes.sum())
        t1, b1 = host_libzstd(zs, chunks, 1)
        t3, b3 = host_libzstd(zs, chunks, 3)
        n = len(raw)
        print(f"{name:<18} {n / zbytes:>10.2f} {n / tz / 1e6:>10.2f} {n / dbytes:>14.2f} {n / td / 1e6:>13.2f} "
              f"{n / b1:>15.2f} {n / t1 / 1e9:>6.2f} {n / b3:>15.2f} {n / t3 / 1e9:>6.2f}")
    print(f"{args.steps} timed calls after {args.warmup} warm-up calls; host libzstd on {os.cpu_count()} threads")


if __name__ == "__main__":
    main()
