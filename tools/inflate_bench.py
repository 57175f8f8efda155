"""Time batched Deflate and Gzip decompression (nvcompBatched{Deflate,Gzip}DecompressAsync) on one GPU, next to the
host's zlib on all cores.

    python tools/inflate_bench.py [--chunks 10000] [--steps 20] [--warmup 5] [--level 6]

Each dataset (datagen.tabular_f32, the flagship workload's data, and the typed runlength_i32) is cut into 64 KB
chunks, compressed by zlib on the host as raw Deflate and as Gzip, and decoded on cuda:0.  Before any timing a
parity gate checks every status, size and byte.  The GPU figure is K back-to-back calls between two CUDA events,
after warm-up; the definitions are bench.py's: GB/s = uncompressed bytes / time, roofline share = (compressed +
uncompressed + 44 B per chunk) / time / 3.35 TB/s.  The size query (GetDecompressSizeAsync) runs the same decoder
with its stores disabled, so its time is the symbol decode alone.  The host figure is zlib.decompress over a thread
pool of all cores (zlib releases the GIL).  Card name and power limit are read in the same run.  Needs a CUDA GPU:
there is no fallback.  Prints one JSON line per measurement and writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0     # H100 SXM data sheet
CHUNK = 65536
WBITS = {"Deflate": -15, "Gzip": 31}


def card() -> dict:
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, sm = [x.strip() for x in q.split(",")]
        info.update(smi_name=name, power_limit=power, sm_max_clock=sm)
    except Exception as e:  # noqa: BLE001 -- the card name from torch still identifies the part
        info["power_limit"] = f"unavailable ({type(e).__name__})"
    return info


def compress_all(chunks, wbits, level, pool):
    def one(c):
        z = zlib.compressobj(level, zlib.DEFLATED, wbits)
        return z.compress(c) + z.flush()
    return list(pool.map(one, chunks))


def host_zlib(streams, wbits, pool, reps=3) -> float:
    """seconds per pass, best of reps"""
    best = float("inf")
    for _ in range(reps):
        t = time.perf_counter()
        for _ in pool.map(lambda s: zlib.decompress(s, wbits), streams, chunksize=64):
            pass
        best = min(best, time.perf_counter() - t)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--level", type=int, default=6)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("inflate_bench: no CUDA device (this measures the GPU decoder; there is no CPU fallback)")
    torch.cuda.set_device(0)
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import Codec, empty_batch, make_batch

    print(json.dumps({"card": card(), "host_threads": os.cpu_count(), "zlib": zlib.ZLIB_RUNTIME_VERSION}), flush=True)
    pool = ThreadPoolExecutor(os.cpu_count())
    n = args.chunks
    for dataset in ("tabular_f32", "runlength_i32"):
        arr = getattr(datagen, dataset)(n)
        chunks = [arr[i].tobytes() for i in range(n)]
        raw_dev = torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(n, CHUNK)).cuda()
        for fmt in ("Deflate", "Gzip"):
            streams = compress_all(chunks, WBITS[fmt], args.level, pool)
            comp_bytes = sum(len(s) for s in streams)
            codec = Codec(fmt)
            comp = make_batch(streams)
            out = empty_batch(n, CHUNK, fill=0)
            tb = codec.decompress_get_temp_size(n, CHUNK)
            temp = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
            actual = torch.zeros(n, dtype=torch.int64, device="cuda")
            status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            stream = torch.cuda.current_stream().cuda_stream

            def call():
                codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(),
                                       actual.data_ptr(), n, temp.data_ptr(), tb, out.ptrs.data_ptr(),
                                       status.data_ptr(), stream)

            # parity gate: every chunk decodes to its input
            call()
            torch.cuda.synchronize()
            assert bool((status == 0).all()), (fmt, dataset, "status")
            assert bool((actual == CHUNK).all()), (fmt, dataset, "actual")
            got = out.slab[: n * CHUNK].view(n, CHUNK)
            assert torch.equal(got, raw_dev), (fmt, dataset, "bytes")
            for _ in range(args.warmup):
                call()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.steps):
                call()
            t1.record()
            torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / args.steps
            sizes = torch.zeros(n, dtype=torch.int64, device="cuda")

            def size_call():
                codec.get_decompress_size_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), sizes.data_ptr(), n,
                                                stream)

            size_call()
            torch.cuda.synchronize()
            assert bool((sizes == CHUNK).all()), (fmt, dataset, "size query")
            for _ in range(args.warmup):
                size_call()
            t0.record()
            for _ in range(args.steps):
                size_call()
            t1.record()
            torch.cuda.synchronize()
            size_ms = t0.elapsed_time(t1) / args.steps
            uncomp = n * CHUNK
            host_s = host_zlib(streams, WBITS[fmt], pool)
            print(json.dumps({
                "format": fmt, "dataset": dataset, "chunks": n, "level": args.level,
                "ratio": round(uncomp / comp_bytes, 3), "gpu_ms": round(ms, 3),
                "gpu_gbs": round(uncomp / ms / 1e6, 1),
                "roofline_frac": round((comp_bytes + uncomp + 44 * n) / ms / 1e6 / HBM_GBS, 4),
                "size_query_ms": round(size_ms, 3),
                "host_zlib_gbs": round(uncomp / host_s / 1e9, 2), "host_threads": os.cpu_count(),
                "steps": args.steps, "warmup": args.warmup}), flush=True)
            del comp, out, temp
    pool.shutdown()


if __name__ == "__main__":
    main()
