"""Time batched Deflate compression (nvcompBatchedDeflateCompressAsync) on one GPU, next to the host's zlib on all
cores.

    python tools/deflate_compress_bench.py [--chunks 10000] [--steps 10] [--warmup 3]

Each dataset (datagen.tabular_f32, the flagship workload's data, and the typed runlength_i32) is cut into 64 KB
chunks and compressed on cuda:0 with algos 0, 1 and 2.  Before any timing a parity gate inflates every stream with
host zlib and compares it with the input.  The GPU figure is K back-to-back calls between two CUDA events, after
warm-up; GB/s = uncompressed bytes / time, ratio = uncompressed / compressed bytes.  The host figures are zlib levels 1
and 6 (raw Deflate) over a thread pool of all cores (zlib releases the GIL), best of three passes.  Card name and power
limit are read in the same run.  Needs a CUDA GPU: there is no fallback.  Prints one JSON line per measurement and
writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from inflate_bench import card  # noqa: E402

CHUNK = 65536


def host_zlib(chunks, level, pool, reps=3):
    """(seconds per pass, best of reps; compressed bytes)"""
    def one(c):
        z = zlib.compressobj(level, zlib.DEFLATED, -15)
        return len(z.compress(c) + z.flush())
    best, size = float("inf"), 0
    for _ in range(reps):
        t = time.perf_counter()
        size = sum(pool.map(one, chunks, chunksize=64))
        best = min(best, time.perf_counter() - t)
    return best, size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("deflate_compress_bench: no CUDA device (this measures the GPU encoder; there is no CPU fallback)")
    torch.cuda.set_device(0)
    from nvcomp_b200 import datagen
    from nvcomp_b200._lib import DeflateOpts
    from nvcomp_b200.batched import Codec, empty_batch, make_batch

    print(json.dumps({"card": card(), "host_threads": os.cpu_count(), "zlib": zlib.ZLIB_RUNTIME_VERSION}), flush=True)
    pool = ThreadPoolExecutor(os.cpu_count())
    n = args.chunks
    for dataset in ("tabular_f32", "runlength_i32"):
        arr = getattr(datagen, dataset)(n)
        chunks = [arr[i].tobytes() for i in range(n)]
        uncomp = n * CHUNK
        inp = make_batch(chunks)
        stream = torch.cuda.current_stream().cuda_stream
        for algo in (0, 1, 2):
            codec = Codec("Deflate", opts=DeflateOpts(algo))
            max_out = codec.compress_get_max_output_chunk_size(CHUNK)
            tb = codec.compress_get_temp_size(n, CHUNK)
            temp = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
            out = empty_batch(n, max_out)

            def call():
                codec.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), CHUNK, n, temp.data_ptr(), tb,
                                     out.ptrs.data_ptr(), out.sizes.data_ptr(), stream)

            # parity gate: every stream inflates to its input
            call()
            torch.cuda.synchronize()
            streams = out.to_host(out.sizes.cpu().numpy())
            back = list(pool.map(lambda s: zlib.decompress(s, -15), streams, chunksize=64))
            assert back == chunks, (dataset, algo, "parity")
            comp_bytes = sum(len(s) for s in streams)
            for _ in range(args.warmup):
                call()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.steps):
                call()
            t1.record()
            torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / args.steps
            print(json.dumps({
                "dataset": dataset, "algo": algo, "chunks": n, "ratio": round(uncomp / comp_bytes, 3),
                "gpu_ms": round(ms, 3), "gpu_gbs": round(uncomp / ms / 1e6, 2),
                "steps": args.steps, "warmup": args.warmup}), flush=True)
            del out, temp
        for level in (1, 6):
            s, size = host_zlib(chunks, level, pool)
            print(json.dumps({"dataset": dataset, "host_zlib_level": level, "ratio": round(uncomp / size, 3),
                              "host_gbs": round(uncomp / s / 1e9, 3), "host_threads": os.cpu_count()}), flush=True)
    pool.shutdown()


if __name__ == "__main__":
    main()
