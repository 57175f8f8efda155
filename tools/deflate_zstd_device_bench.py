"""Time the warp-level Deflate, Gzip and Zstd device APIs (include/nvcomp/device/deflate.cuh, gzip.cuh, zstd.cuh)
next to the batched C API on the same chunks, and measure what decoding inside a consuming kernel costs or saves.

    python tools/deflate_zstd_device_bench.py [--chunks 10000] [--steps 20] [--warmup 5] [--zstd-levels 1,3,19]

The workloads are those of tools/inflate_bench.py, tools/zstd_bench.py and tools/deflate_compress_bench.py, so the
figures line up with theirs: --chunks x 64 KB of datagen.tabular_f32 (the flagship workload's data) and runlength_i32,
plus lowentropy_bytes for Zstd;
  Deflate, Gzip   compressed by host zlib at level 6;
  Zstd            compressed by host libzstd at each of --zstd-levels (checksum off) and by pyarrow's default codec;
  compression     algos 0, 1 and 2 on the raw chunks.
The test kernels of build/tests/libdeflate_zstd_device.so run 4 warps per CTA (3 for algo-1 compression), each with
its own shared-memory region, and pull chunks from a global ticket (one wave of resident CTAs).  Timed on cuda:0:
  batched_decompress      nvcompBatched<Format>DecompressAsync
  warp_decompress         decompress_warp, one warp per chunk
  batched_decompress_sum  the batched decompression, then a warp-per-chunk kernel that sums each decoded chunk's
                          32-bit words
  fused_decompress_sum    decompress_warp, and the same warp sums its chunk right after
  batched_compress / warp_compress   nvcompBatchedDeflateCompressAsync against compress_warp, per algo
Before any timing of a workload a parity gate checks that compress_warp's streams equal the batched encoder's byte for
byte, that both decoders return every chunk's status, size and bytes, and that both sums equal numpy's.  Each figure
is K back-to-back calls between two CUDA events, after warm-up; GB/s = uncompressed bytes / time.  The card name and
power limit are read in the same run.  Needs a CUDA GPU (and libzstd.so.1 and pyarrow for the Zstd workloads, which
are skipped with a note without them): there is no fallback.  Prints one JSON line per figure and writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CHUNK = 65536
KIND = {"Deflate": "deflate", "Gzip": "gzip", "Zstd": "zstd"}


def smi(fields: str) -> dict:
    try:
        q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(fields.split(","), [x.strip() for x in q.split(",")]))
    except Exception as e:  # noqa: BLE001 -- the figure is reported as missing, the timing still stands
        return {"unavailable": type(e).__name__}


def time_ms(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def emit(args, **kw) -> None:
    print(json.dumps({**kw, "steps": args.steps, "warmup": args.warmup}), flush=True)


def bench_decode(args, dev, fmt, producer, dataset, arr, streams) -> None:
    from nvcomp_b200.batched import Codec, empty_batch, make_batch
    n = arr.shape[0]
    kind = KIND[fmt]
    codec = Codec(fmt)
    stream = torch.cuda.current_stream().cuda_stream
    raw_dev = torch.from_numpy(arr.reshape(-1)).cuda()
    want_sums = arr.view(np.uint32).astype(np.uint64).sum(axis=1, dtype=np.uint64)
    comp = make_batch(streams)
    outs = {k: empty_batch(n, CHUNK, fill=0) for k in ("batched", "warp", "fused")}
    dtb = codec.decompress_get_temp_size(n, CHUNK)
    dtemp = torch.empty(max(dtb, 1), dtype=torch.uint8, device="cuda")
    actual = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in ("batched", "warp")}
    status = {k: torch.full((n,), -1, dtype=torch.int32, device="cuda") for k in outs}
    sums = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in ("unfused", "fused")}
    ticket = torch.zeros(1, dtype=torch.int64, device="cuda")
    sum_ticket = torch.zeros(1, dtype=torch.int64, device="cuda")

    def batched():
        o = outs["batched"]
        codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), o.sizes.data_ptr(),
                               actual["batched"].data_ptr(), n, dtemp.data_ptr(), dtb, o.ptrs.data_ptr(),
                               status["batched"].data_ptr(), stream)

    def warp():
        ticket.zero_()
        dev.decompress_async(kind, comp, outs["warp"], actual["warp"], status["warp"], ticket)

    def batched_sum():
        batched()
        sum_ticket.zero_()
        dev.sum_async(outs["batched"], actual["batched"], sums["unfused"], sum_ticket)

    def fused():
        ticket.zero_()
        dev.decompress_sum_async(kind, comp, outs["fused"], sums["fused"], status["fused"], ticket)

    for fn in (batched_sum, warp, fused):
        fn()
    torch.cuda.synchronize()
    for k in outs:
        assert bool((status[k] == 0).all()), (fmt, producer, dataset, k, "status")
        assert torch.equal(outs[k].slab[: n * CHUNK], raw_dev), (fmt, producer, dataset, k, "bytes")
    for k in actual:
        assert bool((actual[k] == CHUNK).all()), (fmt, producer, dataset, k, "actual")
    for k in sums:
        assert (sums[k].cpu().numpy().view(np.uint64) == want_sums).all(), (fmt, producer, dataset, k, "sums")
    uncomp = n * CHUNK
    ratio = round(uncomp / sum(len(s) for s in streams), 3)
    for name, fn in (("batched_decompress", batched), ("warp_decompress", warp),
                     ("batched_decompress_sum", batched_sum), ("fused_decompress_sum", fused)):
        ms = time_ms(fn, args.steps, args.warmup)
        emit(args, format=fmt, producer=producer, dataset=dataset, call=name, chunks=n, ratio=ratio,
             ms=round(ms, 3), gbs=round(uncomp / ms / 1e6, 2))
    del outs, comp, raw_dev
    torch.cuda.empty_cache()


def bench_compress(args, dev, dataset, arr) -> None:
    from nvcomp_b200._lib import DeflateOpts
    from nvcomp_b200.batched import Codec, empty_batch, make_batch
    n = arr.shape[0]
    stream = torch.cuda.current_stream().cuda_stream
    inp = make_batch([arr[i] for i in range(n)])
    uncomp = n * CHUNK
    for algo in (0, 1, 2):
        codec = Codec("Deflate", opts=DeflateOpts(algo))
        max_out = codec.compress_get_max_output_chunk_size(CHUNK)
        assert dev.max_compressed_bytes(CHUNK) == max_out
        bout, wout = empty_batch(n, max_out, fill=0), empty_batch(n, max_out, fill=0)
        ctb = codec.compress_get_temp_size(n, CHUNK)
        ctemp = torch.empty(max(ctb, 1), dtype=torch.uint8, device="cuda")
        status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        ticket = torch.zeros(1, dtype=torch.int64, device="cuda")

        def batched():
            codec.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), CHUNK, n, ctemp.data_ptr(), ctb,
                                 bout.ptrs.data_ptr(), bout.sizes.data_ptr(), stream)

        def warp():
            ticket.zero_()
            dev.compress_async(inp, wout, status, algo, ticket)

        batched()
        warp()
        torch.cuda.synchronize()
        assert bool((status == 0).all()), ("compress_warp status", algo)
        sizes = bout.sizes.cpu().numpy()
        assert (wout.sizes.cpu().numpy() == sizes).all(), ("compressed sizes", algo)
        assert wout.to_host(sizes) == bout.to_host(sizes), ("compress_warp stream != batched stream", algo)
        ratio = round(uncomp / int(sizes.sum()), 3)
        for name, fn in (("batched_compress", batched), ("warp_compress", warp)):
            ms = time_ms(fn, args.steps, args.warmup)
            emit(args, format="Deflate", algo=algo, dataset=dataset, call=name, chunks=n, ratio=ratio,
                 ms=round(ms, 3), gbs=round(uncomp / ms / 1e6, 2))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--zstd-levels", default="1,3,19")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deflate_zstd_device_bench.py needs a CUDA GPU")
    from deflate_zstd_device import DeflateZstdDevice
    from nvcomp_b200 import datagen

    torch.cuda.set_device(0)
    card = {"name": torch.cuda.get_device_name(0), **smi("power.limit,clocks.max.sm")}
    print(json.dumps({"card": card}), flush=True)
    dev = DeflateZstdDevice()
    n = args.chunks
    pool = ThreadPoolExecutor(os.cpu_count() or 1)
    data = {name: np.ascontiguousarray(getattr(datagen, name)(n)).view(np.uint8).reshape(n, CHUNK)
            for name in ("tabular_f32", "runlength_i32", "lowentropy_bytes")}

    def zlib_all(arr, wbits):
        def one(c):
            z = zlib.compressobj(6, zlib.DEFLATED, wbits)
            return z.compress(c) + z.flush()
        return list(pool.map(one, [arr[i].tobytes() for i in range(n)]))

    for dataset in ("tabular_f32", "runlength_i32"):
        arr = data[dataset]
        for fmt, wbits in (("Deflate", -15), ("Gzip", 31)):
            bench_decode(args, dev, fmt, "zlib-6", dataset, arr, zlib_all(arr, wbits))
        bench_compress(args, dev, dataset, arr)

    import zstd_writer
    zs = zstd_writer.libzstd_or_none()
    try:
        import pyarrow as pa
    except ImportError:
        pa = None
    if zs is None:
        print(json.dumps({"note": "libzstd.so.1 not available: Zstd workloads skipped"}), flush=True)
        return
    producers = [(f"libzstd-{lv}", lambda c, lv=lv: zs.compress(c, lv)) for lv in map(int, args.zstd_levels.split(","))]
    if pa is not None:
        producers.append(("pyarrow-default", lambda c: pa.Codec("zstd").compress(c, asbytes=True)))
    else:
        print(json.dumps({"note": "pyarrow not available: its Zstd workload skipped"}), flush=True)
    for dataset, arr in data.items():
        chunks = [arr[i].tobytes() for i in range(n)]
        for producer, fn in producers:
            bench_decode(args, dev, "Zstd", producer, dataset, arr, list(pool.map(fn, chunks)))


if __name__ == "__main__":
    main()
