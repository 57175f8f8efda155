"""Time the warp-level LZ4 / Snappy device APIs (include/nvcomp/device/lz4.cuh, snappy.cuh) next to the batched C API
on the same chunks, and measure what decoding inside a consuming kernel costs or saves.

    python tools/lz_device_bench.py --codec lz4|snappy [--chunks 10000] [--steps 20] [--warmup 5]

The workloads are bench.py's: LZ4 on --chunks x 64 KB of run-length int32 + tabular float32 (datagen.lz4_mixed),
Snappy on --chunks x 64 KB of tabular float32 (datagen.tabular_f32), default options.  The test kernels of
build/tests/liblz_device.so run 4 warps per CTA, each with its own shared-memory region, and the decode, sum and
compress kernels pull chunks from a global ticket (one wave of resident CTAs).  Timed on cuda:0:
  batched_decompress      nvcomp<Codec>DecompressAsync (light and dense kernels side by side, cost-ordered lists)
  warp_decompress         decompress_warp, one warp per chunk
  batched_decompress_sum  the batched decompression, then a warp-per-chunk kernel that sums each decoded chunk's
                          32-bit words
  fused_decompress_sum    decompress_warp, and the same warp sums its chunk right after
  batched_compress / warp_compress   nvcomp<Codec>CompressAsync against compress_warp
Before any timing a parity gate checks that compress_warp's streams equal the batched encoder's byte for byte, that
both decoders return every chunk's status, size and bytes, and that both sums equal numpy's.  Each figure is K
back-to-back calls between two CUDA events, after warm-up; GB/s = uncompressed bytes / time.  The card name and power
limit are read in the same run.  Needs a CUDA GPU: there is no fallback.  Prints one JSON line per figure and writes
nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CHUNK = 65536
FMT = {"lz4": "LZ4", "snappy": "Snappy"}
DATASET = {"lz4": "lz4_mixed", "snappy": "tabular_f32"}


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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--codec", choices=sorted(FMT), default="lz4")
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lz_device_bench.py needs a CUDA GPU")
    from lz_device import LzDevice
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import Codec, empty_batch, make_batch

    torch.cuda.set_device(0)
    card = {"name": torch.cuda.get_device_name(0), **smi("power.limit,clocks.max.sm")}
    print(json.dumps({"card": card}), flush=True)
    kind, n = args.codec, args.chunks
    arr = np.ascontiguousarray(datagen.DATASETS[DATASET[kind]](n)).view(np.uint8).reshape(n, CHUNK)
    raw_dev = torch.from_numpy(arr.reshape(-1)).cuda()
    want_sums = arr.view(np.uint32).astype(np.uint64).sum(axis=1, dtype=np.uint64)
    inp = make_batch([arr[i] for i in range(n)])
    dev = LzDevice()
    codec = Codec(FMT[kind])
    stream = torch.cuda.current_stream().cuda_stream
    max_out = codec.compress_get_max_output_chunk_size(CHUNK)
    assert dev.max_compressed_bytes(kind, CHUNK) == max_out
    ticket = torch.zeros(1, dtype=torch.int64, device="cuda")

    # compression, batched and warp-level
    lout = empty_batch(n, max_out, fill=0)
    ctb = codec.compress_get_temp_size(n, CHUNK)
    ctemp = torch.empty(max(ctb, 1), dtype=torch.uint8, device="cuda")

    def llif_compress():
        codec.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), CHUNK, n, ctemp.data_ptr(), ctb,
                             lout.ptrs.data_ptr(), lout.sizes.data_ptr(), stream)

    dout = empty_batch(n, max_out, fill=0)
    cstatus = torch.full((n,), -1, dtype=torch.int32, device="cuda")

    def dev_compress():
        ticket.zero_()
        dev.compress_async(kind, inp, dout, cstatus, 0, ticket)

    llif_compress()
    dev_compress()
    torch.cuda.synchronize()
    assert bool((cstatus == 0).all()), "compress_warp status"
    lsizes = lout.sizes.cpu().numpy()
    assert (dout.sizes.cpu().numpy() == lsizes).all(), "compressed sizes"
    assert dout.to_host(lsizes) == lout.to_host(lsizes), "compress_warp stream != batched stream"
    comp_bytes = int(lsizes.sum())

    # both decoders, the unfused and the fused sum over the batched encoder's streams
    comp = make_batch(lout.to_host(lsizes))
    outs = {k: empty_batch(n, CHUNK, fill=0) for k in ("llif", "dev", "fused")}
    dtb = codec.decompress_get_temp_size(n, CHUNK)
    dtemp = torch.empty(max(dtb, 1), dtype=torch.uint8, device="cuda")
    actual = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in ("llif", "dev")}
    status = {k: torch.full((n,), -1, dtype=torch.int32, device="cuda") for k in outs}
    sums = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in ("unfused", "fused")}
    sum_ticket = torch.zeros(1, dtype=torch.int64, device="cuda")

    def llif_decompress():
        o = outs["llif"]
        codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), o.sizes.data_ptr(),
                               actual["llif"].data_ptr(), n, dtemp.data_ptr(), dtb, o.ptrs.data_ptr(),
                               status["llif"].data_ptr(), stream)

    def dev_decompress():
        ticket.zero_()
        dev.decompress_async(kind, comp, outs["dev"], actual["dev"], status["dev"], ticket)

    def llif_decompress_sum():
        llif_decompress()
        sum_ticket.zero_()
        dev.sum_async(outs["llif"], actual["llif"], sums["unfused"], sum_ticket)

    def fused_sum():
        ticket.zero_()
        dev.decompress_sum_async(kind, comp, outs["fused"], sums["fused"], status["fused"], ticket)

    for fn in (llif_decompress_sum, dev_decompress, fused_sum):
        fn()
    torch.cuda.synchronize()
    for k in outs:
        assert bool((status[k] == 0).all()), (k, "status")
        assert torch.equal(outs[k].slab[: n * CHUNK], raw_dev), (k, "bytes")
    for k in actual:
        assert bool((actual[k] == CHUNK).all()), (k, "actual")
    for k in sums:
        assert (sums[k].cpu().numpy().view(np.uint64) == want_sums).all(), (k, "sums")

    uncomp = n * CHUNK
    for name, fn in (("batched_decompress", llif_decompress), ("warp_decompress", dev_decompress),
                     ("batched_decompress_sum", llif_decompress_sum), ("fused_decompress_sum", fused_sum),
                     ("batched_compress", llif_compress), ("warp_compress", dev_compress)):
        ms = time_ms(fn, args.steps, args.warmup)
        print(json.dumps({"format": FMT[kind], "call": name, "dataset": DATASET[kind], "chunks": n,
                          "ratio": round(uncomp / comp_bytes, 3), "ms": round(ms, 3),
                          "gbs": round(uncomp / ms / 1e6, 2), "steps": args.steps, "warmup": args.warmup}),
              flush=True)


if __name__ == "__main__":
    main()
