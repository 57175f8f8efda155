#!/usr/bin/env python3
"""Developer benchmark: per-dataset compress/decompress throughput of one or more codecs.
(bench.py is the contract benchmark; this one is for kernel iteration.)"""
import argparse
import json
import sys
import os

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nvcomp_b200 import datagen  # noqa: E402
from nvcomp_b200.batched import Batch, Codec, empty_batch  # noqa: E402

FMT = {"lz4": "LZ4", "snappy": "Snappy", "cascaded": "Cascaded", "bitcomp": "Bitcomp", "ans": "ANS"}


def dev_batch(data: np.ndarray) -> Batch:
    n, chunk = data.shape
    slab = torch.from_numpy(data.reshape(-1)).cuda()
    offsets = np.arange(n, dtype=np.int64) * chunk
    return Batch(slab, torch.from_numpy(offsets + slab.data_ptr()).cuda(),
                 torch.full((n,), chunk, dtype=torch.int64, device="cuda"), offsets)


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in evs)
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--codecs", default="lz4,snappy")
    ap.add_argument("--datasets", default="runlength_i32,tabular_f32,snappy_synth,random_bytes")
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--opts", default="")
    ap.add_argument("--no-verify", action="store_true")
    args = ap.parse_args()
    for ds in args.datasets.split(","):
        if ":" in ds:
            name, col = ds.split(":")
            data = datagen.tabular_f32(args.chunks, column=int(col))
        else:
            data = datagen.DATASETS[ds](args.chunks)
        inp = dev_batch(data)
        n, chunk = data.shape
        total = n * chunk
        for ck in args.codecs.split(","):
            opts = None
            if ck == "cascaded":
                from nvcomp_b200._lib import CascadedOpts, Type
                t = Type.LONGLONG if "i64" in ds else Type.INT
                opts = CascadedOpts(4096, t, 1, 1, 1)
            if ck == "bitcomp":
                from nvcomp_b200._lib import BitcompOpts, Type
                t = Type.ULONGLONG if "i64" in ds else Type.UINT
                opts = BitcompOpts(0, t)
            codec = Codec(FMT[ck], opts=opts)
            comp = codec.compress(inp, max_chunk=chunk)
            torch.cuda.synchronize()
            csum = int(comp.sizes.sum().item())
            tb = codec.compress_get_temp_size(n, chunk)
            ctemp = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
            s = torch.cuda.current_stream().cuda_stream
            c_ms, c_best = time_ms(lambda: codec.compress_async(
                inp.ptrs.data_ptr(), inp.sizes.data_ptr(), chunk, n, ctemp.data_ptr(), tb,
                comp.ptrs.data_ptr(), comp.sizes.data_ptr(), s), max(args.iters // 3, 2), 1)
            out = empty_batch(n, chunk)
            dtb = codec.decompress_get_temp_size(n, chunk)
            dtemp = torch.empty(max(dtb, 1), dtype=torch.uint8, device="cuda")
            actual = torch.zeros(n, dtype=torch.int64, device="cuda")
            status = torch.zeros(n, dtype=torch.int32, device="cuda")
            d_ms, d_best = time_ms(lambda: codec.decompress_async(
                comp.ptrs.data_ptr(), comp.sizes.data_ptr(), inp.sizes.data_ptr(), actual.data_ptr(), n,
                dtemp.data_ptr(), dtb, out.ptrs.data_ptr(), status.data_ptr(), s), args.iters, 3)
            ok = True
            if not args.no_verify:
                ok = bool((status == 0).all().item()) and torch.equal(out.slab[:total], inp.slab[:total])
            alg = total + csum + 44 * n
            print(json.dumps({"codec": ck, "dataset": ds, "chunks": n, "ratio": round(total / csum, 3),
                              "comp_GBps": round(total / c_ms / 1e6, 1),
                              "decomp_GBps": round(total / d_ms / 1e6, 1),
                              "decomp_best_GBps": round(total / d_best / 1e6, 1),
                              "decomp_ms": round(d_ms, 3),
                              "roofline_frac": round(alg / d_ms / 1e6 / 3350.0, 4), "ok": ok}), flush=True)


if __name__ == "__main__":
    main()
