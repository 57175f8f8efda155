"""Time the warp-level Cascaded device API (include/nvcomp/device/cascaded.cuh) next to the batched C API on the same
chunks, and measure what fusing the decode into a consuming kernel saves.

    python tools/cascaded_device_bench.py [--chunks 10000] [--steps 20] [--warmup 5]

The workload is bench.py's Cascaded workload: --chunks x 64 KB of sorted int64 (datagen.sorted_i64), options
{chunk_size 4096, LONGLONG, 1 RLE, 1 delta, bit-packing}.  Each warp-level kernel gets decompress_smem_bytes(opts) of
shared memory per warp.  Timed on cuda:0:
  batched_decompress    nvcompBatchedCascadedDecompressAsync (one CTA per chunk, one warp per partition)
  warp_decompress       decompress_warp, one warp per chunk (build/tests/libcascaded_device.so)
  batched_decompress_sum  nvcompBatchedCascadedDecompressAsync, then a warp-per-chunk kernel that sums each decoded
                        chunk as int64 (16-byte loads)
  fused_sum             for_each_block<int64_t>: the same sums, decoded in shared memory and registers, nothing
                        stored to global memory
  fused_sum_check       for_each_block's first pass alone (the partition walk over the run-length streams that makes
                        the visit all-or-nothing); fused_sum minus this is the decode-and-visit pass
  batched_compress / warp_compress   nvcompBatchedCascadedCompressAsync against compress_warp
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
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cascaded_device_bench.py needs a CUDA GPU")
    from cascaded_device import CascadedDevice
    from nvcomp_b200 import datagen
    from nvcomp_b200._lib import CascadedOpts, Type
    from nvcomp_b200.batched import Codec, empty_batch, make_batch

    torch.cuda.set_device(0)
    card = {"name": torch.cuda.get_device_name(0), **smi("power.limit,clocks.max.sm")}
    print(json.dumps({"card": card}), flush=True)
    n = args.chunks
    opts = (4096, int(Type.LONGLONG), 1, 1, 1)
    arr = datagen.sorted_i64(n)
    raw_dev = torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1)).cuda()
    want_sums = arr.view(np.int64).reshape(n, -1).astype(np.uint64).sum(axis=1, dtype=np.uint64).view(np.int64)
    inp = make_batch([arr[i] for i in range(n)])
    dev = CascadedDevice()
    codec = Codec("Cascaded", opts=CascadedOpts(*opts))
    region = dev.decompress_smem_bytes(opts)
    stream = torch.cuda.current_stream().cuda_stream
    max_out = codec.compress_get_max_output_chunk_size(CHUNK)
    assert dev.max_compressed_bytes(CHUNK, opts) == max_out

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
        dev.compress_async(inp, dout, cstatus, opts)

    llif_compress()
    dev_compress()
    torch.cuda.synchronize()
    assert bool((cstatus == 0).all()), "compress_warp status"
    lsizes = lout.sizes.cpu().numpy()
    assert (dout.sizes.cpu().numpy() == lsizes).all(), "compressed sizes"
    assert dout.to_host(lsizes) == lout.to_host(lsizes), "compress_warp stream != batched stream"
    comp_bytes = int(lsizes.sum())

    # both decoders, the unfused sum and the fused sum over the batched encoder's streams
    comp = make_batch(lout.to_host(lsizes))
    outs = {k: empty_batch(n, CHUNK, fill=0) for k in ("llif", "dev")}
    dtb = codec.decompress_get_temp_size(n, CHUNK)
    dtemp = torch.empty(max(dtb, 1), dtype=torch.uint8, device="cuda")
    actual = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in outs}
    status = {k: torch.full((n,), -1, dtype=torch.int32, device="cuda") for k in outs}
    sums = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in ("unfused", "fused")}
    fstatus = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    checked = torch.zeros(n, dtype=torch.int32, device="cuda")

    def llif_decompress():
        o = outs["llif"]
        codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), o.sizes.data_ptr(),
                               actual["llif"].data_ptr(), n, dtemp.data_ptr(), dtb, o.ptrs.data_ptr(),
                               status["llif"].data_ptr(), stream)

    def dev_decompress():
        dev.decompress_async(comp, outs["dev"], actual["dev"], status["dev"], region)

    def llif_decompress_sum():
        llif_decompress()
        dev.sum_i64_async(outs["llif"], actual["llif"], sums["unfused"])

    def fused_sum():
        dev.fused_sum_async(comp, sums["fused"], fstatus, region)

    def fused_sum_check():
        dev.check_async(comp, checked, region)

    for fn in (llif_decompress_sum, dev_decompress, fused_sum, fused_sum_check):
        fn()
    torch.cuda.synchronize()
    for k in outs:
        assert bool((status[k] == 0).all()) and bool((actual[k] == CHUNK).all()), (k, "status / actual")
        assert torch.equal(outs[k].slab[: n * CHUNK], raw_dev), (k, "bytes")
    assert bool((fstatus == 0).all()), "for_each_block status"
    assert bool((checked == 1).all()), "for_each_block check pass"
    for k in sums:
        assert (sums[k].cpu().numpy() == want_sums).all(), (k, "sums")

    uncomp = n * CHUNK
    for name, fn in (("batched_decompress", llif_decompress), ("warp_decompress", dev_decompress),
                     ("batched_decompress_sum", llif_decompress_sum), ("fused_sum", fused_sum),
                     ("fused_sum_check", fused_sum_check), ("batched_compress", llif_compress),
                     ("warp_compress", dev_compress)):
        ms = time_ms(fn, args.steps, args.warmup)
        print(json.dumps({"format": "Cascaded", "call": name, "dataset": "sorted_i64", "opts": list(opts),
                          "smem_per_warp": region, "chunks": n, "ratio": round(uncomp / comp_bytes, 3),
                          "ms": round(ms, 3), "gbs": round(uncomp / ms / 1e6, 2), "steps": args.steps,
                          "warmup": args.warmup}), flush=True)


if __name__ == "__main__":
    main()
