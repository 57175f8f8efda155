"""Time the warp-level ANS device API (include/nvcomp/device/ans.cuh) next to the batched C API on the same chunks.

    python tools/ans_device_bench.py [--chunks 10000] [--steps 20] [--warmup 5]

The workload is bench.py's ANS workload: --chunks x 64 KB low-entropy bytes (datagen.lowentropy_bytes).  Four calls
are timed on cuda:0: nvcompBatchedANSDecompressAsync and nvcompBatchedANSCompressAsync (one CTA per chunk), and the
warp-per-chunk kernels of build/tests/libans_device.so over decompress_warp and compress_warp (4 warps per CTA, one
warp per chunk; a warp decodes a chunk's 4 segments one after another).  Before any timing a parity gate checks that
the device API's streams equal the batched encoder's byte for byte and that both decoders return every chunk's
status, size and bytes.  Each figure is K back-to-back calls between two CUDA events, after warm-up; GB/s =
uncompressed bytes / time.  The card name and power limit are read in the same run.  Needs a CUDA GPU: there is no
fallback.  Prints one JSON line per measurement and writes nothing."""
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
        raise SystemExit("ans_device_bench.py needs a CUDA GPU")
    from ans_device import AnsDevice
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import Codec, empty_batch, make_batch

    torch.cuda.set_device(0)
    card = {"name": torch.cuda.get_device_name(0), **smi("power.limit,clocks.max.sm")}
    print(json.dumps({"card": card}), flush=True)
    n = args.chunks
    arr = datagen.lowentropy_bytes(n)
    raw_dev = torch.from_numpy(np.ascontiguousarray(arr).reshape(-1)).cuda()
    inp = make_batch([arr[i] for i in range(n)])
    dev = AnsDevice()
    codec = Codec("ANS")
    stream = torch.cuda.current_stream().cuda_stream
    max_out = codec.compress_get_max_output_chunk_size(CHUNK)
    assert dev.max_compressed_bytes(CHUNK) == max_out

    # batched compression
    lout = empty_batch(n, max_out, fill=0)
    ctb = codec.compress_get_temp_size(n, CHUNK)
    ctemp = torch.empty(max(ctb, 1), dtype=torch.uint8, device="cuda")

    def llif_compress():
        codec.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), CHUNK, n, ctemp.data_ptr(), ctb,
                             lout.ptrs.data_ptr(), lout.sizes.data_ptr(), stream)

    # warp-level compression
    dout = empty_batch(n, max_out, fill=0)
    dtmp = dev.compress_temp(n)
    cstatus = torch.full((n,), -1, dtype=torch.int32, device="cuda")

    def dev_compress():
        dev.compress_async(inp, dout, cstatus, dtmp)

    llif_compress()
    dev_compress()
    torch.cuda.synchronize()
    assert bool((cstatus == 0).all()), "compress_warp status"
    lsizes = lout.sizes.cpu().numpy()
    assert (dout.sizes.cpu().numpy() == lsizes).all(), "compressed sizes"
    assert dout.to_host(lsizes) == lout.to_host(lsizes), "compress_warp stream != batched stream"
    comp_bytes = int(lsizes.sum())

    # both decoders over the batched encoder's streams
    comp = make_batch(lout.to_host(lsizes))
    outs = {k: empty_batch(n, CHUNK, fill=0) for k in ("llif", "dev")}
    dtb = codec.decompress_get_temp_size(n, CHUNK)
    dtemp = torch.empty(max(dtb, 1), dtype=torch.uint8, device="cuda")
    actual = {k: torch.zeros(n, dtype=torch.int64, device="cuda") for k in outs}
    status = {k: torch.full((n,), -1, dtype=torch.int32, device="cuda") for k in outs}

    def llif_decompress():
        o = outs["llif"]
        codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), o.sizes.data_ptr(),
                               actual["llif"].data_ptr(), n, dtemp.data_ptr(), dtb, o.ptrs.data_ptr(),
                               status["llif"].data_ptr(), stream)

    def dev_decompress():
        dev.decompress_async(comp, outs["dev"], actual["dev"], status["dev"])

    llif_decompress()
    dev_decompress()
    torch.cuda.synchronize()
    for k in outs:
        assert bool((status[k] == 0).all()) and bool((actual[k] == CHUNK).all()), (k, "status / actual")
        assert torch.equal(outs[k].slab[: n * CHUNK], raw_dev), (k, "bytes")

    uncomp = n * CHUNK
    for name, fn in (("batched_decompress", llif_decompress), ("warp_decompress", dev_decompress),
                     ("batched_compress", llif_compress), ("warp_compress", dev_compress)):
        ms = time_ms(fn, args.steps, args.warmup)
        print(json.dumps({"format": "ANS", "call": name, "dataset": "lowentropy_bytes", "chunks": n,
                          "ratio": round(uncomp / comp_bytes, 3), "ms": round(ms, 3),
                          "gbs": round(uncomp / ms / 1e6, 2), "steps": args.steps, "warmup": args.warmup}),
              flush=True)


if __name__ == "__main__":
    main()
