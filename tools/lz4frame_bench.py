"""Time batched LZ4 frame decompression (nvcompBatchedLZ4FrameDecompressAsync, include/nvcomp/lz4frame.h).

    python tools/lz4frame_bench.py [--steps 20] [--warmup 5]

Workloads, timed on cuda:0 with CUDA events (--steps back-to-back calls after --warmup):
  (a) single-block frames   10 000 x 64 KB chunks, half run-length int32 and half tabular float32 (datagen), each one
                            pyarrow LZ4 frame (pyarrow 24 writes FLG 0x60: independent 64 KB blocks, no checksums);
                            frames pyarrow stored as one uncompressed block are left out.  Timed against
                            nvcompBatchedLZ4DecompressAsync on the same block bytes cut out of those frames: each frame
                            holds one block, so the difference is the frame layer's cost.
  (b) large linked frames   160 x 4 MB chunks of linked 64 KB blocks (LZ4F_compressFrame), without and with the
                            content checksum: the difference prices XXH32.
  (c) CPU baseline          host liblz4 LZ4F_decompress on (a) and (b), one thread per core.
Every GPU figure is checked against the input before it is timed.  GB/s = decompressed bytes / time; the HBM share is
(compressed + decompressed bytes) / time over the card's peak HBM bandwidth (3.35 TB/s on the H100 SXM5 80 GB).  The
card name, power limit and maximum SM clock are read in the same run.  Prints one JSON line per figure, writes
nothing."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_PEAK = 3.35e12


def smi() -> dict:
    fields = "name,power.limit,clocks.max.sm"
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


def gpu_case(fmt, chunks, raw, cap, steps, warmup):
    from nvcomp_b200.batched import Codec, make_batch
    codec = Codec(fmt)
    comp = make_batch(chunks)
    out = make_batch([bytes(cap)] * len(chunks))
    out.sizes = torch.full((len(chunks),), cap, dtype=torch.int64, device="cuda")
    n = len(chunks)
    tb = codec.decompress_get_temp_size(n, cap)
    temp = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
    actual = torch.zeros(n, dtype=torch.int64, device="cuda")
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    sh = torch.cuda.current_stream().cuda_stream

    def call():
        codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(), actual.data_ptr(),
                               n, temp.data_ptr(), tb, out.ptrs.data_ptr(), status.data_ptr(), sh)
    call()
    torch.cuda.synchronize()
    assert (status == 0).all().item() and (actual == cap).all().item(), fmt
    slab = out.slab.cpu().numpy()
    assert all(slab[o:o + cap].tobytes() == raw[i] for i, o in enumerate(out.offsets)), fmt
    ms = time_ms(call, steps, warmup)
    ub, cb = n * cap, sum(len(c) for c in chunks)
    return {"ms": round(ms, 4), "GBps": round(ub / ms / 1e6, 1), "hbm_share": round((ub + cb) / ms * 1e3 / HBM_PEAK, 3),
            "ratio": round(ub / cb, 2)}


def cpu_case(lz4f, chunks, cap):
    threads = os.cpu_count() or 1

    def one(c):
        buf = C.create_string_buffer(cap + 64)
        ctx = C.c_void_p()
        lz4f.lib.LZ4F_createDecompressionContext(C.byref(ctx), lz4f.VERSION)
        src = C.create_string_buffer(c, len(c))
        ssz, dsz = C.c_size_t(len(c)), C.c_size_t(cap + 64)
        r = lz4f.lib.LZ4F_decompress(ctx, buf, C.byref(dsz), src, C.byref(ssz), None)
        lz4f.lib.LZ4F_freeDecompressionContext(ctx)
        assert r == 0 and dsz.value == cap
    best = None
    with ThreadPoolExecutor(threads) as ex:
        for _ in range(3):
            t = time.perf_counter()
            list(ex.map(one, chunks))
            dt = time.perf_counter() - t
            best = dt if best is None else min(best, dt)
    return {"ms": round(best * 1e3, 2), "GBps": round(len(chunks) * cap / best / 1e9, 2), "threads": threads}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import pyarrow as pa
    import lz4frame_writer as F
    from nvcomp_b200 import datagen
    card = smi()
    lz4f = F.LibLZ4F()
    emit = lambda d: print(json.dumps({**d, "card": card}), flush=True)   # noqa: E731

    data = np.concatenate([datagen.runlength_i32(5000, seed=61).view(np.uint8),
                           datagen.tabular_f32(5000, seed=62).view(np.uint8)])
    raw = [r.tobytes() for r in data]
    pc = pa.Codec("lz4")
    frames = [pc.compress(r).to_pybytes() for r in raw]
    # one block per frame: 7-byte header (no checksums or optional fields, 64 KB blocks), the 4-byte block size, the
    # block, the EndMark.  pyarrow stores a chunk that does not compress as one uncompressed block: those frames have
    # no LZ4 block to compare with and are left out of both figures.
    keep, blocks = [], []
    for i, f in enumerate(frames):
        assert f[4] & 0x1D == 0 and f[5] == 0x40
        size = int.from_bytes(f[7:11], "little")
        if size < 1 << 31:
            assert 11 + size + 4 == len(f), "one block per frame"
            keep.append(i)
            blocks.append(f[11:11 + size])
    frames, raw = [frames[i] for i in keep], [raw[i] for i in keep]
    emit({"workload": "a_single_block_frames", "api": "LZ4Frame", "chunks": len(frames),
          **gpu_case("LZ4Frame", frames, raw, 65536, args.steps, args.warmup)})
    emit({"workload": "a_single_block_frames", "api": "LZ4 (same blocks)",
          **gpu_case("LZ4", blocks, raw, 65536, args.steps, args.warmup)})
    emit({"workload": "a_single_block_frames", "api": "CPU liblz4 LZ4F_decompress", **cpu_case(lz4f, frames, 65536)})

    big = np.concatenate([datagen.runlength_i32(80 * 64, seed=63).view(np.uint8).reshape(-1),
                          datagen.tabular_f32(80 * 64, seed=64).view(np.uint8).reshape(-1)]).tobytes()
    raw4 = [big[i:i + (4 << 20)] for i in range(0, len(big), 4 << 20)]
    assert len(raw4) == 160
    for cs in (False, True):
        fr = [lz4f.compress_frame(r, 4, True, cs) for r in raw4]
        name = "b_linked_4mb_" + ("content_checksum" if cs else "no_checksum")
        emit({"workload": name, "api": "LZ4Frame", **gpu_case("LZ4Frame", fr, raw4, 4 << 20, args.steps, args.warmup)})
        emit({"workload": name, "api": "CPU liblz4 LZ4F_decompress", **cpu_case(lz4f, fr, 4 << 20)})


if __name__ == "__main__":
    main()
