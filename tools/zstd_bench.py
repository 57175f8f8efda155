"""Time batched Zstd decompression (nvcompBatchedZstdDecompressAsync) on one GPU, next to the host's libzstd on all
cores.

    python tools/zstd_bench.py [--chunks 10000] [--steps 20] [--warmup 5] [--levels 1,3,19]

Each dataset (datagen.tabular_f32, the flagship workload's data, the typed runlength_i32 and lowentropy_bytes) is cut
into 64 KB chunks, compressed on the host by libzstd at each level (checksum off, libzstd's default) and by pyarrow's
default Zstd codec, and decoded on cuda:0.  Before any timing a parity gate checks every status, size and byte.  The
GPU figure is K back-to-back calls between two CUDA events, after warm-up; GB/s = uncompressed bytes / time, roofline
share = (compressed + uncompressed + 44 B per chunk) / time / 3.35 TB/s.  The size query (GetDecompressSizeAsync)
runs pass 1 and the literal decode with every store off, so decode_ms - size_query_ms is the cost of pass 2 (the
second sequence decode and all output writes).  The host figure is libzstd's ZSTD_decompressDCtx in a native
pthread loop on all cores (one context and output buffer per thread, timed in C; compiled into a temporary
directory).  Card name, power limit, and the SM clock and power draw right after the timed calls are
read in the same run.  Needs a CUDA GPU and libzstd.so.1: there is no fallback.  Prints one JSON line per
measurement and writes nothing."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_GBS = 3350.0     # H100 SXM data sheet
CHUNK = 65536


def smi(fields: str) -> dict:
    try:
        q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(fields.split(","), [x.strip() for x in q.split(",")]))
    except Exception as e:  # noqa: BLE001 -- the figure is reported as missing, the timing still stands
        return {"unavailable": type(e).__name__}


# Host baseline: libzstd's ZSTD_decompressDCtx in a native loop, one pthread per core over a contiguous range of
# chunks, one DCtx and one output buffer per thread, timed in C (no Python in the timed region).  Compiled into a
# temporary directory at run time.
_HOST_C = r"""
#include <dlfcn.h>
#include <pthread.h>
#include <stdlib.h>
#include <time.h>
typedef size_t (*dec_t)(void*, void*, size_t, const void*, size_t);
typedef void* (*mk_t)(void);
typedef size_t (*fr_t)(void*);
typedef unsigned (*ie_t)(size_t);
static dec_t dec; static mk_t mk; static fr_t fr; static ie_t ie;
struct job { const void* const* src; const size_t* n; size_t lo, hi, cap; long bad; };
static void* run(void* a) {
  struct job* j = (struct job*)a;
  void* d = mk();
  unsigned char* out = (unsigned char*)malloc(j->cap);
  for (size_t i = j->lo; i < j->hi; ++i) {
    size_t k = dec(d, out, j->cap, j->src[i], j->n[i]);
    if (ie(k) || k != j->cap) ++j->bad;
  }
  free(out);
  fr(d);
  return 0;
}
/* seconds of the fastest of reps passes over all chunks; -1 if libzstd is missing or a chunk failed */
double host_zstd(const void* const* src, const size_t* n, size_t count, size_t cap, int threads, int reps) {
  void* h = dlopen("libzstd.so.1", RTLD_NOW);
  if (!h) return -1;
  dec = (dec_t)dlsym(h, "ZSTD_decompressDCtx"); mk = (mk_t)dlsym(h, "ZSTD_createDCtx");
  fr = (fr_t)dlsym(h, "ZSTD_freeDCtx"); ie = (ie_t)dlsym(h, "ZSTD_isError");
  struct job* jobs = (struct job*)calloc((size_t)threads, sizeof(struct job));
  pthread_t* tid = (pthread_t*)calloc((size_t)threads, sizeof(pthread_t));
  double best = 1e30;
  for (int r = 0; r < reps; ++r) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < threads; ++t) {
      struct job* j = &jobs[t];
      j->src = src; j->n = n; j->cap = cap; j->bad = 0;
      j->lo = count * (size_t)t / (size_t)threads; j->hi = count * (size_t)(t + 1) / (size_t)threads;
      pthread_create(&tid[t], 0, run, j);
    }
    long bad = 0;
    for (int t = 0; t < threads; ++t) { pthread_join(tid[t], 0); bad += jobs[t].bad; }
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (bad) return -1;
    double s = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
    if (s < best) best = s;
  }
  free(jobs); free(tid);
  return best;
}
"""


def host_baseline():
    """ctypes handle of the native host loop (compiled with the system C compiler into a temporary directory)."""
    d = tempfile.mkdtemp(prefix="zstd_bench_")
    src, lib = os.path.join(d, "host.c"), os.path.join(d, "host.so")
    with open(src, "w") as f:
        f.write(_HOST_C)
    subprocess.run(["cc", "-O2", "-shared", "-fPIC", "-o", lib, src, "-ldl", "-lpthread"], check=True)
    h = C.CDLL(lib)
    h.host_zstd.restype = C.c_double
    h.host_zstd.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int]
    shutil.rmtree(d)
    return h


def host_zstd(h, streams, threads, reps=5) -> float:
    """seconds per pass of ZSTD_decompressDCtx over all streams on `threads` threads, best of reps"""
    ptrs = (C.c_char_p * len(streams))(*streams)
    lens = (C.c_size_t * len(streams))(*[len(s) for s in streams])
    s = h.host_zstd(C.cast(ptrs, C.c_void_p), C.cast(lens, C.c_void_p), len(streams), CHUNK, threads, reps)
    assert s > 0, "host libzstd failed on a chunk"
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--levels", default="1,3,19")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("zstd_bench: no CUDA device (this measures the GPU decoder; there is no CPU fallback)")
    torch.cuda.set_device(0)
    import pyarrow as pa
    from zstd_writer import LibZstd
    from nvcomp_b200 import datagen
    from nvcomp_b200.batched import Codec, empty_batch, make_batch

    zs = LibZstd()
    host = host_baseline()
    card = {"name": torch.cuda.get_device_name(0), **smi("power.limit,clocks.max.sm")}
    print(json.dumps({"card": card, "host_threads": os.cpu_count(), "libzstd": zs.version}), flush=True)
    pool = ThreadPoolExecutor(os.cpu_count())
    n = args.chunks
    codec = Codec("Zstd")
    producers = [(f"libzstd-{lv}", lambda c, lv=lv: zs.compress(c, lv)) for lv in map(int, args.levels.split(","))]
    producers.append(("pyarrow-default", lambda c: pa.Codec("zstd").compress(c, asbytes=True)))
    for dataset in ("tabular_f32", "runlength_i32", "lowentropy_bytes"):
        arr = getattr(datagen, dataset)(n)
        chunks = [arr[i].tobytes() for i in range(n)]
        raw_dev = torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(n, CHUNK)).cuda()
        for producer, fn in producers:
            streams = list(pool.map(fn, chunks, chunksize=16))
            comp_bytes = sum(len(s) for s in streams)
            comp = make_batch(streams)
            out = empty_batch(n, CHUNK, fill=0)
            tb = codec.decompress_get_temp_size(n, CHUNK)
            temp = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
            actual = torch.zeros(n, dtype=torch.int64, device="cuda")
            status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            sizes = torch.zeros(n, dtype=torch.int64, device="cuda")
            stream = torch.cuda.current_stream().cuda_stream

            def call():
                codec.decompress_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), out.sizes.data_ptr(),
                                       actual.data_ptr(), n, temp.data_ptr(), tb, out.ptrs.data_ptr(),
                                       status.data_ptr(), stream)

            def size_call():
                codec.get_decompress_size_async(comp.ptrs.data_ptr(), comp.sizes.data_ptr(), sizes.data_ptr(), n,
                                                stream)

            # parity gate: every chunk decodes to its input
            call()
            size_call()
            torch.cuda.synchronize()
            assert bool((status == 0).all()), (producer, dataset, "status")
            assert bool((actual == CHUNK).all()), (producer, dataset, "actual")
            assert bool((sizes == CHUNK).all()), (producer, dataset, "size query")
            assert torch.equal(out.slab[: n * CHUNK].view(n, CHUNK), raw_dev), (producer, dataset, "bytes")
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            timings = {}
            for name, fn in (("decode", call), ("size_query", size_call)):
                for _ in range(args.warmup):
                    fn()
                t0.record()
                for _ in range(args.steps):
                    fn()
                t1.record()
                if name == "decode":
                    during = smi("clocks.sm,power.draw")      # read while the timed calls run
                torch.cuda.synchronize()
                timings[name] = t0.elapsed_time(t1) / args.steps
            ms = timings["decode"]
            uncomp = n * CHUNK
            host_s = host_zstd(host, streams, os.cpu_count())
            print(json.dumps({
                "format": "Zstd", "dataset": dataset, "producer": producer, "chunks": n,
                "ratio": round(uncomp / comp_bytes, 3), "gpu_ms": round(ms, 3),
                "gpu_gbs": round(uncomp / ms / 1e6, 2),
                "roofline_frac": round((comp_bytes + uncomp + 44 * n) / ms / 1e6 / HBM_GBS, 4),
                "size_query_ms": round(timings["size_query"], 3),
                "host_libzstd_gbs": round(uncomp / host_s / 1e9, 2), "host_threads": os.cpu_count(),
                "sm_clock_during": during.get("clocks.sm"), "power_during": during.get("power.draw"),
                "steps": args.steps, "warmup": args.warmup}), flush=True)
            del comp, out, temp
    pool.shutdown()


if __name__ == "__main__":
    main()
