#!/usr/bin/env python3
"""Schedule trace of one batched LZ decode call (Snappy or LZ4): where each chunk ran and when.

    bash tools/build_variants.sh trace                  # -> build/variants/trace/libnvcomp.so (-DB200_LZ_TRACE)
    python tools/lz_trace.py [--lib build/variants/trace/libnvcomp.so] [--codec snappy] [--json out.json]

Runs the bench.py workload (10 000 x 64 KB chunks, bench.py's Workload class: same data, same compressed layout, same
call) three times untimed, then once with the trace buffers cleared, and prints from the trace build's records
(lz_sched.cuh, B200_LZ_TRACE):
  - each kernel's span (first warp in to last warp out);
  - chunk decode latency per list (p50 / p90 / max), and per column for the four-column tabular_f32 data;
  - resident dense and light warps per SM over time (CTA residency: a CTA holds its 4 warp slots from its first warp's
    entry to its last warp's exit), time-weighted mean over the SMs in bins of --bin-us;
  - the last chunk to finish, with its list and start time.
Times are %globaltimer nanoseconds relative to the first warp that entered either kernel.  The trace build adds a few
instructions and registers per chunk, so its times are close to, not equal to, the product build's.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TRACE_CHUNKS = 1 << 16          # lz_sched.cuh kLzTraceChunks
TRACE_WARPS = 1 << 15           # lz_sched.cuh kLzTraceWarps (per list)
WARPS_PER_CTA = 4               # kLzDecWarps
LISTS = ("light", "dense")      # record field `list`: 0 light, 1 dense
CHUNK_T = np.dtype([("list", "<u4"), ("smid", "<u4"), ("t0", "<u8"), ("t1", "<u8")])
WARP_T = np.dtype([("smid", "<u4"), ("chunks", "<u4"), ("t_enter", "<u8"), ("t_exit", "<u8")])


def pct(a, q):
    return round(float(np.percentile(a, q)), 1) if len(a) else None


def run(args):
    import torch
    from nvcomp_b200 import _lib
    _lib.lib_path = lambda: os.path.abspath(args.lib)      # the trace build instead of the product library
    lib = _lib.load()
    clear = getattr(lib, f"b200_lz_trace_clear_{args.codec}", None)
    fetch = getattr(lib, f"b200_lz_trace_fetch_{args.codec}", None)
    if clear is None or fetch is None:
        raise SystemExit(f"{args.lib} has no trace entry points: build it with -DB200_LZ_TRACE")
    fetch.argtypes = [C.c_void_p, C.c_void_p]
    import bench
    dataset = args.dataset or bench.DEFAULT_DATASET[args.codec]
    w = bench.Workload(args.codec, dataset, args.chunks)
    sh = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        w.launch(sh)
    w.check()
    if clear() != 0:
        raise SystemExit("trace clear failed")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    w.launch(sh)
    e1.record()
    torch.cuda.synchronize()
    chunks = np.zeros(TRACE_CHUNKS, dtype=CHUNK_T)
    warps = np.zeros(2 * TRACE_WARPS, dtype=WARP_T)
    if fetch(chunks.ctypes.data, warps.ctypes.data) != 0:
        raise SystemExit("trace fetch failed")
    w.check()
    return summarize(chunks[: w.n], warps.reshape(2, TRACE_WARPS), dataset, args.bin_us, e0.elapsed_time(e1),
                     torch.cuda.get_device_name())


def summarize(chunks, warps, dataset, bin_us, call_ms, device):
    n = len(chunks)
    if not (chunks["t1"] > 0).all():
        raise SystemExit(f"{int((chunks['t1'] == 0).sum())} of {n} chunks have no trace record")
    live = [warps[l][warps[l]["t_enter"] > 0] for l in range(2)]
    origin = min(int(x["t_enter"].min()) for x in live if len(x))
    us = lambda t: (t.astype(np.float64) - origin) / 1e3 if isinstance(t, np.ndarray) else (float(t) - origin) / 1e3
    out = {"device": device, "dataset": dataset, "chunks": n, "call_ms_event": round(call_ms, 4), "kernels": {},
           "latency_us": {}, "residency": {}, "last_chunk": None}
    sms = np.unique(np.concatenate([x["smid"] for x in live]))
    for l, name in enumerate(LISTS):
        x = live[l]
        sel = chunks["list"] == l
        lat = (chunks["t1"][sel] - chunks["t0"][sel]).astype(np.float64) / 1e3
        start = us(chunks["t0"][sel])
        out["kernels"][name] = {"warps": int(len(x)), "chunks": int(sel.sum()),
                                "span_us": [round(float(us(x["t_enter"]).min()), 1), round(float(us(x["t_exit"]).max()), 1)]
                                if len(x) else None,
                                "chunk_start_us": {"first": pct(start, 0), "p50": pct(start, 50), "last": pct(start, 100)}}
        out["latency_us"][name] = {"p50": pct(lat, 50), "p90": pct(lat, 90), "max": pct(lat, 100)}
    if dataset == "tabular_f32":
        names = ("price_walk", "lowcard", "clustered", "sensor")
        lat = (chunks["t1"] - chunks["t0"]).astype(np.float64) / 1e3
        idx = np.arange(n)
        for col in range(4):
            s = idx % 4 == col
            out["latency_us"][f"column{col}_{names[col]}"] = {
                "list": LISTS[int(np.bincount(chunks["list"][s]).argmax())],
                "p50": pct(lat[s], 50), "p90": pct(lat[s], 90), "max": pct(lat[s], 100),
                "start_p50_us": pct(us(chunks["t0"][s]), 50), "end_max_us": pct(us(chunks["t1"][s]), 100)}
    # CTA residency, time-weighted per bin
    end = max(float(us(x["t_exit"]).max()) for x in live if len(x))
    edges = np.arange(0.0, end + bin_us, bin_us)
    rows = {name: np.zeros(len(edges) - 1) for name in LISTS}
    for l, name in enumerate(LISTS):
        ws = warps[l]
        idx = np.nonzero(ws["t_enter"] > 0)[0]
        if not len(idx):
            continue
        cta = idx // WARPS_PER_CTA
        for c in np.unique(cta):
            m = ws[idx[cta == c]]
            a, b = float(us(m["t_enter"]).min()), float(us(m["t_exit"]).max())
            ov = np.clip(np.minimum(edges[1:], b) - np.maximum(edges[:-1], a), 0.0, None)
            rows[name] += WARPS_PER_CTA * ov / bin_us
    out["residency"] = {"bin_us": bin_us, "sms": int(len(sms)),
                        "bins": [{"t_us": round(float(t), 1),
                                  "dense_warps_per_sm": round(float(rows["dense"][i] / len(sms)), 2),
                                  "light_warps_per_sm": round(float(rows["light"][i] / len(sms)), 2)}
                                 for i, t in enumerate(edges[:-1])]}
    k = int(np.argmax(chunks["t1"]))
    out["last_chunk"] = {"chunk": k, "list": LISTS[int(chunks["list"][k])], "smid": int(chunks["smid"][k]),
                         "start_us": round(float(us(chunks["t0"][k])), 1), "end_us": round(float(us(chunks["t1"][k])), 1),
                         "latency_us": round(float(chunks["t1"][k] - chunks["t0"][k]) / 1e3, 1)}
    for l, name in enumerate(LISTS):
        sel = chunks["list"] == l
        if sel.any():
            out["kernels"][name]["last_chunk_end_us"] = round(float(us(chunks["t1"][sel]).max()), 1)
    return out


def show(r):
    print(f"{r['device']}  {r['dataset']}  {r['chunks']} chunks  call {r['call_ms_event']:.3f} ms (trace build, events)")
    for name, k in r["kernels"].items():
        print(f"  {name:5s} kernel: {k['warps']} warps, {k['chunks']} chunks, span {k['span_us']} us, "
              f"chunk starts {k['chunk_start_us']}, last chunk ends {k.get('last_chunk_end_us')} us")
    print("  chunk latency (us):")
    for name, v in r["latency_us"].items():
        print(f"    {name:22s} " + "  ".join(f"{a}={b}" for a, b in v.items()))
    print(f"  resident warps per SM (time-weighted mean over {r['residency']['sms']} SMs):")
    print("    t_us     dense  light")
    for b in r["residency"]["bins"]:
        print(f"    {b['t_us']:7.0f}  {b['dense_warps_per_sm']:5.1f}  {b['light_warps_per_sm']:5.1f}")
    print(f"  last chunk to finish: {r['last_chunk']}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "build", "variants", "trace", "libnvcomp.so"))
    ap.add_argument("--codec", default="snappy", choices=["snappy", "lz4"])
    ap.add_argument("--dataset", default=None, help="default: bench.py's dataset of the codec")
    ap.add_argument("--chunks", type=int, default=10000)
    ap.add_argument("--bin-us", type=float, default=50.0)
    ap.add_argument("--json", default=None, help="also write the summary as JSON to this path")
    args = ap.parse_args()
    if args.chunks > TRACE_CHUNKS:
        ap.error(f"the trace records at most {TRACE_CHUNKS} chunks")
    r = run(args)
    show(r)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(r, f)


if __name__ == "__main__":
    main()
