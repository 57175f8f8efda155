"""Plain reference model of the Cascaded, Bitcomp and ANS streams (test infrastructure, CPU only).

Written from the stream definitions in the headers of nvcomp_b200/csrc/{cascaded,bitcomp,ans}.cu with Python's
arbitrary-precision ints, sharing nothing with oracle/.  For every input it predicts the fields an encoder
chooses -- header words, bit widths, frame-of-reference minima, delta bases, per-layer element counts, block
descriptors, the ANS mode and frequency table, partition / segment offsets, pad bytes and the total size -- and the
parse_* functions read the same fields back out of a stream, so `parse(stream) == model(input)` pins an encoder's
choices without a second bit-packer.

edge_chunks() and friends generate the inputs where typed encoders and decoders tend to go wrong.
numpy is used only to generate inputs."""
from __future__ import annotations

from collections import Counter
from itertools import groupby

import numpy as np

TYPE_SIZE = {0: 1, 1: 1, 2: 2, 3: 2, 4: 4, 5: 4, 6: 8, 7: 8}
SIGNED = {0, 2, 4, 6}
_FMT = {1: "B", 2: "H", 4: "I", 8: "Q"}
M64 = (1 << 64) - 1

CSC_MAGIC = 0x31435343
BTC_MAGIC = 0x31435442
ANS_MAGIC = 0x31534E41
ANS_SEG, ANS_M, ANS_L = 16384, 4096, 65536


def _r8(x: int) -> int:
    return (x + 7) & ~7


def _u32(b: bytes, o: int) -> int:
    return int.from_bytes(b[o:o + 4], "little")


def _u64(b: bytes, o: int) -> int:
    return int.from_bytes(b[o:o + 8], "little")


def elements(data: bytes, ts: int) -> list[int]:
    """The whole little-endian unsigned elements of `data` (trailing bytes dropped)."""
    whole = len(data) - len(data) % ts
    return memoryview(data[:whole]).cast(_FMT[ts]).tolist()


def _signed(v: int, ts: int) -> int:
    w = 8 * ts
    return v - (1 << w) if v >> (w - 1) else v


def _words(count: int, bits: int) -> int:
    return (count * bits + 63) // 64


# ------------------------------------------------------------------------------------------------ Cascaded
def _stream_hdr(vals: list[int], use_bp: bool, signed: bool, ts: int, raw_bits: int) -> tuple[int, int, int]:
    """(count, bits, min) of a packed stream.  Without bit-packing: the raw width and min 0.  With it: the width of
    max - min, the minimum taken in the stream's own signedness and stored as a sign-extended 64-bit word."""
    n = len(vals)
    if not use_bp:
        return (n, raw_bits, 0)
    if n == 0:
        return (0, 0, 0)
    xs = [_signed(v, ts) for v in vals] if signed else vals
    lo, hi = min(xs), max(xs)
    return (n, (hi - lo).bit_length(), lo & M64)


def cascaded_layers(vals: list[int], ts: int, R: int, D: int) -> tuple[list[int], list[int], list[list[int]], list[int]]:
    """Layer i (i < max(R, D)): run-length encode if i < R (values go on, lengths become run list i), then
    delta-encode if i < D (the first value is kept in first[i], the element count entering the layer in cnt_in[i];
    deltas wrap modulo 2^(8*ts)).  Returns (first, cnt_in, run lengths per layer, the values left at the end)."""
    mask = (1 << (8 * ts)) - 1
    cur = list(vals)
    runs, first, cnt_in = [], [], []
    for i in range(max(R, D)):
        if i < R:
            vs, ls = [], []
            for v, g in groupby(cur):
                vs.append(v)
                ls.append(sum(1 for _ in g))
            runs.append(ls)
            cur = vs
        if i < D:
            first.append(cur[0] if cur else 0)
            cnt_in.append(len(cur))
            cur = [(b - a) & mask for a, b in zip(cur, cur[1:])]
    return first, cnt_in, runs, cur


def cascaded_partition(vals: list[int], ts: int, type_signed: bool, R: int, D: int, use_bp: bool) -> dict:
    """cascaded_layers(), then every run list is a stream of 16-bit unsigned lengths and the values left at the end
    are the value stream, bit-packed in the type's own signedness when no delta layer ran, signed after one."""
    first, cnt_in, run_lists, cur = cascaded_layers(vals, ts, R, D)
    runs = [_stream_hdr(ls, use_bp, False, 2, 16) for ls in run_lists]
    vals_hdr = _stream_hdr(cur, use_bp, D > 0 or type_signed, ts, 8 * ts)
    size = 8 * D + _r8(4 * D) + sum(16 + 8 * _words(c, b) for c, b, _ in runs + [vals_hdr])
    return {"first": first, "cnt_in": cnt_in, "runs": runs, "vals": vals_hdr, "size": size, "pad": 0}


def cascaded_model(data: bytes, type_id: int, part: int, R: int, D: int, use_bp: int) -> dict:
    ts = TYPE_SIZE[type_id]
    n = len(data)
    tail = n % ts
    whole = n - tail
    num_parts = (whole + part - 1) // part
    ev = elements(data, ts)
    per = part // ts
    off = _r8(20 + 4 * (num_parts + 1))
    offs, parts = [], []
    for p in range(num_parts):
        offs.append(off)
        m = cascaded_partition(ev[p * per:(p + 1) * per], ts, type_id in SIGNED, R, D, bool(use_bp))
        parts.append(m)
        off += m["size"]
    offs.append(off)
    cfg = type_id | (R << 8) | (D << 16) | ((1 if use_bp else 0) << 24)
    return {"header": (CSC_MAGIC, cfg, n, part, num_parts), "part_off": offs, "hdr_pad": 0, "parts": parts,
            "tail": data[whole:] + bytes(8 - tail) if tail else b"", "size": off + (8 if tail else 0)}


def _stream_at(b: bytes, o: int) -> tuple[tuple[int, int, int], int, int]:
    """Header of the stream at byte o, the bits that pad its last word (must be zero), and its size."""
    count, bits, mn = _u32(b, o), _u32(b, o + 4), _u64(b, o + 8)
    nw = _words(count, bits)
    slack = 0
    used = count * bits
    if nw and used % 64:
        slack = _u64(b, o + 16 + 8 * (nw - 1)) >> (used % 64)
    return (count, bits, mn), slack, 16 + 8 * nw


def parse_cascaded(b: bytes) -> dict:
    """Read back every field cascaded_model() predicts.  Pad bytes are returned as their OR (zero when clear)."""
    magic, cfg, n, part, num_parts = (_u32(b, 4 * i) for i in range(5))
    type_id, R, D = cfg & 0xFF, (cfg >> 8) & 0xFF, (cfg >> 16) & 0xFF
    offs = [_u32(b, 20 + 4 * i) for i in range(num_parts + 1)]
    hdr_end = 20 + 4 * (num_parts + 1)
    parts = []
    for p in range(num_parts):
        o = offs[p]
        first = [_u64(b, o + 8 * i) for i in range(D)]
        cnt_in = [_u32(b, o + 8 * D + 4 * i) for i in range(D)]
        pad = int.from_bytes(b[o + 12 * D:o + 8 * D + _r8(4 * D)], "little")
        q = o + 8 * D + _r8(4 * D)
        runs = []
        for _ in range(R):
            h, slack, sz = _stream_at(b, q)
            runs.append(h)
            pad |= slack
            q += sz
        vals, slack, sz = _stream_at(b, q)
        pad |= slack
        q += sz
        parts.append({"first": first, "cnt_in": cnt_in, "runs": runs, "vals": vals, "size": q - o, "pad": pad})
    ts = TYPE_SIZE.get(type_id, 1)
    tail = n % ts
    return {"header": (magic, cfg, n, part, num_parts), "part_off": offs,
            "hdr_pad": int.from_bytes(b[hdr_end:offs[0]], "little") if num_parts else 0, "parts": parts,
            "tail": b[offs[-1]:offs[-1] + 8] if tail else b"", "size": offs[-1] + (8 if tail else 0)}


# ------------------------------------------------------------------------------------------------- Bitcomp
def _zigzag(d: int, ts: int) -> int:
    s = _signed(d, ts)
    return 2 * s if s >= 0 else -2 * s - 1


def bitcomp_block_bytes(algo: int, desc: int) -> int:
    if algo == 0:
        return 8 + 16 * desc
    nz, bits = desc & 0xFF, desc >> 8
    return 16 + 8 * _words(nz, bits)


def bitcomp_model(data: bytes, algo: int, type_id: int) -> dict:
    """Per 128-element block: algo 0 -- the width of the largest zig-zag delta to the previous element (slot 0 and
    the slots past a ragged end count as 0); algo 1 -- the non-zero count | the width of the largest value << 8."""
    ts = TYPE_SIZE[type_id]
    n = len(data)
    ev = elements(data, ts)
    mask = (1 << (8 * ts)) - 1
    descs = []
    for e0 in range(0, len(ev), 128):
        blk = ev[e0:e0 + 128]
        if algo == 0:
            m = max([_zigzag((b - a) & mask, ts) for a, b in zip(blk, blk[1:])], default=0)
            descs.append(m.bit_length())
        else:
            nz = sum(1 for v in blk if v)
            descs.append(nz | (max(blk).bit_length() << 8))
    size = _r8(16 + 2 * len(descs)) + sum(bitcomp_block_bytes(algo, d) for d in descs)
    tail = n % ts
    return {"header": (BTC_MAGIC, algo | (type_id << 8), n, len(descs)), "descs": descs, "desc_pad": 0,
            "tail": data[n - tail:] + bytes(8 - tail) if tail else b"", "size": size + (8 if tail else 0)}


def parse_bitcomp(b: bytes) -> dict:
    magic, cfg, n, nblocks = (_u32(b, 4 * i) for i in range(4))
    algo, type_id = cfg & 0xFF, (cfg >> 8) & 0xFF
    descs = [int.from_bytes(b[16 + 2 * i:18 + 2 * i], "little") for i in range(nblocks)]
    off = _r8(16 + 2 * nblocks)
    size = off + sum(bitcomp_block_bytes(algo, d) for d in descs)
    tail = n % TYPE_SIZE.get(type_id, 1)
    return {"header": (magic, cfg, n, nblocks), "descs": descs,
            "desc_pad": int.from_bytes(b[16 + 2 * nblocks:off], "little"),
            "tail": b[size:size + 8] if tail else b"", "size": size + (8 if tail else 0)}


# ----------------------------------------------------------------------------------------------------- ANS
def ans_freq(data: bytes) -> tuple[int, list[int]]:
    """(symbols present, normalised frequencies).  f = max(1, count * 4096 // n); a shortfall goes to the most frequent
    symbol (lowest on a tie); an excess is taken from the currently largest frequency (lowest symbol on a tie), never
    below 1."""
    n = len(data)
    hist = Counter(data)
    freq = [0] * 256
    for s, c in hist.items():
        freq[s] = max(1, c * ANS_M // n)
    total = sum(freq)
    if len(hist) > 1:
        if total < ANS_M:
            best = min(hist, key=lambda s: (-hist[s], s))
            freq[best] += ANS_M - total
        while total > ANS_M:
            bf = max(freq)
            bi = freq.index(bf)
            dec = min(total - ANS_M, bf - 1)
            freq[bi] -= dec
            total -= dec
    return len(hist), freq


def ans_encode_segment(seg: bytes, freq: list[int], start: list[int] | None = None) -> tuple[list[int], list[int]]:
    """(32 initial decoder states, 16-bit renormalisation words in the order the decoder reads them) of one segment:
    32 interleaved rANS states (symbol i -> state i % 32), each starting at `start` (default L = 2^16, the state the
    decoder must end in), encoded from the last symbol back; a state emits a word before coding a symbol of frequency
    f when it is >= f << 20."""
    cum = [0] * 256
    acc = 0
    for s in range(256):
        cum[s] = acc
        acc += freq[s]
    x = list(start) if start else [ANS_L] * 32
    words = []
    for i in range(len(seg) - 1, -1, -1):
        s = seg[i]
        f = freq[s]
        v = x[i & 31]
        if v >= f << 20:
            words.append(v & 0xFFFF)
            v >>= 16
        x[i & 31] = ((v // f) << 12) + v % f + cum[s]
    return x, words[::-1]


def ans_segment_words(seg: bytes, freq: list[int]) -> int:
    """Renormalisation words of one segment (ans_encode_segment)."""
    return len(ans_encode_segment(seg, freq)[1])


def ans_model(data: bytes) -> dict:
    """Mode 2 (constant) for one distinct symbol, 1 (stored) for an empty chunk or when the rANS layout is not smaller
    than 16 + n bytes, else 0 with the freq table, nseg and the segment offsets (each segment: 32 states + its words,
    padded to 4 bytes)."""
    n = len(data)
    present, freq = ans_freq(data) if n else (0, [0] * 256)
    if n == 0:
        return {"header": (ANS_MAGIC, 0, 1, 0), "size": 16}
    if present == 1:
        return {"header": (ANS_MAGIC, n, 2, 0), "symbol": data[0], "size": 17}
    nseg = (n + ANS_SEG - 1) // ANS_SEG
    off = (16 + 512 + 4 * (nseg + 1) + 3) & ~3
    offs = []
    for sg in range(nseg):
        offs.append(off)
        nw = ans_segment_words(data[sg * ANS_SEG:(sg + 1) * ANS_SEG], freq)
        off += 128 + ((2 * nw + 3) & ~3)
    offs.append(off)
    if off >= 16 + n:
        return {"header": (ANS_MAGIC, n, 1, 0), "size": 16 + n}
    return {"header": (ANS_MAGIC, n, 0, nseg), "freq": freq, "seg_off": offs, "size": off}


def parse_ans(b: bytes) -> dict:
    magic, n, mode, nseg = (_u32(b, 4 * i) for i in range(4))
    if mode == 2:
        return {"header": (magic, n, mode, nseg), "symbol": b[16], "size": 17}
    if mode == 1:
        return {"header": (magic, n, mode, nseg), "size": 16 + n}
    freq = [int.from_bytes(b[16 + 2 * s:18 + 2 * s], "little") for s in range(256)]
    offs = [_u32(b, 528 + 4 * i) for i in range(nseg + 1)]
    return {"header": (magic, n, mode, nseg), "freq": freq, "seg_off": offs, "size": offs[-1]}


# ------------------------------------------------------------------------------------------------ edge inputs
def _pack(vals, ts: int) -> bytes:
    return np.asarray([int(v) & ((1 << (8 * ts)) - 1) for v in vals], dtype=np.uint64).astype(
        {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[ts]).tobytes()


def _walk(rng, n: int) -> list[int]:
    """Runs of 1..9 equal values, small steps between runs: every layer has something to do."""
    steps = rng.integers(-3, 4, n + 1)
    steps[0] = rng.integers(0, 1 << 16)
    return np.repeat(np.cumsum(steps), rng.integers(1, 10, n + 1))[:n].tolist()


def edge_chunks(type_id: int, part: int = 4096, seed: int = 0):
    """(name, bytes) pairs at the edges of the typed codecs for one element type and Cascaded partition size."""
    ts = TYPE_SIZE[type_id]
    w = 8 * ts
    signed = type_id in SIGNED
    umax = (1 << w) - 1
    tmin, tmax = ((-(1 << (w - 1)), (1 << (w - 1)) - 1) if signed else (0, umax))
    cap = part // ts                            # elements per partition
    n = 3 * cap - 5                             # three partitions (an odd count), the last one not full
    rng = np.random.default_rng(seed * 1000 + type_id * 10 + part % 997)

    def rand(k, lo=0, hi=umax):
        return [int(x) for x in rng.integers(lo, hi, k, dtype=np.uint64, endpoint=True)] if hi > lo else [lo] * k

    out = []
    for nb in sorted({0, 1, ts - 1, ts}):
        out.append((f"len{nb}", bytes(rng.integers(0, 256, nb, dtype=np.uint8))))
    out.append(("const_min", _pack([tmin] * n, ts)))
    out.append(("const_max", _pack([tmax] * n, ts)))
    out.append(("min_max_alternating", _pack([tmin, tmax] * (n // 2), ts)))
    start = int(rng.integers(0, 1 << min(w, 32)))
    out.append(("ramp", _pack(range(start, start + n), ts)))
    out.append(("ramp_wraps_umax", _pack(range(umax - n // 2, umax - n // 2 + n), ts)))
    if signed:
        out.append(("ramp_crosses_zero", _pack(range(-(n // 2), n - n // 2), ts)))
    cyc, vals, k = [1, 2, 7, 8, 9, 31, 32, 33, 127, 128, 129, 4095], [], 0
    while len(vals) < n:
        vals += [rand(1)[0]] * cyc[k % len(cyc)]
        k += 1
    out.append(("run_lengths_cycling", _pack(vals[:n], ts)))
    for runs in (127, 128, 129, 256):
        r = min(runs, cap)
        vals = []
        for p in range(3):
            lens = [cap // r + (1 if i < cap % r else 0) for i in range(r)]
            vals += [(i + p) % 2 * umax // 3 + i for i, ln in enumerate(lens) for _ in range(ln)]
        out.append((f"runs_per_partition_{runs}", _pack(vals, ts)))
    for e in (8, 32):
        for rg in ((1 << e) - 1, 1 << e):
            if rg > umax:
                continue
            lo = -(rg // 2) - 1 if signed else int(rng.integers(0, umax - rg + 1, dtype=np.uint64))
            vals = [lo, lo + rg] + [lo + int(x) for x in rng.integers(0, rg, n - 2, dtype=np.uint64, endpoint=True)]
            out.append((f"range_{rg:#x}", _pack(vals, ts)))
    out.append(("random_full_width", _pack(rand(n), ts)))
    for r in range(1, 8):
        out.append((f"last_partition_{r}", _pack(_walk(rng, cap + r), ts)))
    for np_ in (25, 26, 27, 28):
        out.append((f"partitions_{np_}", _pack(_walk(rng, (np_ - 1) * cap + cap // 2), ts)))
    out.append(("one_partition", _pack(_walk(rng, cap), ts)))
    if ts > 1:
        out.append(("ragged_tail", _pack(_walk(rng, cap + 3), ts) + b"\x5a" * (ts - 1)))
    return out


def bitcomp_edge_chunks(type_id: int, seed: int = 0):
    """edge_chunks() plus blocks that sit on Bitcomp's descriptor edges."""
    ts = TYPE_SIZE[type_id]
    w = 8 * ts
    rng = np.random.default_rng(seed * 1000 + 500 + type_id)
    out = edge_chunks(type_id, seed=seed)
    out.append(("zero_blocks", bytes(ts * 128 * 5)))
    for pos in (0, 63, 64, 127):
        blk = [0] * 128
        blk[pos] = int(rng.integers(1, 1 << min(w, 63)))
        out.append((f"one_nonzero_at_{pos}", _pack(blk * 2 + [0] * 128, ts)))
    out.append(("dense_blocks", _pack([int(x) for x in rng.integers(1, (1 << w) - 1, 128 * 4, dtype=np.uint64,
                                                                     endpoint=True)], ts)))
    for rag in (1, 3, 4, 5, 127):
        out.append((f"ragged_last_block_{rag}", _pack(_walk(rng, 256 + rag), ts)))
    vals, acc = [], int(rng.integers(0, 1 << min(w, 62)))
    for k in range(w + 1):                      # block k: deltas spread over [-2^k / 2, 2^k / 2], zig-zag width k
        h = (1 << k) >> 1
        ds = [int(x) - h for x in rng.integers(0, (1 << k) - 1, 128, dtype=np.uint64, endpoint=True)]
        ds[1] = -h
        for d in ds:
            acc += d
            vals.append(acc)
    out.append(("delta_width_every_k", _pack(vals, ts)))
    return out


def ans_edge_chunks(seed: int = 0, big: bool = True):
    """edge_chunks() of bytes plus inputs that drive the ANS frequency normalisation, the stored-mode decision and the
    segment count."""
    rng = np.random.default_rng(seed * 1000 + 900)
    out = edge_chunks(1, seed=seed)
    rare = bytearray(65536)
    rare[int(rng.integers(0, 65536))] = 1
    out.append(("two_symbols_one_rare", bytes(rare)))                      # 4096 + 1 > 4096: the reduction loop
    out.append(("all_256_symbols", bytes(range(256)) * 40 + bytes(rng.geometric(0.05, 30000).clip(0, 255)
                                                                   .astype(np.uint8))))
    # near the stored-vs-rANS break-even: uniform bytes over 2^k symbols with k close to 8
    for k in (7, 8):
        for n in (700, 3000, 20000):
            out.append((f"uniform_{1 << k}_n{n}", rng.integers(0, 1 << k, n, dtype=np.uint8).tobytes()))
    for n in (600, 1000, 2000):
        out.append((f"skewed_n{n}", np.minimum(rng.geometric(0.02, n), 255).astype(np.uint8).tobytes()))
    for k in (1, 2, 4):
        for d in (-1, 1):
            out.append((f"seg_{k}x16384{d:+d}",
                        np.minimum(rng.geometric(0.2, 16384 * k + d) - 1, 255).astype(np.uint8).tobytes()))
    if big:                                     # nseg = 1024, every entry of the encoder's segment table
        out.append(("16MB", np.minimum(rng.geometric(0.3, 1 << 24) - 1, 255).astype(np.uint8).tobytes()))
    return out
