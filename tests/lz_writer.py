"""Hand-built LZ4 block and Snappy raw streams (test infrastructure).

Encoders only write the shapes they like: liblz4, pyarrow, the oracle and this library's compressor never emit a Snappy
copy-2 of length 1-3, a copy-4 element, a non-canonical literal tag or an over-long varint, nor an LZ4 block whose
last sequence has no literals or whose length extensions sit on a staging boundary.  The decoders parse exactly these
fields, so the writers here take explicit tokens / elements and can spell anything the formats allow (or, for the
invalid list, anything they forbid).  Every writer also returns the output the stream stands for, computed the
byte-serial way (an overlapping match repeats its period), or None when the stream is invalid.

VALID / INVALID: name -> Case.  Every valid case must decode to `out` at capacity `cap` (and any capacity above); every
invalid case must be rejected at capacity `cap`.  `corruption_corpus()` draws seeded corrupted streams from real
producers' output."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class Case:
    codec: str          # "lz4" | "snappy"
    comp: bytes
    out: bytes | None   # expected output (None: invalid)
    cap: int            # capacity the case is stated for


def _copy(out: bytearray, off: int, n: int) -> bool:
    """Append n bytes copied from `off` back, byte-serially (period repeats).  False when the offset is invalid."""
    if off == 0 or off > len(out):
        return False
    if off >= n:
        out += out[len(out) - off:len(out) - off + n]
    else:
        pat = bytes(out[len(out) - off:])
        out += (pat * (n // off + 1))[:n]
    return True


def _ext(n: int) -> bytes:
    """LZ4 length extension: 255-bytes then the remainder (n = length - 15)."""
    return b"\xff" * (n // 255) + bytes([n % 255])


class Lz4:
    """LZ4 block writer.  seq() appends one sequence (literals + match), end() the final literal-only sequence."""

    def __init__(self):
        self.blk = bytearray()
        self.out = bytearray()
        self.ok = True

    def seq(self, lits: bytes, off: int, ml: int, raw_tok: int | None = None) -> "Lz4":
        ll, mc = len(lits), ml - 4
        assert mc >= 0
        self.blk.append(raw_tok if raw_tok is not None else (min(ll, 15) << 4) | min(mc, 15))
        if ll >= 15:
            self.blk += _ext(ll - 15)
        self.blk += lits
        self.blk += bytes([off & 255, (off >> 8) & 255])
        if mc >= 15:
            self.blk += _ext(mc - 15)
        self.out += lits
        self.ok = self.ok and _copy(self.out, off, ml)
        return self

    def end(self, lits: bytes = b"") -> "Lz4":
        ll = len(lits)
        self.blk.append(min(ll, 15) << 4)
        if ll >= 15:
            self.blk += _ext(ll - 15)
        self.blk += lits
        self.out += lits
        return self

    def case(self, cap: int | None = None) -> Case:
        out = bytes(self.out) if self.ok else None
        return Case("lz4", bytes(self.blk), out, len(self.out) if cap is None else cap)


def varint(v: int, extra: int = 0) -> bytes:
    """Snappy preamble: little-endian base-128 varint, padded with `extra` over-long continuation bytes."""
    b = bytearray()
    while True:
        b.append(v & 0x7F)
        v >>= 7
        if not v:
            break
    for _ in range(extra):
        b.append(0)
    for i in range(len(b) - 1):
        b[i] |= 0x80
    return bytes(b)


class Snappy:
    """Snappy raw writer.  The preamble is written last (case()) from the produced length unless overridden."""

    def __init__(self):
        self.body = bytearray()
        self.out = bytearray()
        self.ok = True

    def lit(self, data: bytes, nb: int | None = None) -> "Snappy":
        """Literal element; nb = 1..4 forces tag 59 + nb with that many length bytes (canonical: only above 60)."""
        n1 = len(data) - 1
        assert n1 >= 0
        if nb is None:
            nb = 0 if n1 < 60 else 1 if n1 < 1 << 8 else 2 if n1 < 1 << 16 else 3 if n1 < 1 << 24 else 4
        if nb == 0:
            self.body.append(n1 << 2)
        else:
            self.body.append((59 + nb) << 2)
            self.body += n1.to_bytes(nb, "little")
        self.body += data
        self.out += data
        return self

    def copy1(self, off: int, n: int) -> "Snappy":
        assert 4 <= n <= 11 and off < 2048
        self.body += bytes([1 | (n - 4) << 2 | (off >> 8) << 5, off & 255])
        self.ok = self.ok and _copy(self.out, off, n)
        return self

    def copy2(self, off: int, n: int) -> "Snappy":
        assert 1 <= n <= 64 and off < 65536
        self.body += bytes([2 | (n - 1) << 2, off & 255, off >> 8])
        self.ok = self.ok and _copy(self.out, off, n)
        return self

    def copy4(self, off: int, n: int) -> "Snappy":
        assert 1 <= n <= 64
        self.body += bytes([3 | (n - 1) << 2]) + off.to_bytes(4, "little")
        self.ok = self.ok and _copy(self.out, off, n)
        return self

    def case(self, ulen: int | None = None, extra: int = 0, cap: int | None = None) -> Case:
        n = len(self.out) if ulen is None else ulen
        out = bytes(self.out) if self.ok and n == len(self.out) else None
        return Case("snappy", varint(n, extra) + bytes(self.body), out, len(self.out) if cap is None else cap)


def _rand(rng, n, alphabet=256):
    return rng.integers(0, alphabet, n, dtype=np.uint8).tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# valid streams
# ---------------------------------------------------------------------------------------------------------------------
def _dense_prefix(w: Lz4, rng, upto: int):
    """Short dense sequences (2 literals + 4..8-byte match) until the block is 9..14 bytes short of `upto`."""
    while len(w.blk) + 14 < upto:
        w.seq(_rand(rng, 2), int(rng.integers(1, len(w.out) + 3)) if w.out else 2, int(rng.integers(4, 9)))


def lz4_valid(rng) -> dict[str, Case]:
    v: dict[str, Case] = {}
    base = _rand(rng, 64)
    for ll in (0, 14, 15, 270, 255 * 40 + 15, 255 * 40 + 16):
        w = Lz4().seq(base[:8], 8, 8).seq(_rand(rng, ll), 3, 12).end(_rand(rng, 9))
        v[f"lz4_lit_{ll}"] = w.case()
    for ll in (0, 14, 15, 270, 5000):
        v[f"lz4_end_lit_{ll}"] = Lz4().seq(base[:16], 16, 20).end(_rand(rng, ll)).case()
    for ml in (4, 18, 19, 274, 60000):
        v[f"lz4_match_{ml}"] = Lz4().seq(base[:20], 7, ml).end(b"tail").case()
    for off in list(range(1, 18)) + [31, 32, 33, 4095, 4096, 4097, 65535]:
        w = Lz4().seq(_rand(rng, 15), 15, 40)
        w.seq(_rand(rng, max(0, off - len(w.out) + 1) + 3, 16), off, 37).seq(base[:5], off, 100).end(b"end..")
        v[f"lz4_off_{off}"] = w.case()
    for n in (1, 2, 9, 17, 100):                                               # offset == op: the very first byte
        v[f"lz4_off_eq_op_{n}"] = Lz4().seq(_rand(rng, n), n, 30).seq(b"x", n + 31, 8).end(b"zz").case()
    v["lz4_final_zero_literals"] = Lz4().seq(base[:12], 5, 50).end(b"").case()
    v["lz4_only_empty_final"] = Case("lz4", b"\x00", b"", 0)
    for ln in (192, 193):
        v[f"lz4_serial_lit_{ln}"] = Lz4().seq(base[:4], 4, 8).seq(_rand(rng, ln), 9, 20).end(_rand(rng, 5)).case()
        v[f"lz4_serial_match_{ln}"] = Lz4().seq(_rand(rng, 40), 33, ln).seq(b"a", 100, ln).end(b"q").case()
    # extension bytes and literals straddling 32 * k and 1024 * k of the stream (segment and staged-block edges)
    for edge in (32, 64, 1024, 2048):
        for d in range(-4, 4):
            w = Lz4()
            _dense_prefix(w, rng, edge)
            pad = edge + d - len(w.blk) - 3                                      # token of the long sequence at edge + d
            w.seq(_rand(rng, pad), 3, 4)
            assert len(w.blk) == edge + d
            w.seq(_rand(rng, 15 + 255 + 3), 6, 19 + 255 + 40)                   # literal and match extensions
            w.seq(_rand(rng, 3), 2, 19)                                          # match extension byte 0
            for _ in range(40):                                                  # one-byte extensions the block path
                ll = int(rng.integers(0, 10))                                    # takes (ext < 14 - L) or stops at
                w.seq(_rand(rng, ll), int(rng.integers(1, 40)), 19 + int(rng.integers(0, 16 - ll)))
            _dense_prefix(w, rng, len(w.blk) + 200)
            v[f"lz4_edge_{edge}{d:+d}"] = w.end(_rand(rng, 7)).case()
    # 16 000 tokens, each copying what its predecessor produced (longest dependency chains for the block path)
    w, prev = Lz4(), 0
    w.seq(_rand(rng, 8), 8, 8)
    prev = 16
    for i in range(16000):
        ll, ml = int(rng.integers(0, 3)), int(rng.integers(4, 12))
        w.seq(_rand(rng, ll), prev + ll, ml)
        prev = ll + ml
    v["lz4_chain_16000"] = w.end(_rand(rng, 6)).case()
    # 1 MB and 16 MB chunks with matches that reach far behind the 4 KB ring
    for mb, nseq in ((1, 900), (16, 2200)):
        w = Lz4().seq(_rand(rng, 65535), 1, 4)
        while len(w.out) < (mb << 20) - 70000:
            off = int(rng.integers(40000, 65536))
            ml = int(rng.integers(4, (mb << 20) // nseq))
            w.seq(_rand(rng, int(rng.integers(0, 20))), off, ml)
        v[f"lz4_far_{mb}mb"] = w.end(_rand(rng, 10)).case()
    # a dense chunk (tabular-like) for the straight block path, then the same with one far match every 2 KB
    w = Lz4().seq(_rand(rng, 16), 16, 4)
    while len(w.out) < 65000:
        far = len(w.out) > 8000 and rng.random() < 0.01
        w.seq(_rand(rng, int(rng.integers(0, 5))), int(rng.integers(5000, len(w.out))) if far else
              int(rng.integers(1, min(64, len(w.out) + 1))), int(rng.integers(4, 14)))
    v["lz4_dense_far"] = w.end(_rand(rng, 5)).case()
    return v


def snappy_valid(rng) -> dict[str, Case]:
    v: dict[str, Case] = {}
    base = _rand(rng, 64)
    # preambles of 1..5 bytes, canonical (up to 4 bytes: the 5-byte form needs >= 256 MB) and over-long
    for n in (0, 1, 127, 128, 16383, 16384, 70000):
        s = Snappy()
        if n:
            s.lit(base[:8])
            while len(s.out) < n:
                s.copy2(8, min(64, n - len(s.out)))
        for extra in range(0, 5 - len(varint(n)) + 1):
            v[f"snappy_varint_{n}_x{extra}"] = s.case(extra=extra)
    s = Snappy().lit(base[:16])
    while len(s.out) < (1 << 21) + 5:
        s.copy2(16, min(64, (1 << 21) + 5 - len(s.out)))
    v["snappy_varint_4byte"] = s.case()
    # literal tags 60..63, canonical and not (small lengths spelled with 1..4 length bytes)
    for nb in (1, 2, 3, 4):
        for ln in (1, 5, 60, 61, 256) if nb == 1 else (1, 5, 60, 61, 300):
            v[f"snappy_littag_{59 + nb}_{ln}"] = Snappy().lit(_rand(rng, ln), nb).copy1(1, 4).lit(b"e").case()
    v["snappy_lit_70000"] = Snappy().lit(_rand(rng, 70000)).case()
    # copy-1: all 8 lengths, offsets up to 2047
    s = Snappy().lit(_rand(rng, 60)).lit(_rand(rng, 2048))
    for off in (1, 2, 3, 7, 8, 31, 255, 256, 1024, 2047):
        for n in range(4, 12):
            s.copy1(off, n)
    v["snappy_copy1_all"] = s.case()
    # copy-2: lengths 1..64 (1..3 are never emitted by encoders), near and far offsets
    for off in (1, 3, 8, 33, 4097, 65535):
        s = Snappy().lit(_rand(rng, min(off, 60))).lit(_rand(rng, max(off - 60, 0) + 5)) if off > 60 else \
            Snappy().lit(_rand(rng, 60))
        for n in range(1, 65):
            s.copy2(off, n)
        v[f"snappy_copy2_off{off}"] = s.case()
    # copy-4, offsets below and above 65 536, in chunks over 64 KB
    s = Snappy().lit(_rand(rng, 65536 + 300))
    for off in (1, 5, 64, 65535, 65536, 65537, 65536 + 299):
        for n in (1, 2, 3, 4, 17, 64):
            s.copy4(off, n)
    v["snappy_copy4"] = s.case()
    s = Snappy().lit(_rand(rng, 40))
    for i in range(3000):
        s.copy4(int(rng.integers(1, len(s.out) + 1)), int(rng.integers(1, 65)))
    v["snappy_copy4_many"] = s.case()
    # runs of copy-2 continuations with one offset, broken at every position of a 32-byte window (the direct loop's
    # window holds the literal element and ten continuations) and of the merge the serial path does (32 elements)
    for per in (1, 2, 4, 8, 3):
        for k in range(0, 36):
            s = Snappy().lit(base[:per])
            for _ in range(k):
                s.copy2(per, 64)
            brk = k % 4
            if brk == 0:
                s.copy2(per, int(rng.integers(1, 64)))
            elif brk == 1:
                s.copy2(per + 1 if per < 8 else per * 2, 64)
            elif brk == 2:
                s.copy1(per, 7)
            else:
                s.lit(b"!")
            s.copy2(per, 64).copy2(per, 64)
            v[f"snappy_run_p{per}_k{k}"] = s.case()
    # every literal length 1..8 in front of its copies (the direct loop's window path)
    for ll in range(1, 9):
        s = Snappy()
        for j in range(40):
            s.lit(_rand(rng, ll)).copy2(ll if ll in (1, 2, 4, 8) else ll, int(rng.integers(1, 65)))
            s.copy2(ll, 64).copy1(ll, 4 + j % 8)
        v[f"snappy_window_ll{ll}"] = s.case()
    # dense chunk (short elements) for the block path, with far copies
    s = Snappy().lit(_rand(rng, 32))
    while len(s.out) < 65000:
        r = rng.random()
        if r < 0.4:
            s.lit(_rand(rng, int(rng.integers(1, 6))))
        elif r < 0.7:
            s.copy1(int(rng.integers(1, min(2048, len(s.out) + 1))), int(rng.integers(4, 12)))
        elif r < 0.98:
            s.copy2(int(rng.integers(1, len(s.out) + 1)), int(rng.integers(1, 33)))
        else:
            s.copy4(int(rng.integers(1, len(s.out) + 1)), int(rng.integers(1, 65)))
    v["snappy_dense_mixed"] = s.case()
    return v


def valid_streams(seed: int = 1) -> dict[str, Case]:
    rng = np.random.default_rng(seed)
    v = lz4_valid(rng)
    v.update(snappy_valid(rng))
    for name, c in v.items():
        assert c.out is not None, name
    return v


# ---------------------------------------------------------------------------------------------------------------------
# invalid streams: one per rejection rule (each must be rejected at `cap`)
# ---------------------------------------------------------------------------------------------------------------------
def invalid_streams(seed: int = 2) -> dict[str, Case]:
    rng = np.random.default_rng(seed)
    bad: dict[str, Case] = {}
    lit = _rand(rng, 20)
    # --- LZ4
    good = Lz4().seq(lit, 4, 300).seq(_rand(rng, 300), 10, 30).end(_rand(rng, 6))
    g = good.case()
    n = len(g.out)
    bad["lz4_off0"] = Lz4().seq(lit, 0, 8).end(b"x").case()
    bad["lz4_off_op_plus_1"] = Lz4().seq(lit, 21, 8).end(b"x").case()
    bad["lz4_off_op_plus_1_later"] = Lz4().seq(lit, 4, 8).seq(b"ab", 31, 4).end(b"x").case()
    # the same with 32 more bytes behind the sequence: the direct loop parses it from its register window
    tail = _rand(rng, 40)
    bad["lz4_off_op_plus_1_window"] = Lz4().seq(lit[:4], 5, 8).end(tail).case(65536)
    bad["lz4_off_op_plus_1_window_later"] = Lz4().seq(lit[:8], 8, 8).seq(lit[:3], 20, 8).end(tail).case(65536)
    bad["lz4_off0_window"] = Lz4().seq(lit[:8], 8, 8).seq(lit[:3], 0, 8).end(tail).case(65536)
    # truncations inside each field.  The first sequence is: token, 1 literal-extension byte, 20 literals, 2 offset
    # bytes, 2 match-extension bytes (255, 26)
    t = g.comp
    bad["lz4_trunc_token_only"] = Case("lz4", t[:1], None, n)
    bad["lz4_trunc_in_literals"] = Case("lz4", t[:1 + 1 + 10], None, n)
    bad["lz4_trunc_in_offset"] = Case("lz4", t[:1 + 1 + 20 + 1], None, n)
    bad["lz4_trunc_in_match_ext"] = Case("lz4", t[:1 + 1 + 20 + 2 + 1], None, n)
    w = Lz4().seq(_rand(rng, 300), 5, 8)
    bad["lz4_trunc_in_lit_ext"] = Case("lz4", bytes(w.blk[:2]), None, 400)
    bad["lz4_trunc_final_literals"] = Case("lz4", g.comp[:-1], None, n)
    bad["lz4_ext_runs_off_end"] = Case("lz4", b"\xf0" + b"\xff" * 40, None, 65536)
    bad["lz4_match_ext_runs_off_end"] = Case("lz4", b"\x1f" + b"A" + b"\x01\x00" + b"\xff" * 40, None, 65536)
    bad["lz4_no_final_sequence"] = Case("lz4", bytes(Lz4().seq(lit, 4, 8).blk), None, 65536)
    c = Lz4().seq(lit, 4, 300).end(_rand(rng, 9)).case()
    bad["lz4_over_cap_by_1_literal"] = Case("lz4", c.comp, None, len(c.out) - 1)
    c = Lz4().seq(lit, 4, 300).end(b"").case()
    bad["lz4_over_cap_by_1_match"] = Case("lz4", c.comp, None, len(c.out) - 1)
    c = Lz4().seq(lit, 20, 60000).end(b"").case()
    bad["lz4_over_cap_by_1_long_match"] = Case("lz4", c.comp, None, len(c.out) - 1)
    # --- Snappy
    s = Snappy().lit(lit).copy2(4, 64).copy1(3, 9).copy4(20, 30).lit(_rand(rng, 100))
    sc = s.case()
    n = len(sc.out)
    body = bytes(s.body)
    bad["snappy_off0_copy1"] = Snappy().lit(lit).copy1(0, 4).case()
    bad["snappy_off0_copy2"] = Snappy().lit(lit).copy2(0, 4).case()
    bad["snappy_off0_copy4"] = Snappy().lit(lit).copy4(0, 4).case()
    bad["snappy_off_op_plus_1_copy1"] = Snappy().lit(lit).copy1(21, 4).case()
    bad["snappy_off_op_plus_1_copy2"] = Snappy().lit(lit).copy2(21, 4).case()
    bad["snappy_off_op_plus_1_copy4"] = Snappy().lit(lit).copy4(21, 4).case()
    bad["snappy_off_op_plus_1_first"] = Snappy().copy2(1, 4).case()
    bad["snappy_trunc_varint"] = Case("snappy", varint(n)[:-1], None, n)
    bad["snappy_varint_6_bytes"] = Case("snappy", varint(5, extra=5) + b"\x10abcde", None, 65536)
    bad["snappy_varint_over_32bit"] = Case("snappy", b"\xff\xff\xff\xff\x1f", None, 65536)
    vi = len(varint(n))
    bad["snappy_trunc_in_literal"] = Case("snappy", sc.comp[:vi + 1 + 10], None, n)
    bad["snappy_trunc_in_copy2"] = Case("snappy", sc.comp[:vi + 21 + 2], None, n)
    bad["snappy_trunc_in_copy1"] = Case("snappy", sc.comp[:vi + 21 + 3 + 1], None, n)
    bad["snappy_trunc_in_copy4"] = Case("snappy", sc.comp[:vi + 21 + 3 + 2 + 3], None, n)
    bad["snappy_trunc_in_lit_len"] = Case("snappy", varint(300) + bytes([61 << 2, 0x2B]), None, 300)
    bad["snappy_trunc_last_literal"] = Case("snappy", sc.comp[:-1], None, n)
    bad["snappy_lit_len_ffffffff"] = Case("snappy", varint(10) + bytes([63 << 2]) + b"\xff" * 4 + b"x" * 10, None, 10)
    bad["snappy_preamble_larger"] = Case("snappy", varint(n + 1) + body, None, n + 1)
    bad["snappy_preamble_smaller_literal"] = Case("snappy", varint(n - 1) + body, None, n)
    t2 = Snappy().lit(lit).copy2(4, 64)
    bad["snappy_preamble_smaller_match"] = Case("snappy", varint(len(t2.out) - 1) + bytes(t2.body), None, 1000)
    bad["snappy_over_cap_by_1_literal"] = Case("snappy", sc.comp, None, n - 1)
    bad["snappy_over_cap_by_1_match"] = Case("snappy", t2.case().comp, None, len(t2.out) - 1)
    bad["snappy_empty"] = Case("snappy", b"", None, 64)
    for name, c in bad.items():
        assert c.out is None, name
    return bad


# ---------------------------------------------------------------------------------------------------------------------
# corruption corpus
# ---------------------------------------------------------------------------------------------------------------------
def mutate(rng, codec: str, comp: bytes) -> tuple[str, bytes]:
    """One seeded corruption of a valid stream: bit flips, a truncation, appended bytes, a single-byte insert or delete,
    or (Snappy) a rewritten preamble."""
    kinds = ["flip", "trunc", "append", "insert", "delete"] + (["preamble"] if codec == "snappy" else [])
    kind = kinds[int(rng.integers(0, len(kinds)))]
    b = bytearray(comp)
    if kind == "flip" and b:
        for _ in range(int(rng.integers(1, 4))):
            i = int(rng.integers(0, len(b)))
            b[i] ^= 1 << int(rng.integers(0, 8))
    elif kind == "trunc" and b:
        b = b[:int(rng.integers(0, len(b)))]
    elif kind == "append":
        b += _rand(rng, int(rng.integers(1, 9)))
    elif kind == "insert":
        b.insert(int(rng.integers(0, len(b) + 1)), int(rng.integers(0, 256)))
    elif kind == "delete" and b:
        del b[int(rng.integers(0, len(b)))]
    elif kind == "preamble":
        ip = 0
        while ip < len(b) and b[ip] & 0x80:
            ip += 1
        old = 0
        for k in range(min(ip + 1, len(b))):
            old |= (b[k] & 0x7F) << (7 * k)
        new = max(0, old + int(rng.choice([-2, -1, 1, 2, 64, -64])))
        b = bytearray(varint(new, int(rng.integers(0, 2)))) + b[ip + 1:]
    return kind, bytes(b)


def corpus_cap(i: int, comp: bytes, n: int) -> int:
    """Capacity of corpus stream i (raw length n): exact, exact - 1, exact + 1, max(n, 4 x compressed) or 64 KB in
    turn -- the last two send a dense stream to the light kernel.  (i // 5 shifts the turn, so that every producer of
    corruption_corpus, which takes them in turn too, meets every capacity.)"""
    return (n, max(n - 1, 0), n + 1, max(n, 4 * len(comp)), 65536)[(i + i // 5) % 5]


def corruption_corpus(producers: dict, inputs: list[bytes], n: int = 4000, seed: int = 7):
    """n seeded corrupted streams: (codec, producer, kind, stream, raw length).  producers maps
    (codec, name) -> compress(bytes) -> bytes; inputs are raw chunks, sliced to seeded lengths."""
    rng = np.random.default_rng(seed)
    keys = sorted(producers)
    out = []
    for i in range(n):
        codec, prod = keys[i % len(keys)]
        raw = inputs[int(rng.integers(0, len(inputs)))]
        if len(raw) > 1:
            a = int(rng.integers(0, len(raw)))
            raw = raw[a:a + int(rng.integers(1, 16384))]
        comp = producers[(codec, prod)](raw)
        kind, bad = mutate(rng, codec, comp)
        out.append((codec, prod, kind, bad, len(raw)))
    return out
