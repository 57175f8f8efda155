"""Test infrastructure: a small RFC 1951 (Deflate) / RFC 1952 (Gzip) bit writer that builds streams zlib never emits --
hand-chosen block types, code lengths, header fields and length / distance codes -- and one invalid stream per
rejection rule of the decoder.  Written from the RFCs; zlib (tests/test_inflate_emu.py) pins every stream it builds.

Body items of a fixed or dynamic block:
    int                       a literal byte
    (length, distance)        a match, coded with the usual length / distance codes
    ("L", code, extra, dist)  a match whose length code (257..285) and extra-bit value are given
    ("lit", sym)              the literal/length code of sym, nothing else
    ("dist", sym, extra)      the distance code of sym and its extra bits
    ("bits", value, n)        n raw bits
"""
from __future__ import annotations

import struct
import zlib

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
CLEN_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32


def length_code(n: int) -> tuple[int, int]:
    """(code, extra value) for a match length 3..258 (258 -> 285)."""
    if n == 258:
        return 285, 0
    i = max(k for k in range(28) if LEN_BASE[k] <= n)
    return 257 + i, n - LEN_BASE[i]


def dist_code(d: int) -> tuple[int, int]:
    i = max(k for k in range(30) if DIST_BASE[k] <= d)
    return i, d - DIST_BASE[i]


def canonical(lens) -> dict:
    """symbol -> (code, length) of the canonical code with these lengths (RFC 1951 3.2.2)."""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = {}
    for s, n in enumerate(lens):
        if n:
            out[s] = (nxt[n], n)
            nxt[n] += 1
    return out


def balanced_lengths(symbols, size: int) -> list:
    """A complete code over `symbols` (lengths b-1 and b); one symbol gets length 1 (the incomplete single code)."""
    syms = sorted(set(symbols))
    lens = [0] * size
    if len(syms) == 1:
        lens[syms[0]] = 1
        return lens
    b = (len(syms) - 1).bit_length()
    short = (1 << b) - len(syms)
    for i, s in enumerate(syms):
        lens[s] = b - 1 if i < short else b
    return lens


class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def bits(self, v: int, n: int):
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, c: int, n: int):          # Huffman codes go most significant bit first
        self.bits(int(format(c, f"0{n}b")[::-1], 2), n)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def getvalue(self) -> bytes:
        return bytes(self.out) + (bytes([self.acc & 255]) if self.n else b"")


class DeflateStream:
    """Blocks are appended in order; `data` is what a decoder must produce (valid streams only)."""

    def __init__(self):
        self.w = BitWriter()
        self.data = bytearray()

    def _apply(self, item):
        if isinstance(item, int):
            self.data.append(item)
        elif isinstance(item, tuple) and isinstance(item[0], int):
            self._copy(*item)
        elif item[0] == "L":
            _, code, extra, d = item
            self._copy(LEN_BASE[code - 257] + extra, d)

    def _copy(self, n, d):
        for _ in range(n):
            self.data.append(self.data[-d] if d <= len(self.data) else 0)

    def stored(self, payload: bytes, final=False, nlen=None):
        self.w.bits(int(final), 1)
        self.w.bits(0, 2)
        self.w.align()
        self.w.bits(len(payload), 16)
        self.w.bits((len(payload) ^ 0xFFFF) if nlen is None else nlen, 16)
        for b in payload:
            self.w.bits(b, 8)
        self.data += payload
        return self

    def _body(self, items, lit, dist, eob=True):
        for it in items:
            if isinstance(it, int):
                self.w.code(*lit[it])
            elif isinstance(it, tuple) and isinstance(it[0], int):
                c, e = length_code(it[0])
                self.w.code(*lit[c])
                self.w.bits(e, LEN_EXTRA[c - 257])
                dc, de = dist_code(it[1])
                self.w.code(*dist[dc])
                self.w.bits(de, DIST_EXTRA[dc])
            elif it[0] == "L":
                _, c, e, d = it
                self.w.code(*lit[c])
                self.w.bits(e, LEN_EXTRA[c - 257])
                dc, de = dist_code(d)
                self.w.code(*dist[dc])
                self.w.bits(de, DIST_EXTRA[dc])
            elif it[0] == "lit":
                self.w.code(*lit[it[1]])
            elif it[0] == "dist":
                self.w.code(*dist[it[1]])
                self.w.bits(it[2], DIST_EXTRA[it[1]] if it[1] < 30 else 0)
            elif it[0] == "bits":
                self.w.bits(it[1], it[2])
            self._apply(it)
        if eob:
            self.w.code(*lit[256])

    def fixed(self, items, final=False, eob=True):
        self.w.bits(int(final), 1)
        self.w.bits(1, 2)
        self._body(items, canonical(FIXED_LIT), canonical(FIXED_DIST), eob)
        return self

    def dynamic(self, items, final=False, lit_lens=None, dist_lens=None, hlit=None, hdist=None, clen_lens=None,
                clen_seq=None, hclen=None, rle=False, eob=True):
        """lit_lens / dist_lens default to a complete code over the symbols `items` use (an empty distance set when
        there are no matches); clen_seq, a list of (code-length symbol, extra value), overrides the coded lengths."""
        if lit_lens is None:
            used = {256}
            for it in items:
                if isinstance(it, int):
                    used.add(it)
                elif isinstance(it, tuple) and isinstance(it[0], int):
                    used.add(length_code(it[0])[0])
                elif it[0] == "L":
                    used.add(it[1])
                elif it[0] == "lit":
                    used.add(it[1])
            lit_lens = balanced_lengths(used, max(257, max(used) + 1))
        if dist_lens is None:
            used = {dist_code(it[1])[0] for it in items if isinstance(it, tuple) and isinstance(it[0], int)}
            used |= {dist_code(it[3])[0] for it in items if isinstance(it, tuple) and it[0] == "L"}
            dist_lens = balanced_lengths(used, max(used) + 1) if used else [0]
        hlit = len(lit_lens) if hlit is None else hlit
        hdist = len(dist_lens) if hdist is None else hdist
        if clen_seq is None:
            clen_seq = rle_lengths(list(lit_lens) + list(dist_lens)) if rle else \
                [(n, 0) for n in list(lit_lens) + list(dist_lens)]
        if clen_lens is None:
            used = {s for s, _ in clen_seq} | {18}      # at least two symbols: the code-length code must be complete
            clen_lens = balanced_lengths(used, 19)
        if hclen is None:
            hclen = max([i + 1 for i, s in enumerate(CLEN_ORDER) if clen_lens[s]] + [4])
        w = self.w
        w.bits(int(final), 1)
        w.bits(2, 2)
        w.bits(hlit - 257, 5)
        w.bits(hdist - 1, 5)
        w.bits(hclen - 4, 4)
        for i in range(hclen):
            w.bits(clen_lens[CLEN_ORDER[i]], 3)
        cc = canonical(clen_lens)
        for s, e in clen_seq:
            w.code(*cc[s])
            w.bits(e, {16: 2, 17: 3, 18: 7}.get(s, 0))
        self._body(items, canonical(lit_lens), canonical(dist_lens), eob)
        return self

    def bits(self, v, n):
        self.w.bits(v, n)
        return self

    def finish(self) -> bytes:
        return self.w.getvalue()


def rle_lengths(lens) -> list:
    """Code-length symbols for a length sequence: 17 / 18 for zero runs, 16 for repeats of the previous length."""
    out, i = [], 0
    while i < len(lens):
        n = lens[i]
        run = 1
        while i + run < len(lens) and lens[i + run] == n:
            run += 1
        if n == 0 and run >= 3:
            k = min(run, 138)
            out.append((18, k - 11) if k >= 11 else (17, k - 3))
            i += k
        elif n != 0 and run >= 4:
            out.append((n, 0))
            k = min(run - 1, 6)
            out.append((16, k - 3))
            i += 1 + k
        else:
            out.append((n, 0))
            i += 1
    return out


def gzip_member(body: bytes, data: bytes, extra=None, name=None, comment=None, hcrc=False, crc=None, isize=None,
                flags=0, mtime=0, xfl=0, os_=255) -> bytes:
    """RFC 1952 member around a raw Deflate body.  crc / isize override the trailer; flags adds raw FLG bits."""
    flg = flags | (4 if extra is not None else 0) | (8 if name is not None else 0) | \
        (16 if comment is not None else 0) | (2 if hcrc else 0)
    h = bytearray(b"\x1f\x8b\x08" + bytes([flg]) + struct.pack("<I", mtime) + bytes([xfl, os_]))
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if name is not None:
        h += name + b"\0"
    if comment is not None:
        h += comment + b"\0"
    if hcrc:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xFFFF)
    trailer = struct.pack("<II", zlib.crc32(data) if crc is None else crc,
                          (len(data) & 0xFFFFFFFF) if isize is None else isize)
    return bytes(h) + body + trailer


def _text(n, seed=1):
    x, out = seed, bytearray()
    for _ in range(n):
        x = (x * 1103515245 + 12345) & 0x7FFFFFFF
        out.append(b"abcdefgh "[x % 9])
    return list(bytes(out))


def valid_streams() -> list:
    """(name, raw deflate stream, expected bytes) of hand-built streams zlib accepts."""
    out = []

    def add(name, s):
        out.append((name, s.finish(), bytes(s.data)))

    t = _text(300)
    s = DeflateStream().stored(bytes(range(200))).fixed(t[:100] + [(20, 7)]).dynamic(t[100:] + [(10, 150), (258, 1)])
    add("mixed_stored_fixed_dynamic", s.stored(b"tail", final=True))
    add("empty_stored_blocks", DeflateStream().stored(b"").stored(b"x").stored(b"").fixed([65, (5, 1)])
        .stored(b"", final=True))
    add("empty_final_stored", DeflateStream().stored(b"", final=True))
    add("dynamic_eob_only", DeflateStream().dynamic([], final=True))                  # lit code: 256 alone, length 1
    add("dynamic_eob_only_complete", DeflateStream().dynamic([], final=True, lit_lens=[1] + [0] * 255 + [1]))
    add("lit_single_code_after_data", DeflateStream().fixed([1, 2, 3]).dynamic([], final=True))
    add("empty_distance_set", DeflateStream().dynamic(t[:50], final=True))            # HDIST = 1, length 0
    add("hlit257_hdist1", DeflateStream().dynamic([7, 7, 9], final=True, lit_lens=balanced_lengths({7, 9, 256}, 257),
                                                  dist_lens=[0]))
    ll = balanced_lengths(set(range(0, 256, 3)) | {256, 285}, 286)
    add("hlit286_hdist30", DeflateStream().dynamic([0, 3, 6, (258, 2), (258, 24577)][:4], final=True, lit_lens=ll,
                                                   dist_lens=balanced_lengths(range(30), 30)))
    # lit lengths end in zeros, distance lengths start with zeros: one 18 repeat covers both
    lit = [0] * 277
    for s_ in (97, 98, 256, 257):
        lit[s_] = 2
    dist = [0] * 5 + [1, 1]
    # 97 zeros, 97, 98, 138 + 19 zeros, 256, 257, then 19 literal/length zeros and 5 distance zeros in one 18
    seq = [(18, 97 - 11), (2, 0), (2, 0), (18, 138 - 11), (18, 19 - 11), (2, 0), (2, 0), (18, 24 - 11), (1, 0), (1, 0)]
    add("repeat_crosses_lit_dist_boundary", DeflateStream().dynamic([97, 98] * 5 + [(3, 7), (3, 9)], final=True,
                                                                    lit_lens=lit, dist_lens=dist, clen_seq=seq))
    # 16 repeats the last literal/length length into the distance lengths
    lit2 = balanced_lengths({65, 256, 257, 258}, 259)
    seq2 = rle_lengths(lit2[:257]) + [(2, 0), (2, 0), (16, 0), (2, 0)]
    add("repeat16_crosses_boundary", DeflateStream().dynamic([65, (3, 1), (4, 2), (3, 3)], final=True, lit_lens=lit2,
                                                             dist_lens=[2, 2, 2, 2], clen_seq=seq2))
    add("length258_code285", DeflateStream().fixed([1, 2, (258, 1), (258, 2)], final=True))
    add("length257_code284_extra30", DeflateStream().fixed([5, ("L", 284, 30, 1)], final=True))
    big = _text(40000, 7)
    s = DeflateStream().stored(bytes(big[:32768])).fixed([(258, 32768), (100, 32768), (3, 32767)], final=True)
    add("distance_32768", s)
    # codes of length 15 in both the literal/length and the distance code (second-level tables)
    deep = list(range(1, 16)) + [15]
    lit3 = [0] * 286
    for i, s_ in enumerate([256, 65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 257, 258, 259, 260, 285]):
        lit3[s_] = deep[i]
    dist3 = [0] * 30
    for i, s_ in enumerate([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 29]):
        dist3[s_] = deep[i]
    items = [65, 74, 73, (3, 1), (6, 2), (258, 3), 72, (4, 16), (3, 25000), 66, (5, 12)]
    add("max_length_codes", DeflateStream().stored(bytes(30000)).dynamic(items, lit_lens=lit3, dist_lens=dist3)
        .dynamic(items[:5], final=True, lit_lens=lit3, dist_lens=dist3, rle=True))
    add("overlap_matches", DeflateStream().fixed([1, 2, 3, (255, 1), (100, 3), 9, (258, 50), (40, 33)], final=True))
    return out


def code284_extra31() -> tuple[bytes, bytes]:
    """Length code 284 with extra value 31 (length 258, which code 285 should carry): the verdict is zlib's."""
    s = DeflateStream().fixed([5, ("L", 284, 31, 1)], final=True)
    return s.finish(), bytes(s.data)


def gzip_streams() -> list:
    """(name, gzip member, expected bytes) with every optional header field."""
    t = bytes(_text(5000, 3))
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    body = c.compress(t) + c.flush()
    return [
        ("plain", gzip_member(body, t), t),
        ("fextra", gzip_member(body, t, extra=b"AB\x04\x00data"), t),
        ("fname", gzip_member(body, t, name=b"table.bin"), t),
        ("fcomment", gzip_member(body, t, comment=b"x" * 100), t),
        ("fhcrc", gzip_member(body, t, hcrc=True), t),
        ("all_fields", gzip_member(body, t, extra=bytes(300), name=b"n" * 40, comment=b"c", hcrc=True, mtime=12345,
                                   xfl=2, os_=3), t),
        ("empty_body", gzip_member(DeflateStream().fixed([], final=True).finish(), b""), b""),
        ("trailing_bytes", gzip_member(body, t, name=b"a") + b"\x1f\x8b garbage", t),
    ]


def invalid_streams() -> list:
    """(rule, raw deflate stream) -- one stream per rejection rule of the decoder."""
    t = _text(60)
    out = []
    out.append(("btype3", DeflateStream().bits(1, 1).bits(3, 2).bits(0, 13).finish()))
    out.append(("stored_nlen", DeflateStream().stored(b"abc", final=True, nlen=0x1234).finish()))
    good = DeflateStream().fixed(t + [(30, 5)], final=True).finish()
    out.append(("truncated", good[:-2]))
    out.append(("no_final_block", DeflateStream().fixed(t).finish()))
    out.append(("truncated_stored", DeflateStream().stored(b"abcdefgh", final=True).finish()[:-3]))
    out.append(("hlit_287", DeflateStream().dynamic(t, final=True, hlit=287, lit_lens=balanced_lengths(set(t) | {256}, 287))
                .finish()))
    out.append(("hdist_31", DeflateStream().dynamic(t, final=True, dist_lens=[1] * 31).finish()))
    out.append(("clen_oversubscribed", DeflateStream().dynamic(t, final=True, clen_lens=[1, 1, 1] + [0] * 15 + [1],
                                                               clen_seq=[], eob=False).bits(0, 16).finish()))
    cl = [0] * 19
    cl[1], cl[2], cl[18] = 1, 2, 3                   # incomplete: 1/2 + 1/4 + 1/8
    out.append(("clen_incomplete", DeflateStream().dynamic(t, final=True, clen_lens=cl, clen_seq=[], eob=False)
                .bits(0, 16).finish()))
    cl = [0] * 19
    cl[1] = 1                                        # a single code-length code of length 1 is not allowed
    out.append(("clen_single", DeflateStream().dynamic(t, final=True, clen_lens=cl, clen_seq=[(1, 0)] * 258,
                                                       eob=False).finish()))
    lens = balanced_lengths(set(t) | {256}, 257)
    over = list(lens)
    over[0] = 1
    over[1] = 1
    out.append(("lit_oversubscribed", DeflateStream().dynamic([], final=True, lit_lens=over, eob=False)
                .bits(0, 16).finish()))
    inc = list(lens)
    inc[t[0]] += 1                                   # one code one bit longer: incomplete
    out.append(("lit_incomplete", DeflateStream().dynamic([], final=True, lit_lens=inc, eob=False).bits(0, 16)
                .finish()))
    out.append(("lit_two_length1_plus", DeflateStream().dynamic([], final=True, lit_lens=[1] + [0] * 255 + [2],
                                                                eob=False).bits(0, 16).finish()))
    out.append(("dist_oversubscribed", DeflateStream().dynamic(t, final=True, dist_lens=[1, 1, 1], eob=False)
                .bits(0, 16).finish()))
    out.append(("dist_incomplete", DeflateStream().dynamic(t, final=True, dist_lens=[1, 2], eob=False).bits(0, 16)
                .finish()))
    no_eob = balanced_lengths(set(t) | {255}, 257)
    out.append(("no_eob_code", DeflateStream().dynamic([], final=True, lit_lens=no_eob, eob=False).bits(0, 16)
                .finish()))
    out.append(("repeat16_first", DeflateStream().dynamic(t, final=True, clen_seq=[(16, 0)] + [(0, 0)] * 300,
                                                          eob=False).finish()))
    lit = balanced_lengths(set(t) | {256}, 257)
    seq = rle_lengths(lit) + [(18, 127)]              # 138 zeros where only 1 distance length remains
    out.append(("repeat_past_end", DeflateStream().dynamic(t, final=True, lit_lens=lit, dist_lens=[0], clen_seq=seq,
                                                           eob=False).finish()))
    seq = rle_lengths(lit)[:-1] + [(lit[-1], 0), (16, 3)]   # 16 of 6 where 1 remains
    out.append(("repeat16_past_end", DeflateStream().dynamic(t, final=True, lit_lens=lit, dist_lens=[0], clen_seq=seq,
                                                             eob=False).finish()))
    out.append(("unassigned_lit_code", DeflateStream().fixed([7]).dynamic([("bits", 1, 1)], final=True,
                                                                        lit_lens=[0] * 256 + [1], eob=False)
                .bits(0, 16).finish()))
    out.append(("empty_distance_set_used", DeflateStream().dynamic([65, ("lit", 257), ("bits", 0, 8)], final=True,
                                                                   lit_lens=balanced_lengths({65, 256, 257}, 258),
                                                                   dist_lens=[0], eob=False).bits(0, 16).finish()))
    out.append(("unassigned_dist_code", DeflateStream().dynamic([65, ("lit", 257), ("bits", 1, 1)], final=True,
                                                                lit_lens=balanced_lengths({65, 256, 257}, 258),
                                                                dist_lens=[1], eob=False).bits(0, 16).finish()))
    out.append(("fixed_lit_286", DeflateStream().fixed([65, ("lit", 286)], final=True).finish()))
    out.append(("fixed_lit_287", DeflateStream().fixed([65, ("lit", 287)], final=True).finish()))
    out.append(("fixed_dist_30", DeflateStream().fixed([65, ("lit", 257), ("dist", 30, 0)], final=True).finish()))
    out.append(("fixed_dist_31", DeflateStream().fixed([65, ("lit", 257), ("dist", 31, 0)], final=True).finish()))
    out.append(("distance_too_far", DeflateStream().fixed([1, 2, 3, (4, 4)], final=True).finish()))
    out.append(("distance_too_far_first", DeflateStream().fixed([(3, 1)], final=True).finish()))
    out.append(("distance_32768_short", DeflateStream().stored(bytes(32767)).fixed([(3, 32768)], final=True)
                .finish()))
    return out


def invalid_gzip() -> list:
    """(rule, gzip member, expected verdict: 'bad' or 'checksum')."""
    t = bytes(_text(3000, 5))
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    body = c.compress(t) + c.flush()
    good = gzip_member(body, t)
    return [
        ("bad_id", b"\x1f\x8c" + good[2:], "bad"),
        ("bad_cm", good[:2] + b"\x07" + good[3:], "bad"),
        ("reserved_flag", gzip_member(body, t, flags=0x20), "bad"),
        ("reserved_flag_80", gzip_member(body, t, flags=0x80), "bad"),
        ("bad_hcrc", gzip_member(body, t, hcrc=True)[:-len(body) - 10] + b"\x00\x00" + body + good[-8:], "bad"),
        ("fname_unterminated", good[:3] + b"\x08" + good[4:10] + b"name" * 10, "bad"),
        ("fextra_too_long", gzip_member(body, t, extra=b"ab")[:10] + b"\xff\x00ab", "bad"),
        ("short_header", good[:9], "bad"),
        ("truncated_trailer", good[:-3], "bad"),
        ("no_trailer", good[:-8], "bad"),
        ("bad_crc", gzip_member(body, t, crc=zlib.crc32(t) ^ 1), "checksum"),
        ("bad_isize", gzip_member(body, t, isize=len(t) + 1), "checksum"),
        ("bad_crc_and_isize", gzip_member(body, t, crc=0, isize=0), "checksum"),
    ]


# ---------------------------------------------------------------------------------------------------------------------
# zlib as the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _gzip_body_len(stream: bytes) -> int:
    """Bytes zlib produces for a gzip member whose trailer check fails (fed byte by byte: the body's output arrives
    before the trailer is read)."""
    d = zlib.decompressobj(31)
    n = 0
    for i in range(len(stream)):
        try:
            n += len(d.decompress(stream[i:i + 1]))
        except zlib.error:
            break
    return n


def zlib_expect(stream: bytes, gz: bool, cap: int):
    """The decoder's required verdict: ("ok", bytes), ("checksum", None) or ("bad", None).  A chunk decodes iff
    zlib reaches the end of the stream (raw: the final block; gzip: the trailer) without an error and the output fits
    in cap.  A gzip member whose body decodes but whose CRC-32 / ISIZE disagree is a checksum failure."""
    d = zlib.decompressobj(31 if gz else -15)
    try:
        out = d.decompress(stream)
    except zlib.error as e:
        if gz and ("incorrect data check" in str(e) or "incorrect length check" in str(e)):
            return ("checksum", None) if _gzip_body_len(stream) <= cap else ("bad", None)
        return "bad", None
    if not d.eof or len(out) > cap:
        return "bad", None
    return "ok", out


def compress(data: bytes, gz: bool, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem_level=8, flushes=()) -> bytes:
    """zlib stream of data; flushes: (offset, mode) points where a Z_SYNC_FLUSH / Z_FULL_FLUSH is issued."""
    c = zlib.compressobj(level, zlib.DEFLATED, 31 if gz else -15, mem_level, strategy)
    out, pos = [], 0
    for off, mode in flushes:
        out.append(c.compress(data[pos:off]))
        out.append(c.flush(mode))
        pos = off
    out.append(c.compress(data[pos:]))
    out.append(c.flush())
    return b"".join(out)


def _campaign_data(rng) -> bytes:
    import numpy as np
    n = int(rng.choice([0, 1, 5, 64, 300, 1000, 2048, 4096, 8192]))
    kind = int(rng.integers(0, 5))
    if kind == 0:
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == 1:
        return rng.integers(0, int(rng.choice([2, 4, 16])), n, dtype=np.uint8).tobytes()
    if kind == 2:
        walk = np.round(100 + rng.normal(0, 0.05, n // 4 + 1).cumsum(), 2).astype(np.float32)
        return walk.view(np.uint8)[:n].tobytes()
    if kind == 3:
        per = rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes()
        return (per * (n // len(per) + 1))[:n]
    return bytes(_text(n, int(rng.integers(1, 1 << 30))))


def corruption_corpus(seed: int, cases: int) -> list:
    """(gz, stream, cap) of seeded corruptions of zlib streams: bit flips, truncations, appended bytes and garbage."""
    import numpy as np
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < cases:
        gz = bool(rng.integers(0, 2))
        data = _campaign_data(rng)
        good = compress(data, gz, level=int(rng.choice([0, 1, 6, 9])),
                        strategy=int(rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY,
                                                 zlib.Z_RLE, zlib.Z_FIXED])),
                        mem_level=int(rng.choice([1, 8, 9])))
        cap = len(data) + int(rng.choice([0, 0, 1, 100]))
        kind = int(rng.integers(0, 5))
        b = bytearray(good)
        if kind <= 1:                                             # 1-4 bit flips (kind 1: inside the first bytes)
            span = min(len(b), 24) if kind == 1 else len(b)
            for _ in range(int(rng.integers(1, 5))):
                i = int(rng.integers(0, span))
                b[i] ^= 1 << int(rng.integers(0, 8))
        elif kind == 2:                                           # truncation
            b = b[: int(rng.integers(0, len(b)))]
        elif kind == 3:                                           # appended bytes: ignored after the end
            b += rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes()
        else:                                                     # garbage, raw or behind a valid gzip header
            g = rng.integers(0, 256, int(rng.integers(1, 3000)), dtype=np.uint8).tobytes()
            b = bytearray((good[:10] + g) if gz and rng.random() < 0.5 else g)
            cap = 65536
        out.append((gz, bytes(b), cap))
    return out
