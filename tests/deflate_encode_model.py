"""Test infrastructure: a plain Python model of the Deflate encoder's stream rules (nvcomp_b200/csrc/deflate_compress.cuh).

Given a chunk and the encoder's parse (its literal runs and matches), `encode` rebuilds the stream the rules call for:
  * block choice: the exact bit cost of one stored encoding (65 535-byte blocks), one fixed-code block and one
    dynamic-code block; the cheapest wins, ties go to stored, then fixed;
  * code lengths: package-merge with limit 15 (literal/length, distance) and 7 (code lengths); leaves ordered by
    (frequency, symbol), a leaf before a package of equal weight; one used symbol gets length 1; a block without
    matches carries distance code 0 with length 1;
  * header: minimal HLIT >= 257 and HDIST >= 1, the lengths run-length coded greedily with 16 / 17 / 18, HCLEN trimmed;
  * the last byte zero-padded.
`parse_stream` reads any raw Deflate stream back into blocks and tokens.  Tables and the bit writer come from
deflate_writer.py.
"""
from __future__ import annotations

import heapq

import deflate_writer as W

CLEN_ORDER = W.CLEN_ORDER
STORED_MAX = 65535


def max_output_size(m: int) -> int:
    return m + 5 * (m // 65535 + 1)


def len_extra(sym: int) -> int:
    return W.LEN_EXTRA[sym - 257]


def pm_lengths(freq, limit: int) -> list:
    """Optimal length-limited code lengths by package-merge, with the encoder's tie rules."""
    lens = [0] * len(freq)
    syms = sorted((s for s in range(len(freq)) if freq[s]), key=lambda s: (freq[s], s))
    n = len(syms)
    if n <= 1:
        for s in syms:
            lens[s] = 1
        return lens
    leaves = [freq[s] for s in syms]
    cur = [(w, 0, i) for i, w in enumerate(leaves)]          # (weight, 0 = leaf / 1 = package, index)
    levels = [cur]                                             # deepest first
    for _ in range(limit - 1):
        pk = [(cur[2 * k][0] + cur[2 * k + 1][0], 1, k) for k in range(len(cur) // 2)]
        cur = list(heapq.merge([(w, 0, i) for i, w in enumerate(leaves)], pk))
        levels.append(cur)
    k = 2 * n - 2
    by_rank = [0] * n
    for lvl in reversed(levels):                               # top level first
        ell = sum(1 for it in lvl[:k] if it[1] == 0)
        for r in range(ell):
            by_rank[r] += 1
        k = 2 * (k - ell)
    for r, s in enumerate(syms):
        lens[s] = by_rank[r]
    return lens


def rle(lens) -> list:
    """(code-length symbol, extra value, extra bits) for a length sequence, greedy."""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        r = run
        if v == 0:
            while r >= 3:
                k = min(r, 138)
                out.append((18, k - 11, 7) if k >= 11 else (17, k - 3, 3))
                r -= k
        else:
            out.append((v, 0, 0))
            r -= 1
            while r >= 3:
                k = min(r, 6)
                out.append((16, k - 3, 2))
                r -= k
        out += [(v, 0, 0)] * r
        i += run
    return out


def tokens_from_parse(data: bytes, triples) -> list:
    """(literal run, distance, length) triples -> items: literal ints and (length, distance) tuples."""
    items, p = [], 0
    for ll, d, ml in triples:
        items += list(data[p:p + ll])
        p += ll
        if ml:
            items.append((ml, d))
            p += ml
    assert p == len(data), (p, len(data))
    return items


def histograms(items):
    lit, dist = [0] * 286, [0] * 30
    lit[256] = 1
    for it in items:
        if isinstance(it, int):
            lit[it] += 1
        else:
            lit[W.length_code(it[0])[0]] += 1
            dist[W.dist_code(it[1])[0]] += 1
    return lit, dist


def plan(data: bytes, items) -> dict:
    """The encoder's decisions for this parse: block type, costs and (for a dynamic block) every header field."""
    lit, dist = histograms(items)
    extra = sum(lit[s] * len_extra(s) for s in range(257, 286)) + sum(dist[d] * W.DIST_EXTRA[d] for d in range(30))
    fixed_bits = 3 + sum(lit[s] * W.FIXED_LIT[s] for s in range(286)) + 5 * sum(dist) + extra
    n = len(data)
    blocks = max(1, -(-n // STORED_MAX))
    stored_bits = 8 * (n + 5 * blocks)
    lit_lens = pm_lengths(lit, 15)
    dist_lens = pm_lengths(dist, 15)
    if not any(dist_lens):
        dist_lens[0] = 1
    hlit = max(257, max(s for s in range(286) if lit_lens[s]) + 1)
    hdist = max(1, max(d for d in range(30) if dist_lens[d]) + 1)
    seq = rle(lit_lens[:hlit] + dist_lens[:hdist])
    cfreq = [0] * 19
    for s, _, _ in seq:
        cfreq[s] += 1
    clen_lens = pm_lengths(cfreq, 7)
    hclen = max([i + 1 for i, s in enumerate(CLEN_ORDER) if clen_lens[s]] + [4])
    body = sum(lit[s] * lit_lens[s] for s in range(286)) + sum(dist[d] * dist_lens[d] for d in range(30)) + extra
    dyn_bits = 3 + 14 + 3 * hclen + sum(cfreq[s] * clen_lens[s] for s in range(19)) + sum(nb for _, _, nb in seq) + body
    dyn_ok = sum(1 for x in clen_lens if x) >= 2
    if stored_bits <= fixed_bits and (not dyn_ok or stored_bits <= dyn_bits):
        kind = "stored"
    elif fixed_bits <= dyn_bits or not dyn_ok:
        kind = "fixed"
    else:
        kind = "dynamic"
    return dict(kind=kind, stored_bits=stored_bits, fixed_bits=fixed_bits, dyn_bits=dyn_bits, lit=lit, dist=dist,
                lit_lens=lit_lens, dist_lens=dist_lens, hlit=hlit, hdist=hdist, hclen=hclen, seq=seq,
                clen_lens=clen_lens, cfreq=cfreq)


def encode(data: bytes, items) -> bytes:
    """The stream the rules call for, for this chunk and parse."""
    p = plan(data, items)
    w = W.BitWriter()
    if p["kind"] == "stored":
        out, pos = bytearray(), 0
        blocks = max(1, -(-len(data) // STORED_MAX))
        for b in range(blocks):
            chunk = data[pos:pos + STORED_MAX]
            n = len(chunk)
            out += bytes([int(b + 1 == blocks), n & 255, n >> 8, ~n & 255, (~n >> 8) & 255]) + chunk
            pos += n
        return bytes(out)
    if p["kind"] == "fixed":
        w.bits(3, 3)
        lit_c, dist_c = W.canonical(W.FIXED_LIT), W.canonical(W.FIXED_DIST)
    else:
        w.bits(5, 3)
        w.bits(p["hlit"] - 257, 5)
        w.bits(p["hdist"] - 1, 5)
        w.bits(p["hclen"] - 4, 4)
        for i in range(p["hclen"]):
            w.bits(p["clen_lens"][CLEN_ORDER[i]], 3)
        cc = W.canonical(p["clen_lens"])
        for s, ev, nb in p["seq"]:
            w.code(*cc[s])
            w.bits(ev, nb)
        lit_c, dist_c = W.canonical(p["lit_lens"]), W.canonical(p["dist_lens"])
    for it in items:
        if isinstance(it, int):
            w.code(*lit_c[it])
        else:
            c, e = W.length_code(it[0])
            w.code(*lit_c[c])
            w.bits(e, len_extra(c))
            dc, de = W.dist_code(it[1])
            w.code(*dist_c[dc])
            w.bits(de, W.DIST_EXTRA[dc])
    w.code(*lit_c[256])
    return w.getvalue()


class _Reader:
    def __init__(self, data: bytes):
        self.data, self.pos = data, 0

    def bits(self, n: int) -> int:
        v = 0
        for i in range(n):
            byte = self.data[self.pos >> 3]
            v |= ((byte >> (self.pos & 7)) & 1) << i
            self.pos += 1
        return v

    def sym(self, table: dict) -> int:
        code, n = 0, 0
        while True:
            code = (code << 1) | self.bits(1)
            n += 1
            if (code, n) in table:
                return table[(code, n)]
            assert n <= 15, "invalid code"


def _decode_table(lens) -> dict:
    return {cl: s for s, cl in W.canonical(lens).items()}


def parse_stream(stream: bytes) -> list:
    """Blocks of a raw Deflate stream: dicts with kind, final, and items (stored: the payload) plus, for a dynamic
    block, hlit / hdist / hclen / clen_lens / seq / lit_lens / dist_lens.  The padding after the last block must be
    zero bits, and nothing may follow it."""
    r, blocks = _Reader(stream), []
    while True:
        final, btype = r.bits(1), r.bits(2)
        blk = dict(final=final)
        if btype == 0:
            r.pos = (r.pos + 7) & ~7
            n, nn = r.bits(16), r.bits(16)
            assert n ^ nn == 0xFFFF
            blk.update(kind="stored", payload=stream[r.pos >> 3:(r.pos >> 3) + n])
            r.pos += 8 * n
        else:
            assert btype in (1, 2)
            if btype == 1:
                lit_lens, dist_lens = W.FIXED_LIT, W.FIXED_DIST
                blk["kind"] = "fixed"
            else:
                hlit, hdist, hclen = r.bits(5) + 257, r.bits(5) + 1, r.bits(4) + 4
                clen_lens = [0] * 19
                for i in range(hclen):
                    clen_lens[CLEN_ORDER[i]] = r.bits(3)
                ct = _decode_table(clen_lens)
                lens, seq = [], []
                while len(lens) < hlit + hdist:
                    s = r.sym(ct)
                    nb = {16: 2, 17: 3, 18: 7}.get(s, 0)
                    ev = r.bits(nb)
                    seq.append((s, ev, nb))
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + ev)
                    else:
                        lens += [0] * ((3 if s == 17 else 11) + ev)
                assert len(lens) == hlit + hdist
                lit_lens, dist_lens = lens[:hlit] + [0] * (286 - hlit), lens[hlit:] + [0] * (30 - hdist)
                blk.update(kind="dynamic", hlit=hlit, hdist=hdist, hclen=hclen, clen_lens=clen_lens, seq=seq,
                           lit_lens=lit_lens, dist_lens=dist_lens)
            lt, dt = _decode_table(lit_lens), _decode_table(dist_lens)
            items = []
            while True:
                s = r.sym(lt)
                if s < 256:
                    items.append(s)
                elif s == 256:
                    break
                else:
                    length = W.LEN_BASE[s - 257] + r.bits(len_extra(s))
                    d = r.sym(dt)
                    items.append((length, W.DIST_BASE[d] + r.bits(W.DIST_EXTRA[d])))
            blk["items"] = items
        blocks.append(blk)
        if final:
            break
    end = (r.pos + 7) >> 3
    assert end == len(stream), ("trailing bytes", end, len(stream))
    if r.pos & 7:
        assert stream[-1] >> (r.pos & 7) == 0, "nonzero padding"
    return blocks
