"""Test infrastructure: a plain Python model of the Zstd encoder's stream rules (include/nvcomp/device/detail/
zstd_encode.cuh), in the style of deflate_encode_model.py.

Given a chunk and the matcher's parse (its literal runs and matches, before block cutting), `encode` rebuilds the
frame the rules call for:
  * frame: a 6- or 7-byte single-segment header without checksum;
  * blocks: 16 KB of input each; a match crossing a block end is split there and a piece under 4 bytes becomes
    literals; a block of >= 2 equal bytes is RLE, otherwise Compressed when its body is strictly smaller than the
    block, else Raw; an empty chunk is one empty Raw block;
  * repeat offsets: history (1, 4, 8), codes checked rep0, rep1, rep2 (rep1, rep2 without literals), updated only by
    Compressed blocks, by the slot the code names;
  * literals: Raw, RLE or Huffman by exact size (ties Raw, then RLE), the smallest Size_Format; package-merge lengths
    limited to 11 bits, weights mb + 1 - len, codes by weight then symbol; direct or FSE weights (ties direct); one
    stream below 256 literals, else four of (L + 3) / 4, each written last literal first and closed with a 1 bit;
  * sequences: Predefined, RLE or FSE per table by the 1/256-bit cost estimate (ties Predefined, then RLE), libzstd's
    normalisation and FSE_writeNCount, states started on the first cell of the last sequence's code, and the RFC's
    bitstream order.
`plan` returns every decision and size behind the frame; `parse_frame` reads any frame of this encoder back into its
blocks, literals, Huffman weights, normalised counts and sequences, without using the rules above.  The FSE decode
tables come from zstd_writer._fse_table, and the encoder's state tables are read off them as the encoder does.
"""
from __future__ import annotations

import deflate_encode_model as DM
import zstd_writer as W

BLOCK = 16384
MIN_MATCH = 4
MAX_OFFSET = 65535
HUF_LIMIT = 11
NAMES = ("LL", "OF", "ML")
# per table: predefined normalised counts, predefined log, largest accuracy log
PREDEFINED = {"LL": (W._LL_DEF, 6, 9), "OF": (W._OF_DEF, 5, 8), "ML": (W._ML_DEF, 6, 9)}
DECODER_MAX_CODE = {"LL": 35, "OF": 31, "ML": 52}


def highbit(v: int) -> int:
    return v.bit_length() - 1


class Bits:
    """LSB-first bit writer."""

    def __init__(self):
        self.out, self.acc, self.nb = bytearray(), 0, 0

    def add(self, v: int, n: int):
        assert 0 <= v < (1 << n) or (n == 0 and v == 0), (v, n)
        self.acc |= v << self.nb
        self.nb += n
        while self.nb >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.nb -= 8

    def pad(self):
        if self.nb:
            self.out.append(self.acc & 255)
        self.acc, self.nb = 0, 0

    def close(self):
        self.add(1, 1)
        self.pad()


# ---------------------------------------------------------------------------------------------------------------------
# FSE
# ---------------------------------------------------------------------------------------------------------------------
def cost(c: int, log: int) -> int:
    """Cost in 1/256 bit of a symbol of probability c / 2^log: log2 taken as highbit plus a linear mantissa."""
    hb = highbit(c)
    return (log << 8) - ((hb << 8) + ((c << 8) >> hb) - 256)


def table_log(max_log: int, n: int, max_sym: int) -> int:
    """libzstd's FSE_optimalTableLog(max_log, n, max_sym) for n >= 5 symbols.  Below 5 libzstd's unsigned
    highbit(n - 1) - 2 wraps and it keeps max_log; the encoder uses 5 there, which lets a block of 4 sequences take
    an FSE table that would cost more than Predefined at max_log."""
    if n < 5:
        return 5
    log = min(max_log, highbit(n - 1) - 2)
    log = max(log, min(highbit(n) + 1, highbit(max(max_sym, 1)) + 2))
    return min(max(log, 5), max_log)


def normalize(hist, max_sym: int, total: int, log: int) -> list:
    """Each used code gets max(1, count * 2^log / total); a positive remainder goes to the most frequent code (the
    lowest on ties); a negative one is taken from the largest counts (the lowest code on ties) down to 1."""
    norm = [max(1, (hist[s] << log) // total) if hist[s] else 0 for s in range(max_sym + 1)]
    big = 0
    for s in range(max_sym + 1):
        if hist[s] > hist[big]:
            big = s
    diff = (1 << log) - sum(norm)
    if diff > 0:
        norm[big] += diff
    while diff < 0:
        m = 0
        for s in range(1, max_sym + 1):
            if norm[s] > norm[m]:
                m = s
        take = min(-diff, norm[m] - 1)
        norm[m] -= take
        diff += take
    return norm


def write_ncount(bo: Bits, norm, max_sym: int, log: int):
    """RFC 8878 4.1.1 (libzstd's FSE_writeNCount), padded to a byte."""
    bo.add(log - 5, 4)
    remaining, threshold, nbits = (1 << log) + 1, 1 << log, log + 1
    s, prev0 = 0, False
    while s <= max_sym and remaining > 1:
        if prev0:
            start = s
            while norm[s] == 0:
                s += 1
            while s >= start + 3:
                bo.add(3, 2)
                start += 3
            bo.add(s - start, 2)
        count = norm[s]
        s += 1
        mx = 2 * threshold - 1 - remaining
        remaining -= abs(count)
        count += 1
        if count >= threshold:
            count += mx
        bo.add(count, nbits - (1 if count < mx else 0))
        prev0 = count == 1
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    bo.pad()


def ncount_bytes(norm, max_sym: int, log: int) -> bytes:
    bo = Bits()
    write_ncount(bo, norm, max_sym, log)
    return bytes(bo.out)


class FseState:
    """One encoder state over the decode table W._fse_table(norm, log): cnt[s] cells per symbol, st[cum[s] + r] the
    cell whose state is cnt[s] + r."""

    def __init__(self, norm, log: int):
        self.log = log
        tab = W._fse_table(norm, log)
        size = 1 << log
        self.cnt = [0] * len(norm)
        for s, _, _ in tab:
            self.cnt[s] += 1
        self.cum, c = [], 0
        for k in self.cnt:
            self.cum.append(c)
            c += k
        self.st = [0] * size
        for u, (s, nb, base) in enumerate(tab):
            self.st[self.cum[s] + ((base + size) >> nb) - self.cnt[s]] = u
        self.x = 0

    def init(self, s: int):
        self.x = (1 << self.log) + self.st[self.cum[s]]

    def enc(self, bo: Bits, s: int):
        c = self.cnt[s]
        k = self.log - highbit(c)
        nb = k - (1 if (self.x >> k) < c else 0)
        bo.add(self.x & ((1 << nb) - 1), nb)
        self.x = (1 << self.log) + self.st[self.cum[s] + (self.x >> nb) - c]

    def flush(self, bo: Bits):
        bo.add(self.x - (1 << self.log), self.log)


_PRE_CELLS = {t: FseState(PREDEFINED[t][0], PREDEFINED[t][1]).cnt for t in NAMES}


# ---------------------------------------------------------------------------------------------------------------------
# literals section
# ---------------------------------------------------------------------------------------------------------------------
def raw_lit_header_size(L: int) -> int:
    return 1 if L <= 31 else 2 if L <= 4095 else 3


def huf_lit_header_size(L: int, csz: int, single: bool) -> int:
    m = max(L, csz)
    return 3 if single or m <= 1023 else 4 if m <= 16383 else 5


def canonical_codes(wt, mb: int) -> dict:
    """symbol -> (code, length): by weight, then symbol, as the decoder's table is laid out."""
    start = [0] * 16
    for w in wt:
        if w:
            start[w] += 1 << (w - 1)
    acc = 0
    for k in range(1, mb + 1):
        start[k], acc = acc, acc + start[k]
    codes = {}
    for s, k in enumerate(wt):
        if k:
            codes[s] = (start[k] >> (k - 1), mb + 1 - k)
            start[k] += 1 << (k - 1)
    return codes


def fse_weights(w) -> bytes | None:
    """The FSE form of the weights w (without the header byte), or None when it is not allowed: fewer than two
    distinct values, fewer than two weights, or more than 127 bytes."""
    nw = len(w)
    h = [0] * 16
    for x in w:
        h[x] += 1
    used = [s for s in range(16) if h[s]]
    if len(used) < 2 or nw < 2:
        return None
    max_w = used[-1]
    log = table_log(6, nw, max_w)
    norm = normalize(h, max_w, nw, log)
    bo = Bits()
    write_ncount(bo, norm, max_w, log)
    s1, s2 = FseState(norm, log), FseState(norm, log)
    if nw & 1:
        s1.init(w[nw - 1])
        s2.init(w[nw - 2])
        if nw >= 3:
            s1.enc(bo, w[nw - 3])
        i = nw - 3 if nw >= 3 else 0
    else:
        s2.init(w[nw - 1])
        s1.init(w[nw - 2])
        i = nw - 2
    while i > 0:
        s2.enc(bo, w[i - 1])
        s1.enc(bo, w[i - 2])
        i -= 2
    s2.flush(bo)
    s1.flush(bo)
    bo.close()
    return bytes(bo.out) if len(bo.out) <= 127 else None


def plan_literals(lits: bytes) -> dict:
    """Every literal mode's size and the choice."""
    L = len(lits)
    hist = [0] * 256
    for c in lits:
        hist[c] += 1
    used = [s for s in range(256) if hist[s]]
    lh_raw = raw_lit_header_size(L)
    p = dict(L=L, hist=hist, lh_raw=lh_raw, sizes={"raw": lh_raw + L})
    if len(used) == 1:
        p["sizes"]["rle"] = lh_raw + 1
    if len(used) >= 2:
        maxsym = used[-1]
        lens = DM.pm_lengths(hist, HUF_LIMIT)
        mb = max(lens)
        wt = [mb + 1 - x if x else 0 for x in lens[:maxsym + 1]]
        fse = fse_weights(wt[:maxsym])
        direct_sz = (maxsym + 1) // 2 if maxsym < 128 else 0
        p.update(lens=lens, mb=mb, wt=wt, maxsym=maxsym, fse_weights=fse, direct_sz=direct_sz)
        if direct_sz or fse is not None:
            direct = direct_sz != 0 and (fse is None or direct_sz <= len(fse))
            if direct:
                tree = bytes([127 + maxsym]) + bytes((wt[2 * i] << 4) | (wt[2 * i + 1] if 2 * i + 1 < maxsym else 0)
                                                     for i in range(direct_sz))
            else:
                tree = bytes([len(fse)]) + fse
            codes = canonical_codes(wt, mb)
            single = L < 256
            seg = L if single else (L + 3) // 4
            streams = []
            for k in range(1 if single else 4):
                lo, hi = k * seg, (L if single or k == 3 else (k + 1) * seg)
                bo = Bits()
                for i in range(hi - 1, lo - 1, -1):
                    bo.add(*codes[lits[i]])
                bo.close()
                streams.append(bytes(bo.out))
            csz = len(tree) + (0 if single else 6) + sum(map(len, streams))
            lh = huf_lit_header_size(L, csz, single)
            p.update(weights_form="direct" if direct else "fse", tree=tree, codes=codes, streams=streams, csz=csz,
                     lh=lh, single=single)
            p["sizes"]["huffman"] = lh + csz
    s = p["sizes"]
    p["mode"] = "raw"
    if "rle" in s and s["rle"] < s[p["mode"]]:
        p["mode"] = "rle"
    if "huffman" in s and s["huffman"] < s[p["mode"]]:
        p["mode"] = "huffman"
    return p


def literals_section(lits: bytes, p: dict) -> bytes:
    L, lh = p["L"], p["lh_raw"]
    if p["mode"] in ("raw", "rle"):
        hv = (L << 3) if lh == 1 else (1 << 2) | (L << 4) if lh == 2 else (3 << 2) | (L << 4)
        hv |= p["mode"] == "rle"
        return hv.to_bytes(lh, "little") + (lits if p["mode"] == "raw" else lits[:1])
    lh = p["lh"]
    sf = 0 if p["single"] else {3: 1, 4: 2, 5: 3}[lh]
    fb = {3: 10, 4: 14, 5: 18}[lh]
    hv = 2 | (sf << 2) | (L << 4) | (p["csz"] << (4 + fb))
    jump = b"" if p["single"] else b"".join(len(s).to_bytes(2, "little") for s in p["streams"][:3])
    return hv.to_bytes(lh, "little") + p["tree"] + jump + b"".join(p["streams"])


# ---------------------------------------------------------------------------------------------------------------------
# sequences section
# ---------------------------------------------------------------------------------------------------------------------
def ll_code(v: int) -> int:
    if v < 16:
        return v
    return 16 + max(i for i, (b, _) in enumerate(W._LL_EXTRA) if b <= v)


def ml_code(v: int) -> int:
    if v < 35:
        return v - 3
    return 32 + max(i for i, (b, _) in enumerate(W._ML_EXTRA) if b <= v)


def offset_values(seqs, rep):
    """(ll, Offset_Value, ml) per sequence and the history after them."""
    rep = list(rep)
    out = []
    for ll, off, ml in seqs:
        if ll and off == rep[0]:
            ov = 1
        elif off == rep[1]:
            ov = 2 if ll else 1
        elif off == rep[2]:
            ov = 3 if ll else 2
        else:
            ov = off + 3
        slot = 3 if ov > 3 else ov - 1 + (ll == 0)
        if slot >= 2:
            rep[2] = rep[1]
        if slot >= 1:
            rep[1], rep[0] = rep[0], off
        out.append((ll, ov, ml))
    return out, rep


def plan_table(name: str, codes, nseq: int) -> dict:
    """The mode of one of LL / OF / ML by cost, with the costs."""
    hist = [0] * 64
    for c in codes:
        hist[c] += 1
    used = [s for s in range(64) if hist[s]]
    mx = used[-1]
    pnorm, plog, max_log = PREDEFINED[name]
    pcost = sum(hist[s] * cost(_PRE_CELLS[name][s], plog) for s in used)
    log = table_log(max_log, nseq, mx)
    norm = normalize(hist, mx, nseq, log)
    hdr = ncount_bytes(norm, mx, log)
    fcost = sum(hist[s] * cost(norm[s], log) for s in used) + (len(hdr) << 11)
    mode, best = "predefined", pcost
    if len(used) == 1 and (8 << 8) < best:
        mode, best = "rle", 8 << 8
    if fcost < best:
        mode = "fse"
    return dict(mode=mode, hist=hist, max=mx, pcost=pcost, rle_cost=(8 << 8) if len(used) == 1 else None,
                fcost=fcost, log=log, norm=norm, ncount=hdr)


def plan_sequences(seqs, rep) -> dict:
    recs, nrep = offset_values(seqs, rep)
    p = dict(recs=recs, rep_after=nrep, nseq=len(recs))
    if recs:
        codes = {"LL": [ll_code(ll) for ll, _, _ in recs], "OF": [highbit(ov) for _, ov, _ in recs],
                 "ML": [ml_code(ml) for _, _, ml in recs]}
        p["codes"] = codes
        p["tables"] = {t: plan_table(t, codes[t], len(recs)) for t in NAMES}
    return p


def sequences_section(p: dict) -> bytes:
    nseq = p["nseq"]
    if nseq == 0:
        return b"\x00"
    out = bytearray([nseq] if nseq < 128 else [(nseq >> 8) + 128, nseq & 255])
    tabs = p["tables"]
    mcode = {"predefined": 0, "rle": 1, "fse": 2}
    out.append((mcode[tabs["LL"]["mode"]] << 6) | (mcode[tabs["OF"]["mode"]] << 4) | (mcode[tabs["ML"]["mode"]] << 2))
    states = {}
    for t in NAMES:
        tb = tabs[t]
        if tb["mode"] == "rle":
            out.append(tb["max"])
        elif tb["mode"] == "fse":
            out += tb["ncount"]
            states[t] = FseState(tb["norm"], tb["log"])
        else:
            states[t] = FseState(PREDEFINED[t][0], PREDEFINED[t][1])
    bo = Bits()
    codes = p["codes"]
    for k in range(nseq - 1, -1, -1):
        ll, ov, ml = p["recs"][k]
        c = {t: codes[t][k] for t in NAMES}
        if k == nseq - 1:
            for t in ("LL", "OF", "ML"):
                if t in states:
                    states[t].init(c[t])
        else:
            for t in ("OF", "ML", "LL"):
                if t in states:
                    states[t].enc(bo, c[t])
        llb, llx = W._ll_code(c["LL"])
        mlb, mlx = W._ml_code(c["ML"])
        bo.add(ll - llb, llx)
        bo.add(ml - mlb, mlx)
        bo.add(ov - (1 << c["OF"]), c["OF"])
    for t in ("ML", "OF", "LL"):
        if t in states:
            states[t].flush(bo)
    bo.close()
    return bytes(out + bo.out)


# ---------------------------------------------------------------------------------------------------------------------
# blocks and frame
# ---------------------------------------------------------------------------------------------------------------------
def split_blocks(data: bytes, parse) -> list:
    """The parse cut into 16 KB blocks: [(start, end, literals, [(ll, offset, ml)])]."""
    n = len(data)
    blocks = []
    st = dict(bstart=0, bend=min(BLOCK, n), pos=0, lits=bytearray(), seqs=[], mark=0)

    def close():
        blocks.append((st["bstart"], st["pos"], bytes(st["lits"]), st["seqs"]))
        st.update(bstart=st["pos"], bend=min(st["pos"] + BLOCK, n), lits=bytearray(), seqs=[], mark=0)

    def advance(k):
        st["pos"] += k
        if st["pos"] == st["bend"] and st["pos"] < n:
            close()

    def literals(ll):
        while ll:
            k = min(ll, st["bend"] - st["pos"])
            st["lits"] += data[st["pos"]:st["pos"] + k]
            ll -= k
            advance(k)

    for ll, off, ml in parse[:-1]:
        literals(ll)
        while ml:
            k = min(ml, st["bend"] - st["pos"])
            if k >= MIN_MATCH:
                st["seqs"].append((len(st["lits"]) - st["mark"], off, k))
                st["mark"] = len(st["lits"])
            else:
                st["lits"] += data[st["pos"]:st["pos"] + k]
            ml -= k
            advance(k)
    literals(parse[-1][0])
    close()
    return blocks


def frame_header(n: int) -> bytes:
    return W.MAGIC.to_bytes(4, "little") + (bytes([0x20, n]) if n <= 255 else bytes([0x60]) + (n - 256).to_bytes(2,
                                                                                                               "little"))


def plan(data: bytes, parse) -> list:
    """Per block: its type, the candidate sizes, and the literal and sequence plans of its Compressed form."""
    rep = [1, 4, 8]
    out = []
    for start, end, lits, seqs in split_blocks(data, parse):
        b = data[start:end]
        blen = len(b)
        p = dict(start=start, end=end, lits=lits, seqs=seqs, rep_before=list(rep), sizes={"raw": blen})
        if blen >= 2 and b.count(b[0]) == blen:
            p["sizes"]["rle"] = 1
        elif blen:
            p["lit"] = plan_literals(lits)
            p["seq"] = plan_sequences(seqs, rep)
            p["body"] = literals_section(lits, p["lit"]) + sequences_section(p["seq"])
            p["sizes"]["compressed"] = len(p["body"])
        s = p["sizes"]
        p["type"] = "rle" if "rle" in s else "compressed" if s.get("compressed", blen) < blen else "raw"
        if p["type"] == "compressed":
            rep = p["seq"]["rep_after"]
        out.append(p)
    return out


def encode(data: bytes, parse) -> bytes:
    """The frame the rules call for, for this chunk and parse."""
    out = bytearray(frame_header(len(data)))
    blocks = plan(data, parse)
    for i, p in enumerate(blocks):
        last = int(i + 1 == len(blocks))
        b = data[p["start"]:p["end"]]
        if p["type"] == "rle":
            out += W.block_header(1, len(b), last) + b[:1]
        elif p["type"] == "compressed":
            out += W.block_header(2, len(p["body"]), last) + p["body"]
        else:
            out += W.block_header(0, len(b), last) + b
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# frame -> blocks, literals, weights, counts and sequences
# ---------------------------------------------------------------------------------------------------------------------
def _read_weights(b: bytes) -> dict:
    """Huffman tree description at b[0]: its form, size, the explicit weights and, for the FSE form, its counts."""
    h = b[0]
    if h >= 128:
        n = h - 127
        w = [(b[1 + i // 2] >> 4) if i % 2 == 0 else (b[1 + i // 2] & 15) for i in range(n)]
        return dict(form="direct", size=1 + (n + 1) // 2, weights=w)
    norm, log, hs = W._read_ncount(b[1:1 + h], 15)
    tab = W._fse_table(norm, log)
    br = W._BackBits(b[1 + hs:1 + h])
    st = [br.read(log), br.read(log)]
    w, k = [], 0
    while True:
        sym, nb, base = tab[st[k]]
        w.append(sym)
        st[k] = base + br.read(nb)
        if br.pos < 0:
            w.append(tab[st[1 - k]][0])
            break
        k ^= 1
    return dict(form="fse", size=1 + h, weights=w, norm=norm, log=log, ncount=bytes(b[1:1 + hs]))


def _huffman_lengths(weights) -> tuple:
    """Explicit weights -> (code length per symbol, table log); the last symbol's weight is implied."""
    total = sum(1 << (x - 1) for x in weights if x)
    log = total.bit_length()
    rest = (1 << log) - total
    assert rest and rest & (rest - 1) == 0, "weights do not complete a power of two"
    w = list(weights) + [rest.bit_length()]
    return [log + 1 - x if x else 0 for x in w], log


def _huffman_decode(stream: bytes, lens, log: int, n: int) -> bytes:
    """n symbols of a backward Huffman stream, which must end exactly on its first bit."""
    w = [log + 1 - x if x else 0 for x in lens]
    table = []
    for wt in range(1, log + 1):
        for sym, x in enumerate(w):
            if x == wt:
                table += [(sym, log + 1 - wt)] * (1 << (wt - 1))
    br = W._BackBits(stream)
    out = bytearray()
    for _ in range(n):
        sym, nb = table[br.read(log)]
        br.pos += log - nb
        out.append(sym)
    assert br.pos == 0, "the Huffman stream does not end on its first bit"
    return bytes(out)


def _parse_literals(b: bytes, blk: dict) -> int:
    """The literals section at b[0]; returns its size."""
    lt, sf = b[0] & 3, (b[0] >> 2) & 3
    if lt < 2:
        lh = {0: 1, 2: 1, 1: 2, 3: 3}[sf]
        L = int.from_bytes(b[:lh], "little") >> (3 if lh == 1 else 4)
        blk.update(lit_mode=("raw", "rle")[lt], lit_header=lh, L=L,
                   literals=b[lh:lh + L] if lt == 0 else b[lh:lh + 1] * L)
        return lh + (L if lt == 0 else 1)
    assert lt == 2, "treeless literals"
    lh = {0: 3, 1: 3, 2: 4, 3: 5}[sf]
    hv = int.from_bytes(b[:lh], "little")
    fb = {3: 10, 4: 14, 5: 18}[lh]
    L, csz = (hv >> 4) & ((1 << fb) - 1), hv >> (4 + fb)
    sec = b[lh:lh + csz]
    tree = _read_weights(sec)
    lens, log = _huffman_lengths(tree["weights"])
    nstreams = 1 if sf == 0 else 4
    body = sec[tree["size"]:]
    if nstreams == 1:
        cuts, sizes = [0, len(body)], [len(body)]
    else:
        sizes = [int.from_bytes(body[2 * i:2 * i + 2], "little") for i in range(3)]
        sizes.append(len(body) - 6 - sum(sizes))
        cuts = [6, 6 + sizes[0], 6 + sizes[0] + sizes[1], 6 + sum(sizes[:3]), len(body)]
    seg = L if nstreams == 1 else (L + 3) // 4
    lits = b"".join(_huffman_decode(body[cuts[k]:cuts[k + 1]], lens, log,
                                    seg if k < nstreams - 1 else L - seg * (nstreams - 1)) for k in range(nstreams))
    blk.update(lit_mode="huffman", lit_header=lh, L=L, csz=csz, tree=tree, huf_lens=lens, huf_log=log,
               lit_streams=nstreams, stream_sizes=sizes, literals=lits)
    return lh + csz


def _parse_sequences(b: bytes, blk: dict, rep: list):
    nb = b[0]
    if nb < 128:
        nseq, sp = nb, 1
    else:
        assert nb < 255
        nseq, sp = ((nb - 128) << 8) + b[1], 2
    blk.update(nseq=nseq, nseq_bytes=sp, sequences=[], tables={})
    if nseq == 0:
        assert sp == len(b), "bytes after an empty sequences section"
        return
    modes = b[sp]
    sp += 1
    assert modes & 3 == 0, "reserved bits of the modes byte"
    kinds = [(modes >> 6) & 3, (modes >> 4) & 3, (modes >> 2) & 3]
    tabs = []
    for t, k in zip(NAMES, kinds):
        assert k < 3, "Repeat mode"
        if k == 0:
            pnorm, plog, _ = PREDEFINED[t]
            tabs.append((W._fse_table(pnorm, plog), plog))
            blk["tables"][t] = dict(mode="predefined")
        elif k == 1:
            tabs.append(([(b[sp], 0, 0)], 0))
            blk["tables"][t] = dict(mode="rle", symbol=b[sp])
            sp += 1
        else:
            norm, log, hs = W._read_ncount(b[sp:], DECODER_MAX_CODE[t])
            tabs.append((W._fse_table(norm, log), log))
            blk["tables"][t] = dict(mode="fse", norm=norm, log=log, ncount=bytes(b[sp:sp + hs]))
            sp += hs
    br = W._BackBits(b[sp:])
    (tll, lll), (tof, lof), (tml, lml) = tabs
    sll, sof, sml = br.read(lll), br.read(lof), br.read(lml)
    for k in range(nseq):
        llc, ofc, mlc = tll[sll][0], tof[sof][0], tml[sml][0]
        ov = (1 << ofc) + br.read(ofc)
        mlb, mlx = W._ml_code(mlc)
        ml = mlb + br.read(mlx)
        llb, llx = W._ll_code(llc)
        ll = llb + br.read(llx)
        rep_before = list(rep)
        if ov > 3:
            off = ov - 3
            rep[:] = [off, rep[0], rep[1]]
        else:
            idx = ov + (ll == 0)
            off = rep[idx - 1] if idx < 4 else rep[0] - 1
            if idx == 2:
                rep[:] = [rep[1], rep[0], rep[2]]
            elif idx >= 3:
                rep[:] = [off, rep[0], rep[1]]
        blk["sequences"].append(dict(ll=ll, ov=ov, ml=ml, off=off, rep=rep_before, codes=(llc, ofc, mlc)))
        if k + 1 < nseq:
            e = tll[sll]
            sll = e[2] + br.read(e[1])
            e = tml[sml]
            sml = e[2] + br.read(e[1])
            e = tof[sof]
            sof = e[2] + br.read(e[1])
    assert br.pos == 0, "the sequence bitstream does not end on its first bit"


def parse_frame(frame: bytes) -> dict:
    """One single-segment frame of this encoder -> dict(n, header, blocks, content).  Each block dict has type, start,
    end and size; a Compressed one also has its literals section (mode, header size, literals, and for Huffman the
    weights, code lengths and stream sizes) and its sequences section (count, per-table mode and counts, and every
    sequence with its Offset_Value, offset and the repeat history before it)."""
    assert int.from_bytes(frame[:4], "little") == W.MAGIC
    fhd = frame[4]
    assert fhd in (0x20, 0x60), hex(fhd)
    n = frame[5] if fhd == 0x20 else int.from_bytes(frame[5:7], "little") + 256
    p = 6 if fhd == 0x20 else 7
    out = bytearray()
    rep = [1, 4, 8]
    blocks = []
    while True:
        bh = int.from_bytes(frame[p:p + 3], "little")
        last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
        p += 3
        blk = dict(type=("raw", "rle", "compressed", "reserved")[btype], start=len(out), last=bool(last))
        if btype == 0:
            out += frame[p:p + bsize]
            p += bsize
        elif btype == 1:
            out += frame[p:p + 1] * bsize
            p += 1
        else:
            assert btype == 2
            body = frame[p:p + bsize]
            ls = _parse_literals(body, blk)
            _parse_sequences(body[ls:], blk, rep)
            blk.update(lit_section=ls, seq_section=bsize - ls)
            lits, lp = blk["literals"], 0
            for s in blk["sequences"]:
                out += lits[lp:lp + s["ll"]]
                lp += s["ll"]
                assert 1 <= s["off"] <= len(out), "offset past the start of the frame"
                for _ in range(s["ml"]):
                    out.append(out[-s["off"]])
            out += lits[lp:]
            p += bsize
        blk.update(end=len(out), size=bsize)
        blocks.append(blk)
        if last:
            break
    assert p == len(frame), "bytes after the last block"
    return dict(n=n, header=6 if fhd == 0x20 else 7, blocks=blocks, content=bytes(out))
