"""Hand-built and mutated Zstandard (RFC 8878) streams for the Zstd decoder tests, and libzstd as their oracle.

  (a) describe(stream): a header parser -- frames, block types, literal modes and stream counts, the
      Number_of_Sequences form, the LL / OF / ML symbol-compression modes, and (decoding the sequences) the repeat-offset
      cases used.
  (b) assembly helpers: frame headers with every FCS field size, single-segment and windowed frames, raw / RLE /
      zero-size blocks, skippable and concatenated frames, libzstd's compressed blocks re-wrapped under other headers.
  (c) one mutator per rejection rule, at parsed field offsets (mutations()).
  (d) xxh64(): the content checksum, pinned to the checksums libzstd writes.
Every verdict used by the tests is libzstd's (LibZstd.expect), never reasoned out from the RFC alone."""
import ctypes as C
import random
import struct

MAGIC = 0xFD2FB528
BLOCK_MAX = 1 << 17

# ---------------------------------------------------------------------------------------------------------------------
# libzstd (1.5.x) through ctypes
# ---------------------------------------------------------------------------------------------------------------------
C_LEVEL, C_WINDOWLOG, C_STRATEGY, C_CONTENTSIZE, C_CHECKSUM = 100, 101, 107, 200, 201


class LibZstd:
    def __init__(self):
        self.lib = C.CDLL("libzstd.so.1")
        L = self.lib
        L.ZSTD_versionNumber.restype = C.c_uint
        L.ZSTD_compressBound.restype = C.c_size_t
        L.ZSTD_compressBound.argtypes = [C.c_size_t]
        L.ZSTD_createCCtx.restype = C.c_void_p
        L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
        L.ZSTD_CCtx_setParameter.restype = C.c_size_t
        L.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ZSTD_compress2.restype = C.c_size_t
        L.ZSTD_compress2.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        L.ZSTD_decompress.restype = C.c_size_t
        L.ZSTD_decompress.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        L.ZSTD_isError.restype = C.c_uint
        L.ZSTD_isError.argtypes = [C.c_size_t]
        L.ZSTD_getErrorName.restype = C.c_char_p
        L.ZSTD_getErrorName.argtypes = [C.c_size_t]
        self.version = L.ZSTD_versionNumber()

    def compress(self, data: bytes, level=3, strategy=None, window_log=None, checksum=False, content_size=True):
        L = self.lib
        cctx = L.ZSTD_createCCtx()
        try:
            for p, v in ((C_LEVEL, level), (C_STRATEGY, strategy), (C_WINDOWLOG, window_log),
                         (C_CHECKSUM, int(checksum)), (C_CONTENTSIZE, int(content_size))):
                if v is not None:
                    r = L.ZSTD_CCtx_setParameter(cctx, p, v)
                    assert not L.ZSTD_isError(r), (p, v, L.ZSTD_getErrorName(r))
            cap = L.ZSTD_compressBound(len(data))
            out = C.create_string_buffer(cap)
            n = L.ZSTD_compress2(cctx, out, cap, data, len(data))
            assert not L.ZSTD_isError(n), L.ZSTD_getErrorName(n)
            return out.raw[:n]
        finally:
            L.ZSTD_freeCCtx(cctx)

    def expect(self, stream: bytes, cap: int):
        """libzstd's verdict on one chunk: ("ok", bytes), ("checksum", None) or ("bad", None)."""
        out = C.create_string_buffer(max(cap, 1))
        n = self.lib.ZSTD_decompress(out, cap, stream, len(stream))
        if self.lib.ZSTD_isError(n):
            name = self.lib.ZSTD_getErrorName(n).decode()
            return ("checksum", None) if "checksum" in name.lower() else ("bad", None)
        return "ok", out.raw[:n]


# The verdicts the decoder follows are libzstd 1.5.5's (reserved modes bits ignored, 4-stream literal ends not
# checked, raw blocks over 128 KB accepted); later releases are stricter in places, so the tests pin the version.
LIBZSTD_VERSION = 10505


def libzstd_or_none():
    """libzstd 1.5.5, or None when libzstd.so.1 is missing or another release."""
    try:
        z = LibZstd()
    except OSError:
        return None
    return z if z.version == LIBZSTD_VERSION else None


# ---------------------------------------------------------------------------------------------------------------------
# (d) XXH64
# ---------------------------------------------------------------------------------------------------------------------
_P1, _P2, _P3, _P4, _P5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63,
                           0x27D4EB2F165667C5)
_M = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, v):
    return (_rotl((acc + v * _P2) & _M, 31) * _P1) & _M


def xxh64(data: bytes, seed=0) -> int:
    n = len(data)
    i = 0
    if n >= 32:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed, (seed - _P1) & _M]
        while i + 32 <= n:
            for k in range(4):
                v[k] = _round(v[k], struct.unpack_from("<Q", data, i + 8 * k)[0])
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for x in v:
            h = ((h ^ _round(0, x)) * _P1 + _P4) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while i + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", data, i)[0]), 27) * _P1 + _P4) & _M
        i += 8
    if i + 4 <= n:
        h = (_rotl(h ^ ((struct.unpack_from("<I", data, i)[0] * _P1) & _M), 23) * _P2 + _P3) & _M
        i += 4
    while i < n:
        h = (_rotl(h ^ ((data[i] * _P5) & _M), 11) * _P1) & _M
        i += 1
    h ^= h >> 33
    h = (h * _P2) & _M
    h ^= h >> 29
    h = (h * _P3) & _M
    h ^= h >> 32
    return h


# ---------------------------------------------------------------------------------------------------------------------
# (a) parser
# ---------------------------------------------------------------------------------------------------------------------
class _BackBits:
    """Backward bit reader of an FSE / Huffman stream (sentinel in the last byte; bits before the start read as 0)."""

    def __init__(self, b: bytes):
        assert b and b[-1], "stream without a sentinel"
        self.v = int.from_bytes(b, "little")
        self.pos = 8 * len(b) - 1 - (8 - b[-1].bit_length()) - 0    # bits left above the sentinel
        self.pos = 8 * (len(b) - 1) + b[-1].bit_length() - 1

    def read(self, n):
        if n == 0:
            return 0
        self.pos -= n
        if self.pos >= 0:
            return (self.v >> self.pos) & ((1 << n) - 1)
        return ((self.v << -self.pos) & ((1 << n) - 1)) if self.pos > -n else 0


def _read_ncount(b: bytes, max_sv: int):
    """FSE table description -> (norm counts, accuracy log, header bytes) for well-formed headers."""
    v = int.from_bytes(b[:64] + bytes(8), "little")
    bit = 0

    def get(n):
        nonlocal bit
        r = (v >> bit) & ((1 << n) - 1)
        bit += n
        return r
    log = get(4) + 5
    remaining = (1 << log) + 1
    threshold = 1 << log
    nb = log + 1
    norm = []
    while remaining > 1 and len(norm) <= max_sv:
        mx = 2 * threshold - 1 - remaining
        low = (v >> bit) & (threshold - 1)
        if low < mx:
            count = low
            bit += nb - 1
        else:
            count = (v >> bit) & (2 * threshold - 1)
            if count >= threshold:
                count -= mx
            bit += nb
        count -= 1
        remaining -= abs(count)
        norm.append(count)
        if count == 0:
            while True:
                rep = get(2)
                norm.extend([0] * rep)
                if rep != 3:
                    break
        while remaining < threshold:
            nb -= 1
            threshold >>= 1
    return norm, log, (bit + 7) // 8


def _fse_table(norm, log):
    size = 1 << log
    high = size - 1
    sym = [0] * size
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
    step = (size >> 1) + (size >> 3) + 3
    pos = 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    nxt = [1 if c == -1 else max(c, 0) for c in norm]
    tab = []
    for u in range(size):
        s = sym[u]
        ns = nxt[s]
        nxt[s] += 1
        nbits = log - (ns.bit_length() - 1)
        tab.append((s, nbits, (ns << nbits) - size))
    return tab


_LL_DEF = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1,
           -1, -1]
_ML_DEF = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
_OF_DEF = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
_LL_EXTRA = [(16, 1), (18, 1), (20, 1), (22, 1), (24, 2), (28, 2), (32, 3), (40, 3), (48, 4)] + \
            [(1 << b, b) for b in range(6, 17)]
_ML_EXTRA = [(35, 1), (37, 1), (39, 1), (41, 1), (43, 2), (47, 2), (51, 3), (59, 3), (67, 4), (83, 4), (99, 5)] + \
            [((1 << b) + 3, b) for b in range(7, 17)]


def _ll_code(c):
    return (c, 0) if c < 16 else _LL_EXTRA[c - 16]


def _ml_code(c):
    return (c + 3, 0) if c < 32 else _ML_EXTRA[c - 32]


MODES = ("predefined", "rle", "fse", "repeat")
LIT_MODES = ("raw", "rle", "huffman", "treeless")


def describe(stream: bytes):
    """Parse a well-formed chunk.  Returns a list of frames; each frame is a dict with its header fields and offsets
    and a list of block dicts (type, offsets, literal mode / streams, sequence count form, the three modes, and the
    repeat-offset cases seen: (repeat index 1..3, ll == 0))."""
    frames = []
    pos = 0
    while pos < len(stream):
        magic = struct.unpack_from("<I", stream, pos)[0]
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            size = struct.unpack_from("<I", stream, pos + 4)[0]
            frames.append({"skippable": True, "offset": pos, "size": 8 + size})
            pos += 8 + size
            continue
        assert magic == MAGIC, hex(magic)
        fhd = stream[pos + 4]
        fcs_flag, single, checksum, did_flag = fhd >> 6, (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
        did_size = [0, 1, 2, 4][did_flag]
        fcs_size = [single, 2, 4, 8][fcs_flag]
        fr = {"skippable": False, "offset": pos, "fhd_offset": pos + 4, "single": bool(single),
              "checksum": bool(checksum), "fcs_size": fcs_size, "did_size": did_size, "blocks": []}
        p = pos + 5 + (0 if single else 1)
        fr["did_offset"] = p
        p += did_size
        fr["fcs_offset"] = p
        fcs = int.from_bytes(stream[p:p + fcs_size], "little") if fcs_size else None
        if fcs_size == 2:
            fcs += 256
        fr["fcs"] = fcs
        p += fcs_size
        st = {"rep": [1, 4, 8], "tabs": [None, None, None], "huf": False}
        while True:
            bh = int.from_bytes(stream[p:p + 3], "little")
            last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
            blk = {"offset": p, "type": ("raw", "rle", "compressed", "reserved")[btype], "size": bsize,
                   "last": bool(last)}
            p += 3
            if btype == 2:
                _describe_block(stream[p:p + bsize], blk, st)
            fr["blocks"].append(blk)
            p += 1 if btype == 1 else bsize
            if last:
                break
        if checksum:
            fr["checksum_offset"] = p
            p += 4
        fr["end"] = p
        frames.append(fr)
        pos = p
    return frames


def _describe_block(b: bytes, blk, st):
    b0 = b[0]
    lt, lhl = b0 & 3, (b0 >> 2) & 3
    blk["lit_mode"] = LIT_MODES[lt]
    if lt < 2:
        lh = {0: 1, 2: 1, 1: 2, 3: 3}[lhl]
        lit = int.from_bytes(b[:lh], "little") >> (3 if lh == 1 else 4)
        sec = lh + (lit if lt == 0 else 1)
        blk["lit_streams"] = 0
    else:
        lh = {0: 3, 1: 3, 2: 4, 3: 5}[lhl]
        hdr = int.from_bytes(b[:lh], "little")
        lit = (hdr >> 4) & ((1 << [10, 10, 14, 18][lhl]) - 1)
        csz = hdr >> [14, 14, 18, 22][lhl]
        blk["lit_streams"] = 1 if lhl == 0 else 4
        sec = lh + csz
        if lt == 2:
            blk["huf_offset"] = lh
    blk["lit_size"] = lit
    blk["seq_offset"] = sec
    sp = sec
    nb = b[sp]
    if nb < 128:
        nseq, form = nb, 1
        sp += 1
    elif nb < 255:
        nseq, form = ((nb - 128) << 8) + b[sp + 1], 2
        sp += 2
    else:
        nseq, form = b[sp + 1] + (b[sp + 2] << 8) + 0x7F00, 3
        sp += 3
    blk["nseq"], blk["nseq_form"] = nseq, form
    blk["reps"] = set()
    if form == 1 and not nseq:
        return
    blk["modes_offset"] = sp
    modes = b[sp]
    sp += 1
    kinds = [(modes >> 6) & 3, (modes >> 4) & 3, (modes >> 2) & 3]
    blk["modes"] = tuple(MODES[k] for k in kinds)
    maxes, defs, dlogs = (35, 31, 52), (_LL_DEF, _OF_DEF, _ML_DEF), (6, 5, 6)
    for i, k in enumerate(kinds):
        if k == 0:
            st["tabs"][i] = (_fse_table(defs[i], dlogs[i]), dlogs[i])
        elif k == 1:
            st["tabs"][i] = ([(b[sp], 0, 0)], 0)
            sp += 1
        elif k == 2:
            norm, log, hs = _read_ncount(b[sp:], maxes[i])
            blk.setdefault("fse_offsets", {})[("LL", "OF", "ML")[i]] = sp
            st["tabs"][i] = (_fse_table(norm, log), log)
            sp += hs
    blk["bitstream_offset"] = sp
    if not nseq:                       # a 2-byte zero count: tables built, no bitstream
        return
    br = _BackBits(b[sp:])
    (tll, lll), (tof, lof), (tml, lml) = st["tabs"]
    sll, sof, sml = br.read(lll), br.read(lof), br.read(lml)
    rep = st["rep"]
    for k in range(nseq):
        llc, ofc, mlc = tll[sll][0], tof[sof][0], tml[sml][0]
        ofv = (1 << ofc) + br.read(ofc)
        mlb, mlx = _ml_code(mlc)
        ml = mlb + br.read(mlx)
        llb, llx = _ll_code(llc)
        ll = llb + br.read(llx)
        if ofv > 3:
            rep[:] = [ofv - 3, rep[0], rep[1]]
        else:
            idx = ofv + (ll == 0)
            blk["reps"].add((ofv, ll == 0))
            if idx == 1:
                pass
            elif idx == 2:
                rep[:] = [rep[1], rep[0], rep[2]]
            elif idx == 3:
                rep[:] = [rep[2], rep[0], rep[1]]
            else:
                rep[:] = [max(rep[0] - 1, 1), rep[0], rep[1]]
        if k + 1 < nseq:
            e = tll[sll]
            sll = e[2] + br.read(e[1])
            e = tml[sml]
            sml = e[2] + br.read(e[1])
            e = tof[sof]
            sof = e[2] + br.read(e[1])


def features(stream: bytes):
    """The coverage features of one well-formed chunk (a set of tuples)."""
    out = set()
    for fr in describe(stream):
        if fr["skippable"]:
            out.add(("skippable",))
            continue
        for blk in fr["blocks"]:
            out.add(("block", blk["type"]))
            if blk["type"] != "compressed":
                continue
            out.add(("lit", blk["lit_mode"], blk["lit_streams"]))
            out.add(("nseq_form", blk["nseq_form"]))
            if blk["nseq"] == 0 and blk["nseq_form"] == 2:
                out.add(("nseq_zero_2byte",))
            if blk["nseq"] >= 0x7F00:
                out.add(("nseq_ge_7f00",))
            for name, m in zip(("LL", "OF", "ML"), blk.get("modes", ())):
                out.add(("mode", name, m))
            for r, ll0 in blk["reps"]:
                out.add(("rep", r, ll0))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# (b) assembly
# ---------------------------------------------------------------------------------------------------------------------
def block_header(btype: int, size: int, last: bool) -> bytes:
    return (int(last) | (btype << 1) | (size << 3)).to_bytes(3, "little")


def raw_block(data: bytes, last=True) -> bytes:
    return block_header(0, len(data), last) + data


def rle_block(byte: int, n: int, last=True) -> bytes:
    return block_header(1, n, last) + bytes([byte])


def frame_header(content_size=None, fcs_bytes=None, single=False, window_log=17, checksum=False, dict_id=None,
                 did_bytes=0) -> bytes:
    """fcs_bytes: 0 (absent), 1 (single-segment only), 2 (+256 bias), 4, 8; default: the smallest that fits."""
    if content_size is None:
        fcs_bytes = 0 if not single else fcs_bytes
    elif fcs_bytes is None:
        fcs_bytes = 1 if single and content_size < 256 else 2 if 256 <= content_size < 65536 + 256 else 4 \
            if content_size < 1 << 32 else 8
    if dict_id is not None and not did_bytes:
        did_bytes = 4
    fcs_flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fcs_bytes]
    assert not (fcs_bytes == 1 and not single)
    did_flag = {0: 0, 1: 1, 2: 2, 4: 3}[did_bytes]
    fhd = (fcs_flag << 6) | (int(single) << 5) | (int(checksum) << 2) | did_flag
    h = struct.pack("<IB", MAGIC, fhd)
    if not single:
        h += bytes([(window_log - 10) << 3])
    if did_bytes:
        h += (dict_id or 0).to_bytes(did_bytes, "little")
    if fcs_bytes:
        v = content_size - 256 if fcs_bytes == 2 else content_size
        h += v.to_bytes(fcs_bytes, "little")
    return h


def frame(blocks: bytes, content: bytes, checksum=False, **kw) -> bytes:
    """A frame around already-assembled blocks whose decoded bytes are `content`."""
    kw.setdefault("content_size", len(content))
    out = frame_header(checksum=checksum, **kw) + blocks
    if checksum:
        out += struct.pack("<I", xxh64(content) & 0xFFFFFFFF)
    return out


def skippable(payload: bytes, nibble=0) -> bytes:
    return struct.pack("<II", 0x184D2A50 | nibble, len(payload)) + payload


def blocks_of(stream: bytes) -> bytes:
    """The block bytes of a single-frame libzstd stream (to re-wrap them under another frame header)."""
    fr = describe(stream)[0]
    return stream[fr["blocks"][0]["offset"]:fr["end"] - (4 if fr["checksum"] else 0)]


def _nseq_bytes(n: int) -> bytes:
    if n < 128:
        return bytes([n])
    if n < 0x7F00:
        return bytes([(n >> 8) + 128, n & 255])
    return bytes([255]) + (n - 0x7F00).to_bytes(2, "little")


def rle_sequences_block(lit_section: bytes, lits: bytes, n: int, ll_sym: int, of_sym: int, ml_sym: int,
                        bits: bytes, history: bytes, last=True, repeat=False):
    """A compressed block whose LL / OF / ML tables are all RLE (one symbol each), so its sequence bitstream holds
    only extra bits: `bits` (sentinel included).  repeat: the block's modes byte says Repeat for all three tables
    (the symbols are those of the tables an earlier block left).  Returns (block, decoded bytes) given the frame's
    earlier bytes."""
    tables = bytes([0xFC]) if repeat else bytes([0x54, ll_sym, of_sym, ml_sym])
    body = lit_section + _nseq_bytes(n) + tables + bits
    br = _BackBits(bits)
    out = bytearray(history)
    rep = [1, 4, 8]
    lp = 0
    for _ in range(n):
        ofv = (1 << of_sym) + br.read(of_sym)
        mlb, mlx = _ml_code(ml_sym)
        ml = mlb + br.read(mlx)
        llb, llx = _ll_code(ll_sym)
        ll = llb + br.read(llx)
        idx = ofv + (ll == 0) if ofv <= 3 else 0
        if idx == 0:
            off = ofv - 3
            rep[:] = [off, rep[0], rep[1]]
        elif idx == 1:
            off = rep[0]
        elif idx == 2:
            off = rep[1]
            rep[:] = [rep[1], rep[0], rep[2]]
        elif idx == 3:
            off = rep[2]
            rep[:] = [rep[2], rep[0], rep[1]]
        else:
            off = max(rep[0] - 1, 1)
            rep[:] = [off, rep[0], rep[1]]
        out += lits[lp:lp + ll]
        lp += ll
        for _ in range(ml):
            out.append(out[-off])
    out += lits[lp:]
    return block_header(2, len(body), last) + body, bytes(out[len(history):])


def rle_table_streams():
    """Hand-built blocks the libzstd corpus does not produce: a block of 0x7F05 sequences (the 3-byte
    Number_of_Sequences form), RLE literals, and repeat offset 3 with ll == 0 (rep1 - 1)."""
    hist = b"abcdefgh"
    out = []
    # 0x7F05 sequences (ll 0, ml 3, offset code 0: repeat 2 swapped with repeat 1), no extra bits
    blk, dec = rle_sequences_block(b"\x00", b"", 0x7F05, 0, 0, 0, b"\x01", hist)
    out.append(("rle_tables_0x7f05_sequences", frame(raw_block(hist, False) + blk, hist + dec, checksum=True),
                hist + dec))
    # RLE literals 'z' x 5 after 4 sequences of offset code 1 with extra bit 1 and ll 0: rep1 - 1
    blk, dec = rle_sequences_block(bytes([(5 << 3) | 1]) + b"z", b"zzzzz", 4, 0, 1, 2, b"\x1f", hist)
    out.append(("rle_literals_rep1_minus_1", frame(raw_block(hist, False) + blk, hist + dec), hist + dec))
    # ll > 0 with RLE literals: LL symbol 1, 3 sequences
    blk, dec = rle_sequences_block(bytes([(6 << 3) | 1]) + b"q", b"qqqqqq", 3, 1, 2, 1, b"\x40", hist)
    out.append(("rle_literals_ll1", frame(raw_block(hist, False) + blk, hist + dec), hist + dec))
    return out


ZERO_COUNT_2BYTE = b"\x80\x00"         # Number_of_Sequences = 0 in the 2-byte form: the modes byte still follows


def zero_count_block(tables: bytes, lits=b"", last=True, trailer=b"") -> bytes:
    """A compressed block with raw literals and a 2-byte zero sequence count followed by `tables` (the modes byte and
    table descriptions) and `trailer` (bytes libzstd ignores)."""
    body = bytes([len(lits) << 3]) + lits + ZERO_COUNT_2BYTE + tables + trailer
    return block_header(2, len(body), last) + body


def zero_count_streams():
    """Valid chunks with a 2-byte zero sequence count: its tables are built and a later Repeat block uses them."""
    hist = b"abcdefgh"
    out = []
    blk = zero_count_block(bytes([0x54, 0, 2, 1]), b"abc", trailer=b"\x17\x00")
    out.append(("zero_count_2byte_tables_trailer", frame(raw_block(hist, False) + blk, hist + b"abc"), hist + b"abc"))
    # block A: RLE tables (ll 2, offset 1, ml 3); block B: zero count, RLE tables (ll 0, offset 1, ml 4);
    # block C: Repeat tables -> B's tables, not A's
    a, da = rle_sequences_block(bytes([2 << 3]) + b"xy", b"xy", 1, 2, 2, 0, b"\x04", hist, last=False)
    b = zero_count_block(bytes([0x54, 0, 2, 1]), last=False)
    c, dc = rle_sequences_block(b"\x00", b"", 1, 0, 2, 1, b"\x04", hist + da, repeat=True)
    want = hist + da + dc
    out.append(("zero_count_tables_then_repeat", frame(raw_block(hist, False) + a + b + c, want), want))
    return out


def zero_count_mutations():
    """(rule, stream, libzstd's verdict) for malformed 2-byte zero sequence counts."""
    hist = b"abcdefgh"
    pre = raw_block(hist, False)
    out = [("zero_count_2byte_without_modes", frame(pre + zero_count_block(b"", b"abc"), hist + b"abc"), "bad"),
           ("zero_count_2byte_repeat_in_first_block", frame(pre + zero_count_block(b"\xFC", b"abc"), hist + b"abc"),
            "bad"),
           ("zero_count_2byte_rle_ll_symbol_over_35",
            frame(pre + zero_count_block(bytes([0x54, 0xFF, 0, 0]), b"abc"), hist + b"abc"), "bad")]
    # a zero-count block does not allow Repeat in the next block by itself: libzstd enables Repeat only once a block
    # has decoded sequences
    b = zero_count_block(bytes([0x54, 0, 2, 1]), last=False)
    c, dc = rle_sequences_block(b"\x00", b"", 1, 0, 2, 1, b"\x04", hist, repeat=True)
    out.append(("zero_count_tables_do_not_enable_repeat", frame(pre + b + c, hist + dc), "bad"))
    return out


def valid_streams(zs: LibZstd, inputs):
    """(name, stream, intended bytes) for the hand-built valid chunks."""
    text, rnd = inputs["text"], inputs["random_777"]
    out = [("empty_chunk", b"", b""),
           ("empty_frame_raw", frame(raw_block(b""), b""), b""),
           ("empty_frame_single", frame(raw_block(b""), b"", single=True), b""),
           ("raw_single_fcs1", frame(raw_block(rnd[:200]), rnd[:200], single=True), rnd[:200]),
           ("raw_fcs2_bias", frame(raw_block(rnd[:300]), rnd[:300]), rnd[:300]),
           ("raw_fcs2_low_edge", frame(raw_block(text[:256]), text[:256]), text[:256]),
           ("raw_fcs4", frame(raw_block(rnd), rnd, fcs_bytes=4), rnd),
           ("raw_fcs8", frame(raw_block(rnd), rnd, fcs_bytes=8), rnd),
           ("raw_no_fcs", frame(raw_block(rnd), rnd, content_size=None), rnd),
           ("raw_checksum", frame(raw_block(rnd), rnd, checksum=True), rnd),
           ("rle_block", frame(rle_block(7, 5000), bytes([7]) * 5000, checksum=True), bytes([7]) * 5000),
           ("zero_size_blocks", frame(raw_block(b"", False) + rle_block(1, 0, False) + raw_block(b"ab"), b"ab"),
            b"ab"),
           ("raw_rle_mix", frame(raw_block(text[:1000], False) + rle_block(0, 3000, False) + raw_block(rnd),
                                 text[:1000] + bytes(3000) + rnd, checksum=True), text[:1000] + bytes(3000) + rnd),
           ("dict_id_zero", frame(raw_block(rnd), rnd, dict_id=0, did_bytes=1), rnd),
           ("window_10", frame(raw_block(rnd), rnd, window_log=10), rnd)]
    c1 = zs.compress(text, 3, checksum=True)
    c2 = zs.compress(rnd + text, 19)
    out += [("two_frames", c1 + c2, text + rnd + text),
            ("skippable_then_frame", skippable(b"metadata", 5) + c1, text),
            ("frame_skippable_frame", c1 + skippable(b"", 15) + c1, text + text),
            ("only_skippable", skippable(b"xyz"), b"")]
    out += rle_table_streams() + zero_count_streams()
    # libzstd's compressed blocks under other frame headers
    for name, data in (("text", text), ("price_walk", inputs["price_walk"]), ("lowentropy", inputs["lowentropy"])):
        body = blocks_of(zs.compress(data, 3, content_size=False))
        out += [(f"rewrap_{name}_single", frame(body, data, single=True, checksum=True), data),
                (f"rewrap_{name}_fcs8", frame(body, data, fcs_bytes=8), data),
                (f"rewrap_{name}_nofcs_w31", frame(body, data, content_size=None, window_log=31), data)]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# (c) mutators: (rule, stream, libzstd's verdict)
# ---------------------------------------------------------------------------------------------------------------------
def _set(s: bytes, off: int, val: bytes) -> bytes:
    return s[:off] + val + s[off + len(val):]


def mutations(zs: LibZstd, inputs):
    text, pw = inputs["text"], inputs["price_walk"]
    base = zs.compress(pw, 3, checksum=True)          # FSE-compressed tables, Huffman literals
    fr = describe(base)[0]
    blk = fr["blocks"][0]
    bo = blk["offset"] + 3
    out = []
    fhd = fr["fhd_offset"]
    out.append(("header_reserved_bit", _set(base, fhd, bytes([base[fhd] | 0x08])), "bad"))
    out.append(("dictionary_id", frame(raw_block(text[:100]), text[:100], dict_id=7), "bad"))
    out.append(("window_over_2_31", frame(raw_block(text[:100]), text[:100], window_log=32), "bad"))
    out.append(("reserved_block_type", _set(base, blk["offset"], bytes([base[blk["offset"]] | 0x06])), "bad"))
    big = bytes(BLOCK_MAX + 1)
    out.append(("compressed_block_over_max", frame(block_header(2, BLOCK_MAX, True) + bytes(BLOCK_MAX), bytes(0),
                                                   content_size=None), "bad"))
    out.append(("raw_block_over_max", frame(raw_block(big), big), zs.expect(frame(raw_block(big), big),
                                                                              len(big))[0]))
    out.append(("block_past_input", base[:blk["offset"] + 3 + 10], "bad"))
    # FSE table description: accuracy log over the limit, counts that do not sum
    if "fse_offsets" in blk:
        k, o = next(iter(blk["fse_offsets"].items()))
        a = bo + o
        out.append((f"fse_log_over_limit_{k}", _set(base, a, bytes([(base[a] & 0xF0) | 0x0F])), "bad"))
        out.append((f"fse_counts_do_not_sum_{k}", _set(base, a, bytes([base[a] ^ 0x10])), "bad"))
    # Huffman tree description (direct weights): weights that do not complete a power of two, weight over 12
    if "huf_offset" in blk:
        h = bo + blk["huf_offset"]
        w_bad = bytes([128 + 4, 0x11, 0x13])       # 5 weights 1,1,1,3,? -> 2^0.5 sums
        out.append(("huffman_weights_incomplete", _set(base, h, w_bad), "bad"))
        out.append(("huffman_weight_over_12", _set(base, h, bytes([128 + 2, 0xD1])), "bad"))
    # jump table past the end (4-stream literals), stream not consumed exactly (sentinel moved)
    nb = blk["offset"] + 3 + blk["bitstream_offset"]
    end = nb + (blk["size"] - blk["bitstream_offset"]) - 1
    out.append(("sequence_stream_sentinel_moved", _set(base, end, bytes([base[end] | 0x80 if base[end] < 0x80
                                                                          else base[end] >> 1])),
                zs.expect(_set(base, end, bytes([base[end] | 0x80 if base[end] < 0x80 else base[end] >> 1])),
                          len(pw))[0]))
    # libzstd 1.5.5 does not check the reserved bits of the modes byte
    out.append(("modes_reserved_bits", _set(base, bo + blk["modes_offset"],
                                            bytes([base[bo + blk["modes_offset"]] | 1])), "ok"))
    out.append(("repeat_mode_in_first_block", _set(base, bo + blk["modes_offset"],
                                                   bytes([base[bo + blk["modes_offset"]] | 0xFC & 0xC0])), "bad"))
    b0 = base[bo]
    if b0 & 3 == 2:
        out.append(("treeless_in_first_block", _set(base, bo, bytes([b0 | 3])), "bad"))
    # an offset past history: a later block moved to the first block of a new frame
    rnd = inputs["random_64k"]
    rng = random.Random(1)
    tail = bytes(rng.randrange(256) for _ in range(70000))
    multi = zs.compress(rnd + tail + rnd[:20000], 3)  # block 2: literals, then a match 134 KB back
    b2 = describe(multi)[0]["blocks"][1]
    assert b2["type"] == "compressed" and b2["nseq"] > 0
    body = block_header(2, b2["size"], True) + multi[b2["offset"] + 3:b2["offset"] + 3 + b2["size"]]
    out.append(("offset_past_history_transplant", frame_header(None) + body, "bad"))
    out.append(("fcs_mismatch", _set(base, fr["fcs_offset"], bytes([base[fr["fcs_offset"]] ^ 1])), "bad"))
    cs = fr["checksum_offset"]
    out.append(("checksum_flipped", _set(base, cs, bytes([base[cs] ^ 0x40])), "checksum"))
    out.append(("checksum_truncated", base[:-2], "checksum"))
    out.append(("truncated_in_block", base[:len(base) // 2], "bad"))
    out.append(("trailing_byte", base + b"\x00", "bad"))
    out.append(("truncated_header", base[:7], "bad"))
    out.append(("skippable_truncated", skippable(b"abcdef")[:-1], "bad"))
    return out + zero_count_mutations()


def _huffman_tree(b: bytes):
    """Huffman tree description at b[0] -> (decode table of (symbol, nbBits), table log, description bytes), or None
    when libzstd's HUF_readStats rules reject it."""
    if not b:
        return None
    isize = b[0]
    if isize >= 128:
        n = isize - 127
        size = 1 + (n + 1) // 2
        if size > len(b):
            return None
        w = [(b[1 + i // 2] >> 4) if i % 2 == 0 else (b[1 + i // 2] & 15) for i in range(n)]
    else:
        size = 1 + isize
        if size > len(b):
            return None
        norm, flog, hs = _read_ncount(b[1:size], 255)
        if flog > 6 or hs >= isize or sum(abs(c) for c in norm) != 1 << flog:
            return None
        tab = _fse_table(norm, flog)
        stream = b[1 + hs:size]
        if not stream[-1]:
            return None
        br = _BackBits(stream)
        st = [br.read(flog), br.read(flog)]
        w, k = [], 0
        while True:                     # two interleaved states; after an update reads past the start, one more
            if len(w) > 253:
                return None
            sym, nb, base = tab[st[k]]
            w.append(sym)
            st[k] = base + br.read(nb)
            if br.pos < 0:
                w.append(tab[st[1 - k]][0])
                break
            k ^= 1
    if any(x > 12 for x in w):
        return None
    total = sum(1 << (x - 1) for x in w if x)
    if not total or total.bit_length() > 12:
        return None
    log = total.bit_length()
    rest = (1 << log) - total
    if rest & (rest - 1):
        return None
    w.append(rest.bit_length())
    ones = w.count(1)
    if ones < 2 or ones & 1:
        return None
    table = []
    for wt in range(1, log + 1):
        for sym, x in enumerate(w):
            if x == wt:
                table += [(sym, log + 1 - wt)] * (1 << (wt - 1))
    return table, log, size


def _huffman_stream_ends_exactly(stream: bytes, table, log: int, n: int) -> bool:
    """Decode n symbols; True when the stream is then consumed exactly to its sentinel bit."""
    if not stream or not stream[-1]:
        return False
    br = _BackBits(stream)
    for _ in range(n):
        _, nb = table[br.read(log)]
        br.pos += log - nb
        if br.pos < 0:
            return False
    return br.pos == 0


def four_stream_end_mismatch(s: bytes) -> bool:
    """True when a block of chunk s has 4-stream Huffman literals whose header, tree and jump table are valid but one
    of whose four streams does not end exactly on its first bit after its quarter of the literals.  This decoder
    rejects such a block; libzstd 1.5.5 decodes 4-stream literals with a fast Huffman loop that checks each stream
    fills its quarter but not where it ends, so it may decode the block (to wrong bytes, usually caught by the content
    checksum or size).  This is the one place the two verdicts may differ."""
    try:
        pos = 0
        while pos < len(s):
            magic = struct.unpack_from("<I", s, pos)[0]
            if magic & 0xFFFFFFF0 == 0x184D2A50:
                pos += 8 + struct.unpack_from("<I", s, pos + 4)[0]
                continue
            if magic != MAGIC:
                return False
            fhd = s[pos + 4]
            single = (fhd >> 5) & 1
            p = pos + 5 + (1 - single) + [0, 1, 2, 4][fhd & 3] + [single, 2, 4, 8][fhd >> 6]
            huf = None
            while True:
                bh = int.from_bytes(s[p:p + 3], "little")
                if len(s) - p < 3:
                    return False
                last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
                p += 3
                body = s[p:p + (1 if btype == 1 else bsize)]
                if btype == 2 and len(body) == bsize and bsize >= 5 and (body[0] & 3) >= 2:
                    lt, lhl = body[0] & 3, (body[0] >> 2) & 3
                    lh = [3, 3, 4, 5][lhl]
                    hdr = int.from_bytes(body[:lh], "little")
                    lit = (hdr >> 4) & ((1 << [10, 10, 14, 18][lhl]) - 1)
                    csz = hdr >> [14, 14, 18, 22][lhl]
                    sec = body[lh:lh + csz]
                    if len(sec) != csz:
                        return False
                    if lt == 2:
                        huf = _huffman_tree(sec)
                        if huf is None or huf[2] >= csz:
                            return False
                        sec = sec[huf[2]:]
                    elif huf is None:
                        return False
                    if lhl and lit >= 6 and len(sec) >= 10:
                        l1, l2, l3 = struct.unpack_from("<HHH", sec)
                        seg = (lit + 3) // 4
                        if l1 + l2 + l3 + 6 > len(sec) or 3 * seg > lit:
                            return False
                        cuts = [6, 6 + l1, 6 + l1 + l2, 6 + l1 + l2 + l3, len(sec)]
                        for k in range(4):
                            n = seg if k < 3 else lit - 3 * seg
                            if not _huffman_stream_ends_exactly(sec[cuts[k]:cuts[k + 1]], huf[0], huf[1], n):
                                return True
                p += len(body)
                if last:
                    break
            pos = p + (4 if (fhd >> 2) & 1 else 0)
    except (IndexError, struct.error, AssertionError, ValueError):
        return False
    return False


def corrupt(stream: bytes, seed: int) -> bytes:
    """One seeded corruption: bit flips, byte replacements, truncation, extension, or a header-field rewrite."""
    rng = random.Random(seed)
    s = bytearray(stream)
    kind = seed % 5
    if kind == 0 and s:
        for _ in range(rng.randint(1, 3)):
            i = rng.randrange(len(s))
            s[i] ^= 1 << rng.randrange(8)
    elif kind == 1 and s:
        for _ in range(rng.randint(1, 4)):
            s[rng.randrange(len(s))] = rng.randrange(256)
    elif kind == 2:
        del s[rng.randrange(len(s) + 1):]
    elif kind == 3:
        s += bytes(rng.randrange(256) for _ in range(rng.randint(1, 9)))
    elif s:
        # rewrite one parsed header field: the frame header byte, a block header, a literals / sequences header byte
        try:
            fr = describe(stream)[0]
            cands = [fr["fhd_offset"]]
            for b in fr["blocks"]:
                cands += [b["offset"], b["offset"] + 1, b["offset"] + 2]
                if b["type"] == "compressed":
                    cands += [b["offset"] + 3, b["offset"] + 3 + b["seq_offset"]]
                    if "modes_offset" in b:
                        cands.append(b["offset"] + 3 + b["modes_offset"])
            i = rng.choice([c for c in cands if c < len(s)])
        except Exception:
            i = rng.randrange(len(s))
        s[i] = rng.randrange(256)
    return bytes(s)
