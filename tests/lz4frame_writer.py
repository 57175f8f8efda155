"""LZ4 frame-format chunks built by hand, and liblz4's LZ4F_* API as the oracle (tests only).

`LibLZ4F` is a ctypes view of liblz4.so.1's frame API.  `LibLZ4F.verdict(chunk, cap)` states what the library's
LZ4 frame decoder must return for a chunk at a capacity: a loop of LZ4F_decompress calls over zero or more frames,
restarting after each frame end, decides the verdict, and the status follows include/nvcomp/lz4frame.h.

`frame(...)` writes one frame from its parts (every FLG / BD field can be set, wrong ones included), `corpus()` the
hand-built frames and one mutated frame per rejection rule.  Every case is pinned to LZ4F_decompress's verdict before
any decoder sees it (tests/test_lz4frame_emu.py)."""
from __future__ import annotations

import ctypes as C
import struct

import lz_writer as W

MAGIC = 0x184D2204
SKIP_MAGIC = 0x184D2A50
LEGACY_MAGIC = 0x184C2102
BLOCK_MAX = {4: 1 << 16, 5: 1 << 18, 6: 1 << 20, 7: 1 << 22}

SUCCESS, CANNOT, BAD_CHECKSUM = 0, 12, 13       # nvcompStatus_t
CHECKSUM_ERRORS = ("ERROR_headerChecksum_invalid", "ERROR_blockChecksum_invalid", "ERROR_contentChecksum_invalid")

_P1, _P2, _P3, _P4, _P5 = 0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D, 0x27D4EB2F, 0x165667B1
_M = 0xFFFFFFFF


def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & _M


def xxh32(data: bytes, seed: int = 0) -> int:
    """XXH32 (the LZ4 frame checksums), restated from the public xxHash specification."""
    n, p = len(data), 0
    if n >= 16:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed & _M, (seed - _P1) & _M]
        while p + 16 <= n:
            for i in range(4):
                w = struct.unpack_from("<I", data, p + 4 * i)[0]
                v[i] = (_rotl((v[i] + w * _P2) & _M, 13) * _P1) & _M
            p += 16
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while p + 4 <= n:
        h = (_rotl((h + struct.unpack_from("<I", data, p)[0] * _P3) & _M, 17) * _P4) & _M
        p += 4
    while p < n:
        h = (_rotl((h + data[p] * _P5) & _M, 11) * _P1) & _M
        p += 1
    h ^= h >> 15
    h = (h * _P2) & _M
    h ^= h >> 13
    h = (h * _P3) & _M
    h ^= h >> 16
    return h


# ---------------------------------------------------------------------------------------------------------------------
# liblz4's frame API
# ---------------------------------------------------------------------------------------------------------------------
class FrameInfo(C.Structure):
    _fields_ = [("blockSizeID", C.c_int), ("blockMode", C.c_int), ("contentChecksumFlag", C.c_int),
                ("frameType", C.c_int), ("contentSize", C.c_ulonglong), ("dictID", C.c_uint),
                ("blockChecksumFlag", C.c_int)]


class Prefs(C.Structure):
    _fields_ = [("frameInfo", FrameInfo), ("compressionLevel", C.c_int), ("autoFlush", C.c_uint),
                ("favorDecSpeed", C.c_uint), ("reserved", C.c_uint * 3)]


class LibLZ4F:
    """liblz4 1.9.4's LZ4F_* frame API (liblz4.so.1, no header needed)."""
    VERSION = 100
    STEP = 1 << 23          # output room per LZ4F_decompress call

    def __init__(self):
        lib = self.lib = C.CDLL("liblz4.so.1")
        vp, sz, szp = C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)
        lib.LZ4F_createDecompressionContext.argtypes = [C.POINTER(vp), C.c_uint]
        lib.LZ4F_createDecompressionContext.restype = sz
        lib.LZ4F_freeDecompressionContext.argtypes = [vp]
        lib.LZ4F_freeDecompressionContext.restype = sz
        lib.LZ4F_decompress.argtypes = [vp, vp, szp, vp, szp, vp]
        lib.LZ4F_decompress.restype = sz
        lib.LZ4F_isError.argtypes = [sz]
        lib.LZ4F_isError.restype = C.c_uint
        lib.LZ4F_getErrorName.argtypes = [sz]
        lib.LZ4F_getErrorName.restype = C.c_char_p
        lib.LZ4F_compressFrameBound.argtypes = [sz, C.POINTER(Prefs)]
        lib.LZ4F_compressFrameBound.restype = sz
        lib.LZ4F_compressFrame.argtypes = [vp, sz, vp, sz, C.POINTER(Prefs)]
        lib.LZ4F_compressFrame.restype = sz
        lib.LZ4_compress_default.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
        lib.LZ4_compressBound.argtypes = [C.c_int]

    # ---- compression
    def compress_frame(self, data: bytes, bsid=4, linked=True, content_sum=False, block_sum=False,
                       content_size=False, level=0) -> bytes:
        p = Prefs()
        p.frameInfo.blockSizeID = bsid
        p.frameInfo.blockMode = 0 if linked else 1
        p.frameInfo.contentChecksumFlag = int(content_sum)
        p.frameInfo.blockChecksumFlag = int(block_sum)
        p.frameInfo.contentSize = len(data) if content_size else 0
        p.compressionLevel = level
        cap = self.lib.LZ4F_compressFrameBound(len(data), C.byref(p))
        out = C.create_string_buffer(cap)
        n = self.lib.LZ4F_compressFrame(out, cap, data, len(data), C.byref(p))
        assert not self.lib.LZ4F_isError(n), self.lib.LZ4F_getErrorName(n)
        return out.raw[:n]

    def compress_block(self, data: bytes) -> bytes:
        cap = self.lib.LZ4_compressBound(len(data))
        out = C.create_string_buffer(max(cap, 1))
        n = self.lib.LZ4_compress_default(data, out, len(data), cap)
        assert n > 0
        return out.raw[:n]

    # ---- decompression
    def _run(self, chunk: bytes, feed: int):
        """Decode the chunk frame after frame with `feed` input bytes per call.  Returns (error, output, at, fstart):
        error is None, "truncated" or liblz4's error name; output what liblz4 produced before the error; at the input
        position after the byte that completed the failing check; fstart the output length where its frame began."""
        ctx = C.c_void_p()
        assert not self.lib.LZ4F_isError(self.lib.LZ4F_createDecompressionContext(C.byref(ctx), self.VERSION))
        try:
            buf = C.create_string_buffer(self.STEP)
            src = C.create_string_buffer(chunk, len(chunk) + 1)
            base = C.addressof(src)
            out, pos, n = bytearray(), 0, len(chunk)
            while pos < n:
                fstart, hint = len(out), 1
                while hint != 0:       # a frame end (hint 0) resets the context: the next frame starts fresh
                    if pos >= n:
                        return "truncated", bytes(out), pos, fstart
                    take = min(feed, n - pos)
                    ssz, dsz = C.c_size_t(take), C.c_size_t(self.STEP)
                    hint = self.lib.LZ4F_decompress(ctx, buf, C.byref(dsz), base + pos, C.byref(ssz), None)
                    if self.lib.LZ4F_isError(hint):
                        return self.lib.LZ4F_getErrorName(hint).decode(), bytes(out), pos + take, fstart
                    out += buf.raw[:dsz.value]
                    pos += ssz.value
            return None, bytes(out), pos, 0
        finally:
            self.lib.LZ4F_freeDecompressionContext(ctx)

    def decode(self, chunk: bytes):
        """(error, output): error None and the decoded chunk, or liblz4's first error and the output before it."""
        err, out, _, _ = self._run(chunk, len(chunk) or 1)
        if err in CHECKSUM_ERRORS:
            # the output produced before the failing check: the same run, one input byte per call
            err, out, _, _ = self._run(chunk, 1)
        return err, out

    def verdict(self, chunk: bytes, cap: int):
        """(status, output) the LZ4 frame decoder must return at capacity cap (include/nvcomp/lz4frame.h)."""
        err, out = self.decode(chunk)
        if err is None:
            return (SUCCESS, out) if len(out) <= cap else (CANNOT, None)
        if err in CHECKSUM_ERRORS and len(out) <= cap:
            return BAD_CHECKSUM, None
        return CANNOT, None

    def size_verdict(self, chunk: bytes) -> int:
        """What the size query returns: the decoded total with every content checksum taken as correct, else 0."""
        chunk = bytearray(chunk)
        while True:
            err, out, at, fstart = self._run(bytes(chunk), len(chunk) or 1)
            if err == "ERROR_contentChecksum_invalid":
                err, out, at, fstart = self._run(bytes(chunk), 1)
            if err != "ERROR_contentChecksum_invalid":
                return len(out) if err is None else 0
            # the failing checksum is chunk[at - 4:at], over the frame output since fstart: put the right one in
            chunk[at - 4:at] = struct.pack("<I", xxh32(out[fstart:]))


# ---------------------------------------------------------------------------------------------------------------------
# hand-built frames
# ---------------------------------------------------------------------------------------------------------------------
def header(*, linked=True, block_sum=False, content_sum=False, content_size=None, dict_id=None, bsid=4, version=1,
           flg_reserved=0, bd_reserved=0, bd_high=0, hc=None, magic=MAGIC) -> bytes:
    flg = (version << 6) | ((0 if linked else 1) << 5) | (int(block_sum) << 4) | (int(content_size is not None) << 3)
    flg |= (int(content_sum) << 2) | (flg_reserved << 1) | int(dict_id is not None)
    bd = (bd_high << 7) | ((bsid & 7) << 4) | bd_reserved
    desc = bytes([flg, bd])
    if content_size is not None:
        desc += struct.pack("<Q", content_size)
    if dict_id is not None:
        desc += struct.pack("<I", dict_id)
    if hc is None:
        hc = (xxh32(desc) >> 8) & 0xFF
    return struct.pack("<I", magic) + desc + bytes([hc])


def block(payload: bytes, *, raw=False, block_sum=False, bad_sum=False) -> bytes:
    b = struct.pack("<I", len(payload) | (0x80000000 if raw else 0)) + payload
    if block_sum:
        b += struct.pack("<I", xxh32(payload) ^ (1 if bad_sum else 0))
    return b


def frame(blocks, content: bytes, *, linked=True, block_sum=False, content_sum=False, content_size=False,
          dict_id=None, bsid=4, bad_content_sum=False, **hdr) -> bytes:
    """blocks: [(payload, raw)], content: the frame's decoded bytes (for the size field and the content checksum)."""
    cs = len(content) if content_size is True else (content_size if content_size is not False else None)
    out = header(linked=linked, block_sum=block_sum, content_sum=content_sum, content_size=cs, dict_id=dict_id,
                 bsid=bsid, **hdr)
    for payload, raw in blocks:
        out += block(payload, raw=raw, block_sum=block_sum)
    out += struct.pack("<I", 0)
    if content_sum:
        out += struct.pack("<I", xxh32(content) ^ (1 if bad_content_sum else 0))
    return out


def skippable(payload: bytes, nibble: int = 0) -> bytes:
    return struct.pack("<II", SKIP_MAGIC | nibble, len(payload)) + payload


def _data(rng_seed: int, n: int) -> bytes:
    import numpy as np
    rng = np.random.default_rng(rng_seed)
    words = rng.integers(0, 40, n // 4 + 1, dtype=np.uint32)
    return (np.repeat(words, 3)[: n // 4 + 1].tobytes() + bytes(range(256)) * (n // 256 + 1))[:n]


def _blocks_of(z: LibLZ4F, data: bytes, bs: int, raw_every: int = 0):
    blocks = []
    for k, i in enumerate(range(0, len(data), bs)):
        part = data[i:i + bs]
        raw = raw_every and k % raw_every == raw_every - 1
        blocks.append((part, True) if raw else (z.compress_block(part), False))
    return blocks


def reach_frames() -> dict[str, bytes]:
    """Matches at exact reaches, from lz_writer sequences: block 1 of 1 000 literal bytes, block 2 a match back."""
    out = {}
    lit = bytes((i * 7 + 3) & 255 for i in range(1000))
    first = W.Lz4().end(lit)
    for name, back, linked in (("to_frame_start", 1000 + 20, True), ("before_frame_start", 1000 + 21, True),
                               ("prev_block_linked", 500, True), ("prev_block_independent", 500, False),
                               ("own_block_independent", 10, False)):
        w = W.Lz4()
        w.out = bytearray(lit if linked else b"")
        w.seq(bytes(20), back, 40).end(bytes(30))
        content = bytes(w.out) if linked else lit + bytes(w.out)
        blocks = [(bytes(first.blk), False), (bytes(w.blk), False)]
        out[f"reach_{name}"] = frame(blocks, content if w.ok else lit, linked=linked, content_size=False)
    return out


def valid_frames(z: LibLZ4F) -> dict[str, bytes]:
    """Every FLG / BD combination, uncompressed blocks, skippable frames, several frames in one chunk."""
    out = {}
    data = _data(1, 150_000)
    for bsid in (4, 5, 6, 7):
        for linked in (True, False):
            for block_sum in (False, True):
                for content_sum in (False, True):
                    for cs in (False, True):
                        for dict_id in (None, 0x12345678):
                            bs = min(BLOCK_MAX[bsid], 40_000)
                            blocks = _blocks_of(z, data[:100_000], bs, raw_every=3 if block_sum else 0)
                            name = f"b{bsid}_{'L' if linked else 'I'}{int(block_sum)}{int(content_sum)}{int(cs)}" \
                                   f"{'d' if dict_id is not None else ''}"
                            out[name] = frame(blocks, data[:100_000], linked=linked, block_sum=block_sum,
                                              content_sum=content_sum, content_size=cs, dict_id=dict_id, bsid=bsid)
    for lvl in (0, 9):
        for linked in (True, False):
            out[f"compressFrame_l{lvl}_{'L' if linked else 'I'}"] = z.compress_frame(data, 4, linked, True, True, True,
                                                                                      lvl)
    out["empty_chunk"] = b""
    out["empty_frame"] = frame([], b"")
    out["empty_frame_sums"] = frame([], b"", block_sum=True, content_sum=True, content_size=True)
    out["uncompressed_only"] = frame([(data[:5000], True), (data[5000:9000], True)], data[:9000], content_sum=True)
    out["uncompressed_max_block"] = frame([(data[:65536], True)], data[:65536])
    out["one_byte_block"] = frame([(b"\x00", False)], b"")
    out["skippable_only"] = skippable(b"meta" * 10, 5)
    out["skippable_empty"] = skippable(b"", 15)
    two = z.compress_frame(data[:3000]) + skippable(b"xyz", 3) + z.compress_frame(data[3000:7000], 5, False, True)
    out["three_frames"] = two
    out["frames_back_to_back"] = frame([(data[:100], True)], data[:100]) + frame([(data[100:300], True)], data[100:300])
    out["content_size_zero_unchecked"] = frame([(data[:100], True)], data[:100], content_size=0)
    out.update(reach_frames())
    return out


def mutants(z: LibLZ4F) -> dict[str, bytes]:
    """One frame per rejection rule (and truncations inside every field)."""
    data = _data(2, 70_000)
    base_blocks = _blocks_of(z, data[:20_000], 8_000)
    good = frame(base_blocks, data[:20_000], block_sum=True, content_sum=True, content_size=True, dict_id=7)
    m = {}
    m["bad_magic"] = struct.pack("<I", MAGIC ^ 0x100) + good[4:]
    m["legacy_magic"] = struct.pack("<I", LEGACY_MAGIC) + good[4:]
    m["version_0"] = frame(base_blocks, data[:20_000], version=0)
    m["version_2"] = frame(base_blocks, data[:20_000], version=2)
    m["flg_reserved"] = frame(base_blocks, data[:20_000], flg_reserved=1)
    m["bd_reserved_low"] = frame(base_blocks, data[:20_000], bd_reserved=1)
    m["bd_reserved_high"] = frame(base_blocks, data[:20_000], bd_high=1)
    for bsid in range(4):
        m[f"bsid_{bsid}"] = frame(base_blocks, data[:20_000], bsid=bsid)
    hdr = header(block_sum=True, content_sum=True, content_size=20_000, dict_id=7)
    m["wrong_hc"] = frame(base_blocks, data[:20_000], block_sum=True, content_sum=True, content_size=True, dict_id=7,
                          hc=hdr[-1] ^ 0x5A)
    m["compressed_over_max"] = header() + struct.pack("<I", 65537) + bytes(65537) + struct.pack("<I", 0)
    m["raw_over_max"] = header() + struct.pack("<I", 65537 | 0x80000000) + bytes(65537) + struct.pack("<I", 0)
    over = W.Lz4().seq(b"a", 1, 65536).end(bytes(10))          # decodes to 65 547 bytes in a 64 KB frame
    m["decoded_over_max"] = frame([(bytes(over.blk), False)], bytes(over.out))
    bs = bytearray(frame(base_blocks, data[:20_000], block_sum=True))
    first_sum = 7 + 4 + len(base_blocks[0][0])
    bs[first_sum] ^= 1
    m["block_sum_flipped"] = bytes(bs)
    raw_bs = bytearray(frame([(data[:3000], True)], data[:3000], block_sum=True))
    raw_bs[7 + 4 + 3000] ^= 1
    m["raw_block_sum_flipped"] = bytes(raw_bs)
    m["content_sum_flipped"] = frame(base_blocks, data[:20_000], content_sum=True, bad_content_sum=True)
    m["content_size_plus1"] = frame(base_blocks, data[:20_000], content_size=20_001)
    m["content_size_minus1"] = frame(base_blocks, data[:20_000], content_size=19_999)
    m["trailing_byte"] = good + b"\x00"
    m["trailing_magic"] = good + struct.pack("<I", MAGIC)
    # truncation inside every field: magic, FLG, BD, content size, dictID, HC, block size, block data, block
    # checksum, EndMark, content checksum
    fields = {"magic": 2, "flg": 4, "bd": 5, "content_size": 9, "dict_id": 16, "hc": 18, "block_size": 21,
              "block_data": 19 + 4 + 100, "block_sum": 19 + 4 + len(base_blocks[0][0]) + 2,
              "endmark": len(good) - 6, "content_sum": len(good) - 2}
    for f, cut in fields.items():
        m[f"truncated_{f}"] = good[:cut]
    m["truncated_skippable"] = skippable(b"abcdef")[:-1]
    return m


def corpus(z: LibLZ4F) -> dict[str, bytes]:
    return {**valid_frames(z), **{f"mut_{k}": v for k, v in mutants(z).items()}}


def has_offset0_match(chunk: bytes) -> bool:
    """Does a compressed block of the chunk hold a match with offset 0?  liblz4 1.9.4 accepts such a match when it
    lies far enough from the block end and copies the destination's own bytes; the LZ4 block grammar has no offset 0,
    and this library rejects it in LZ4 frames as nvcompBatchedLZ4DecompressAsync does in raw blocks."""
    try:
        p = 0
        while p < len(chunk):
            magic = int.from_bytes(chunk[p:p + 4], "little")
            if magic & 0xFFFFFFF0 == SKIP_MAGIC:
                p += 8 + int.from_bytes(chunk[p + 4:p + 8], "little")
                continue
            flg = chunk[p + 4]
            p += 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)
            while True:
                b = int.from_bytes(chunk[p:p + 4], "little")
                p += 4
                n = b & 0x7FFFFFFF
                if n == 0:
                    break
                if not b >> 31 and _block_has_offset0(chunk[p:p + n]):
                    return True
                p += n + (4 if flg & 0x10 else 0)
            p += 4 if flg & 4 else 0
    except IndexError:
        pass
    return False


def _block_has_offset0(blk: bytes) -> bool:
    ip, n = 0, len(blk)

    def length(ip, v):
        if v != 15:
            return ip, v
        while ip < n:
            b = blk[ip]
            ip += 1
            v += b
            if b != 255:
                break
        return ip, v

    while ip < n:
        t = blk[ip]
        ip, ll = length(ip + 1, t >> 4)
        ip += ll
        if ip + 2 > n:
            return False
        if blk[ip] == 0 and blk[ip + 1] == 0:
            return True
        ip, _ = length(ip + 2, t & 15)
    return False
