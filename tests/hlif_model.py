"""Host model of the high-level interface's container (nvcomp_b200/csrc/hlif.cu), the format every
nvcomp::*Manager writes and reads.  Plain Python, independent of the library:

    header (72 bytes, little-endian)
        0  u32 magic = 0x3242564e          32  u64 uncompressed_bytes      56  u64 total_bytes
        4  u32 format                      40  u64 chunk_bytes             64  u32 CRC-32 of the uncompressed buffer
        8  opts[24] (options struct,       48  u32 num_chunks              68  u32 CRC-32 of container[72:total_bytes]
           zero-padded)                    52  u32 flags (bit 0: checksums present)
    u64 size[num_chunks]
    chunk 0, chunk 1, ...                  each at the next 8-byte boundary, zero-padded to 8 bytes

total_bytes = 72 + 8 * num_chunks + sum(round8(size[i])).  The CRC-32 is zlib's."""
from __future__ import annotations

import struct
import zlib
from dataclasses import dataclass, field

MAGIC = 0x3242564E
HEADER_BYTES = 72
FORMATS = {"LZ4": 1, "Snappy": 2, "Cascaded": 3, "Bitcomp": 4, "ANS": 5, "Deflate": 6}
FLAG_CHECKSUMS = 1

# (name, offset, struct code)
FIELDS = (
    ("magic", 0, "<I"),
    ("format", 4, "<I"),
    ("opts", 8, "<24s"),
    ("uncompressed_bytes", 32, "<Q"),
    ("chunk_bytes", 40, "<Q"),
    ("num_chunks", 48, "<I"),
    ("flags", 52, "<I"),
    ("total_bytes", 56, "<Q"),
    ("checksum_uncomp", 64, "<I"),
    ("checksum_comp", 68, "<I"),
)
OFFSET = {name: off for name, off, _ in FIELDS}


def round8(n: int) -> int:
    return (n + 7) & ~7


def total_bytes(sizes) -> int:
    return HEADER_BYTES + 8 * len(sizes) + sum(round8(s) for s in sizes)


@dataclass
class Container:
    magic: int
    format: int
    opts: bytes
    uncompressed_bytes: int
    chunk_bytes: int
    num_chunks: int
    flags: int
    total_bytes: int
    checksum_uncomp: int
    checksum_comp: int
    sizes: list = field(default_factory=list)
    chunks: list = field(default_factory=list)


def pack_header(c: Container) -> bytes:
    out = bytearray(HEADER_BYTES)
    for name, off, code in FIELDS:
        struct.pack_into(code, out, off, getattr(c, name))
    return bytes(out)


def parse(buf) -> Container:
    """Parse a container and assert every layout rule (the buffer may extend past total_bytes)."""
    buf = memoryview(bytes(buf))
    assert len(buf) >= HEADER_BYTES, len(buf)
    vals = {name: struct.unpack_from(code, buf, off)[0] for name, off, code in FIELDS}
    c = Container(**vals)
    assert c.magic == MAGIC, hex(c.magic)
    assert c.format in FORMATS.values(), c.format
    assert c.flags & ~FLAG_CHECKSUMS == 0, c.flags
    assert c.chunk_bytes > 0
    want = 0 if c.uncompressed_bytes == 0 else -(-c.uncompressed_bytes // c.chunk_bytes)
    assert c.num_chunks == want, (c.num_chunks, want)
    n = c.num_chunks
    assert len(buf) >= HEADER_BYTES + 8 * n
    c.sizes = list(struct.unpack_from(f"<{n}Q", buf, HEADER_BYTES))
    assert c.total_bytes == total_bytes(c.sizes), (c.total_bytes, total_bytes(c.sizes))
    assert len(buf) >= c.total_bytes, (len(buf), c.total_bytes)
    off = HEADER_BYTES + 8 * n
    for s in c.sizes:
        assert off % 8 == 0
        c.chunks.append(bytes(buf[off:off + s]))
        assert not any(buf[off + s:off + round8(s)]), f"non-zero padding after the chunk at {off}"
        off += round8(s)
    assert off == c.total_bytes
    return c


def payload_crc(buf) -> int:
    """CRC-32 of everything after the header: the size table and every chunk."""
    total = struct.unpack_from("<Q", buf, OFFSET["total_bytes"])[0]
    return zlib.crc32(memoryview(buf)[HEADER_BYTES:total])


def build(fmt: str | int, opts: bytes, chunk_bytes: int, uncompressed, chunks, checksums: bool = False) -> bytes:
    """Assemble a container around any chunk streams.  `uncompressed` is the buffer the chunks encode (its CRC-32 is
    stored when checksums is set) or its length."""
    assert len(opts) <= 24
    n = uncompressed if isinstance(uncompressed, int) else len(uncompressed)
    c = Container(magic=MAGIC, format=FORMATS.get(fmt, fmt), opts=bytes(opts).ljust(24, b"\0"), uncompressed_bytes=n,
                  chunk_bytes=chunk_bytes, num_chunks=len(chunks), flags=FLAG_CHECKSUMS if checksums else 0,
                  total_bytes=total_bytes([len(s) for s in chunks]), checksum_uncomp=0, checksum_comp=0)
    body = bytearray(struct.pack(f"<{len(chunks)}Q", *[len(s) for s in chunks]))
    for s in chunks:
        body += s
        body += bytes(round8(len(s)) - len(s))
    if checksums:
        assert not isinstance(uncompressed, int), "checksums need the uncompressed bytes"
        c.checksum_uncomp = zlib.crc32(uncompressed)
        c.checksum_comp = zlib.crc32(body)
    return pack_header(c) + bytes(body)


def patch(buf: bytes, name: str, value: int) -> bytes:
    """Return buf with one header field replaced."""
    code = dict((n, c) for n, _, c in FIELDS)[name]
    out = bytearray(buf)
    struct.pack_into(code, out, OFFSET[name], value)
    return bytes(out)
