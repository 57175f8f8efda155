"""CPU: the host model of the high-level interface's container (tests/hlif_model.py)."""
import struct
import zlib

import numpy as np
import pytest

import hlif_model as hm


def _chunks(seed, sizes):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, s, dtype=np.uint8).tobytes() for s in sizes]


@pytest.mark.parametrize("checksums", [False, True])
@pytest.mark.parametrize("sizes", [[], [0], [1], [7, 8, 9], [16, 3, 0, 5, 1 << 12], list(range(1, 40))])
def test_build_then_parse_is_identity(sizes, checksums):
    chunk_bytes = 4096
    uncompressed = (bytes(range(256)) * 16 * len(sizes))[:max(len(sizes) - 1, 0) * chunk_bytes + 17 * bool(sizes)]
    streams = _chunks(len(sizes), sizes)
    opts = struct.pack("<QiiiI", 4096, 6, 1, 1, 1)
    buf = hm.build("Cascaded", opts, chunk_bytes, uncompressed, streams, checksums=checksums)
    c = hm.parse(buf + b"\xff" * 13)                  # bytes past total_bytes are not the container's
    assert (c.magic, c.format, c.opts) == (hm.MAGIC, 3, opts)
    assert (c.uncompressed_bytes, c.chunk_bytes, c.num_chunks) == (len(uncompressed), chunk_bytes, len(sizes))
    assert c.sizes == sizes and c.chunks == streams
    assert c.total_bytes == len(buf) == 72 + 8 * len(sizes) + sum((s + 7) // 8 * 8 for s in sizes)
    assert c.flags == int(checksums)
    if checksums:
        assert c.checksum_uncomp == zlib.crc32(uncompressed)
        assert c.checksum_comp == zlib.crc32(buf[72:]) == hm.payload_crc(buf)
    else:
        assert c.checksum_uncomp == c.checksum_comp == 0
    assert hm.pack_header(c) == buf[:72]


def test_offsets_match_the_cpp_test():
    """tests/cpp/hlif_test.cu reads and patches these offsets directly."""
    assert hm.HEADER_BYTES == 72
    assert hm.OFFSET["uncompressed_bytes"] == 32
    assert hm.OFFSET["chunk_bytes"] == 40
    assert hm.OFFSET["num_chunks"] == 48
    assert hm.OFFSET["checksum_uncomp"] == 64 and hm.OFFSET["checksum_comp"] == 68
    assert hm.OFFSET["total_bytes"] == 56 and hm.OFFSET["flags"] == 52
    assert struct.calcsize("<II24sQQIIQII") == 72


@pytest.mark.parametrize("mutate", ["magic", "padding", "total_low", "total_high", "num_chunks", "truncated"])
def test_parse_rejects_layout_violations(mutate):
    streams = _chunks(1, [5, 9, 3])
    buf = hm.build("LZ4", b"\0" * 4, 100, 250, streams)
    if mutate == "magic":
        buf = hm.patch(buf, "magic", 0)
    elif mutate == "padding":
        b = bytearray(buf)
        b[72 + 24 + 5] = 1                             # first pad byte after chunk 0
        buf = bytes(b)
    elif mutate == "total_low":
        buf = hm.patch(buf, "total_bytes", len(buf) - 8)
    elif mutate == "total_high":
        buf = hm.patch(buf, "total_bytes", len(buf) + 8) + bytes(8)
    elif mutate == "num_chunks":
        buf = hm.patch(buf, "num_chunks", 2)
    else:
        buf = buf[:-1]
    with pytest.raises(AssertionError):
        hm.parse(buf)
