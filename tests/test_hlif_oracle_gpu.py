"""-m gpu: the high-level interface (nvcomp::*Manager, create_manager) held to the container model
(tests/hlif_model.py), the CPU oracles and zlib, through build/tests/libhlif_shim.so.

A. Every container a manager writes parses under the model; its header matches the manager's inputs, every chunk
   decodes on the CPU to exactly its slice and equals the low-level encoder's (or the oracle's) stream for that slice,
   and the stored checksums are zlib's CRC-32s.  Up to 2501 chunks (past the 1024-chunk scan tiles).
B. Whole-buffer CRC-32s of buffers past 64 MiB, where one fold thread combines more than one 64 KiB piece.
C. Containers the model assembles from CPU-encoded chunks decode with the matching manager and with create_manager.
D. Inconsistent containers (short / long chunks, wrong total size, wrong table entries, wrong checksums) get the
   right verdict.  Each sits in an allocation with 1 MiB of canary past its end, more than any pointer derived from
   the table can reach, so a missing check shows up as a wrong verdict and never as a fault.
E. The checksum policy matrix, a user scratch buffer, output alignment and chunk sizes the typed codecs cannot use.

Every output region is surrounded by canaries: compress may write only [0, total_bytes) of its output, decompress only
[0, n)."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch

import hlif_model as hm
from conftest import ROOT
from nvcomp_b200._lib import ANSOpts, BitcompOpts, CascadedOpts, DeflateOpts, LZ4Opts, SnappyOpts, Status, Type
from nvcomp_b200.batched import Codec, make_batch

pytestmark = pytest.mark.gpu

SHIM_PATH = os.path.join(ROOT, "build", "tests", "libhlif_shim.so")

# ChecksumPolicy (include/nvcomp/nvcompManager.hpp)
NO_COMPUTE_NO_VERIFY, COMPUTE_NO_VERIFY, VERIFY_IF_PRESENT, COMPUTE_VERIFY_IF_PRESENT, COMPUTE_AND_VERIFY = range(5)
COMPUTES = {COMPUTE_NO_VERIFY, COMPUTE_VERIFY_IF_PRESENT, COMPUTE_AND_VERIFY}
VERIFIES = {VERIFY_IF_PRESENT, COMPUTE_VERIFY_IF_PRESENT, COMPUTE_AND_VERIFY}

CANARY = 0x3C
FILL = 0xA5
GUARD = 4096
MIB = 1 << 20


class ShimError(RuntimeError):
    def __init__(self, fn, status):
        super().__init__(f"{fn} returned {Status(status).name if status in Status._value2member_map_ else status}")
        self.status = status


class Shim:
    def __init__(self):
        if not os.path.exists(SHIM_PATH):
            subprocess.run(["make", "-C", ROOT, "build/tests/libhlif_shim.so"], check=True)
        lib = C.CDLL(SHIM_PATH)
        P, Z, I = C.c_void_p, C.c_size_t, C.c_int
        PP, ZP = C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)
        sigs = {
            "create": [C.c_uint, C.c_char_p, Z, I, P, I, PP],
            "create_from": [P, P, I, I, PP],
            "configure_compression": [P, Z, PP, ZP, ZP],
            "compress": [P, P, P, P],
            "compression_status": [P],
            "configure_decompression": [P, P, PP, ZP, ZP],
            "configure_decompression_cc": [P, P, PP, ZP, ZP],
            "decompress": [P, P, P, P],
            "decompression_status": [P],
            "compressed_output_size": [P, P, ZP],
            "required_scratch": [P, ZP],
            "set_scratch": [P, P],
        }
        for name, args in sigs.items():
            fn = getattr(lib, f"hlif_shim_{name}")
            fn.argtypes, fn.restype = args, I
        for name in ("destroy", "free_compression_config", "free_decompression_config"):
            fn = getattr(lib, f"hlif_shim_{name}")
            fn.argtypes, fn.restype = [P], None
        self.lib = lib

    def call(self, name, *args):
        st = getattr(self.lib, f"hlif_shim_{name}")(*args)
        if st != 0:
            raise ShimError(name, st)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _device():
    return torch.cuda.current_device()


class Config:
    def __init__(self, shim, handle, free, status_fn, **fields):
        self.shim, self.handle, self._free, self._status = shim, handle, free, status_fn
        self.__dict__.update(fields)

    def status(self):
        torch.cuda.synchronize()
        return getattr(self.shim.lib, f"hlif_shim_{self._status}")(self.handle)

    def __del__(self):
        getattr(self.shim.lib, f"hlif_shim_{self._free}")(self.handle)


class Manager:
    def __init__(self, shim, handle):
        self.shim, self.handle = shim, handle

    @classmethod
    def create(cls, shim, fmt, opts, chunk, policy):
        h = C.c_void_p()
        shim.call("create", hm.FORMATS[fmt], bytes(opts).ljust(24, b"\0"), chunk, policy, _stream(), _device(),
                  C.byref(h))
        return cls(shim, h)

    @classmethod
    def from_buffer(cls, shim, comp_ptr, policy):
        h = C.c_void_p()
        shim.call("create_from", comp_ptr, _stream(), _device(), policy, C.byref(h))
        return cls(shim, h)

    def __del__(self):
        self.shim.lib.hlif_shim_destroy(self.handle)

    def configure_compression(self, n):
        h, mx, nc = C.c_void_p(), C.c_size_t(), C.c_size_t()
        self.shim.call("configure_compression", self.handle, n, C.byref(h), C.byref(mx), C.byref(nc))
        return Config(self.shim, h, "free_compression_config", "compression_status", max_comp=mx.value,
                      num_chunks=nc.value)

    def _dconfig(self, name, src):
        h, n, nc = C.c_void_p(), C.c_size_t(), C.c_size_t()
        self.shim.call(name, self.handle, src, C.byref(h), C.byref(n), C.byref(nc))
        return Config(self.shim, h, "free_decompression_config", "decompression_status", decomp_size=n.value,
                      num_chunks=nc.value)

    def configure_decompression(self, comp_ptr):
        return self._dconfig("configure_decompression", comp_ptr)

    def configure_decompression_cc(self, cc):
        return self._dconfig("configure_decompression_cc", cc.handle)

    def compress(self, in_ptr, out_ptr, cc):
        self.shim.call("compress", self.handle, in_ptr, out_ptr, cc.handle)

    def decompress(self, out_ptr, comp_ptr, dc):
        self.shim.call("decompress", self.handle, out_ptr, comp_ptr, dc.handle)

    def compressed_output_size(self, comp_ptr):
        n = C.c_size_t()
        self.shim.call("compressed_output_size", self.handle, comp_ptr, C.byref(n))
        return n.value

    def required_scratch(self):
        n = C.c_size_t()
        self.shim.call("required_scratch", self.handle, C.byref(n))
        return n.value

    def set_scratch(self, ptr):
        self.shim.call("set_scratch", self.handle, ptr)


class Guarded:
    """n usable device bytes at `ptr` (8-byte aligned), `before` / `after` bytes of CANARY around them.  The usable
    bytes start as `content` (then FILL) or all FILL."""

    def __init__(self, n, content=b"", before=GUARD, after=GUARD, fill=FILL):
        host = np.full(before + n + after, CANARY, dtype=np.uint8)
        host[before:before + n] = fill
        host[before:before + len(content)] = np.frombuffer(content, dtype=np.uint8)
        self.slab = torch.from_numpy(host).cuda()
        self.off, self.n = before, n
        self.ptr = self.slab.data_ptr() + before

    def host(self):
        torch.cuda.synchronize()
        return self.slab.cpu().numpy()

    def check(self, lo, hi, what, host=None):
        """Every byte outside [lo, hi) of the usable region, and every guard byte, is still CANARY."""
        h = self.host() if host is None else host
        allowed = np.zeros(h.size, dtype=bool)
        allowed[self.off + lo:self.off + hi] = True
        bad = np.flatnonzero((h != CANARY) & ~allowed)
        assert bad.size == 0, f"{what}: {bad.size} bytes written outside [{lo}, {hi}), first at {int(bad[0]) - self.off}"
        return h

    def xor(self, pos, bit=1):
        i = self.off + pos
        self.slab[i:i + 1] ^= bit


def _dev(data: bytes):
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy() if data else np.zeros(1, np.uint8)).cuda()


def _data(n, seed):
    """Sorted 64-bit words (runs, small deltas) with every fifth 512-byte block random: both matches and literals for
    the byte codecs, both narrow and wide fields for the typed ones."""
    rng = np.random.default_rng(seed)
    words = np.cumsum(rng.integers(0, 48, n // 8 + 1, dtype=np.int64))
    out = words.view(np.uint8)[:n].copy()
    mask = (np.arange(n) // 512) % 5 == 3
    out[mask] = rng.integers(0, 256, int(mask.sum()), dtype=np.uint8)
    return out.tobytes()


def _random(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _slices(data, chunk):
    return [data[i:i + chunk] for i in range(0, len(data), chunk)]


@pytest.fixture(scope="module")
def shim():
    return Shim()


def compress(mgr, data, what):
    """Compress on the GPU into a guarded output; returns (container bytes, config, guarded output)."""
    inp = _dev(data)
    cc = mgr.configure_compression(len(data))
    out = Guarded(cc.max_comp, fill=CANARY)
    mgr.compress(inp.data_ptr(), out.ptr, cc)
    assert cc.status() == 0, what
    total = mgr.compressed_output_size(out.ptr)
    assert 0 < total <= cc.max_comp, (what, total, cc.max_comp)
    h = out.check(0, total, f"{what}: compress")
    return h[out.off:out.off + total].tobytes(), cc, out


def decompress(mgr, comp_ptr, dc, n, what):
    """Decompress into a guarded output; returns (status, output bytes)."""
    out = Guarded(n)
    mgr.decompress(out.ptr, comp_ptr, dc)
    st = dc.status()
    h = out.check(0, n, f"{what}: decompress")
    return st, h[out.off:out.off + n].tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# A. container conformance
# ---------------------------------------------------------------------------------------------------------------------
# (format, options, oracle codec name, oracle encoder keywords: None = the low-level GPU encoder is the reference)
CONFIGS = {
    "lz4_char": ("LZ4", LZ4Opts(Type.CHAR), "lz4", None),
    "lz4_int": ("LZ4", LZ4Opts(Type.INT), "lz4", None),
    "snappy": ("Snappy", SnappyOpts(0), "snappy", None),
    "cascaded_rle_delta_bp": ("Cascaded", CascadedOpts(4096, Type.LONGLONG, 1, 1, 1), "cascaded",
                              dict(chunk_size=4096, type=Type.LONGLONG, num_RLEs=1, num_deltas=1, use_bp=1)),
    "cascaded_rle2_nobp": ("Cascaded", CascadedOpts(1024, Type.INT, 2, 0, 0), "cascaded",
                           dict(chunk_size=1024, type=Type.INT, num_RLEs=2, num_deltas=0, use_bp=0)),
    "bitcomp_a0_u64": ("Bitcomp", BitcompOpts(0, Type.ULONGLONG), "bitcomp", dict(algo=0, type=Type.ULONGLONG)),
    "bitcomp_a1_u64": ("Bitcomp", BitcompOpts(1, Type.ULONGLONG), "bitcomp", dict(algo=1, type=Type.ULONGLONG)),
    "bitcomp_a0_i16": ("Bitcomp", BitcompOpts(0, Type.SHORT), "bitcomp", dict(algo=0, type=Type.SHORT)),
    "bitcomp_a1_i16": ("Bitcomp", BitcompOpts(1, Type.SHORT), "bitcomp", dict(algo=1, type=Type.SHORT)),
    "ans": ("ANS", ANSOpts(0), "ans", {}),
    "deflate0": ("Deflate", DeflateOpts(0), None, None),
    "deflate1": ("Deflate", DeflateOpts(1), None, None),
    "deflate2": ("Deflate", DeflateOpts(2), None, None),
}
TYPED = ("Cascaded", "Bitcomp")
MAX_CHUNK = {"LZ4": 1 << 24, "Snappy": 1 << 24, "Cascaded": 1 << 24, "Bitcomp": 1 << 24, "ANS": 1 << 24,
             "Deflate": 1 << 16}


def _cpu_decode(oracle, oname, stream, cap):
    if oname is None:
        z = zlib.decompressobj(-15)
        try:
            out = z.decompress(stream, cap + 1)
        except zlib.error:
            return None
        return out if z.eof and not z.unconsumed_tail and len(out) <= cap else None
    return oracle.decompress(oname, stream, cap)


def _reference_streams(oracle, cfg, slices, chunk):
    fmt, opts, oname, okw = cfg
    if okw is not None:
        return [oracle.compress_typed(oname, s, **okw) for s in slices]
    if not slices:
        return []
    comp = Codec(fmt, opts=opts).compress(make_batch(slices), max_chunk=chunk)
    torch.cuda.synchronize()
    return comp.to_host(comp.sizes.cpu().numpy())


def _conformance(shim, oracle, key, chunk, lengths):
    cfg = CONFIGS[key]
    fmt, opts, oname, _ = cfg
    for i, n in enumerate(lengths):
        what = f"{key} chunk={chunk} n={n}"
        policy = COMPUTE_AND_VERIFY if i % 2 else NO_COMPUTE_NO_VERIFY
        mgr = Manager.create(shim, fmt, opts, chunk, policy)
        data = _data(n, seed=n ^ chunk)
        comp, cc, out = compress(mgr, data, what)
        slices = _slices(data, chunk)
        assert cc.num_chunks == len(slices), what
        c = hm.parse(comp)
        assert (c.format, c.opts) == (hm.FORMATS[fmt], bytes(opts).ljust(24, b"\0")), what
        assert (c.uncompressed_bytes, c.chunk_bytes, c.num_chunks) == (n, chunk, len(slices)), what
        assert c.total_bytes == len(comp) <= cc.max_comp, what
        if policy in COMPUTES:
            assert c.flags == hm.FLAG_CHECKSUMS, what
            assert c.checksum_uncomp == zlib.crc32(data), what
            assert c.checksum_comp == hm.payload_crc(comp), what
        else:
            assert c.flags == 0, what
        bad = [j for j, (s, raw) in enumerate(zip(c.chunks, slices)) if _cpu_decode(oracle, oname, s, len(raw)) != raw]
        assert not bad, (what, "chunks the CPU reference does not decode to their slice", bad[:10])
        ref = _reference_streams(oracle, cfg, slices, chunk)
        diff = [j for j, (s, r) in enumerate(zip(c.chunks, ref)) if s != r]
        assert not diff, (what, "chunks that differ from the reference encoder's stream", diff[:10])
        # decode through the three configuration paths
        paths = (("header", mgr, lambda m: m.configure_decompression(out.ptr)),
                 ("compression config", mgr, lambda m: m.configure_decompression_cc(cc)),
                 ("create_manager", Manager.from_buffer(shim, out.ptr, policy), lambda m: m.configure_decompression(out.ptr)))
        for name, m, configure in paths:
            dc = configure(m)
            assert (dc.decomp_size, dc.num_chunks) == (n, len(slices)), (what, name)
            st, back = decompress(m, out.ptr, dc, n, f"{what} via {name}")
            assert st == 0 and back == data, (what, name, st)


def _lengths(chunk):
    out = [0, 1, chunk - 1, chunk, chunk + 1]
    if chunk == 4096:
        out += [1023 * chunk, 1024 * chunk, 1025 * chunk, 2500 * chunk + 777]
    return out


@pytest.mark.parametrize("chunk", ["4096", "65536", "odd"])
@pytest.mark.parametrize("key", list(CONFIGS))
def test_container_conformance(shim, oracle, key, chunk):
    fmt = CONFIGS[key][0]
    c = {"4096": 4096, "65536": 65536, "odd": 65528 if fmt in TYPED else 65533}[chunk]
    _conformance(shim, oracle, key, c, _lengths(c))


@pytest.mark.parametrize("key", ["lz4_char", "snappy", "cascaded_rle_delta_bp", "bitcomp_a1_u64", "ans"])
def test_container_conformance_max_chunk(shim, oracle, key):
    c = MAX_CHUNK[CONFIGS[key][0]]
    _conformance(shim, oracle, key, c, [0, c, c + 1])


# ---------------------------------------------------------------------------------------------------------------------
# B. checksums past one 64 KiB piece per fold thread (1024 threads x 64 KiB = 64 MiB)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,kind", [(64 * MIB - 1, "random"), (64 * MIB, "random"), (64 * MIB + 1, "random"),
                                    (150 * MIB + 12345, "random"), (150 * MIB + 12345, "compressible")])
def test_checksums_past_64mib(shim, n, kind):
    data = _random(n, n) if kind == "random" else _data(n, n)
    mgr = Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), 65536, COMPUTE_AND_VERIFY)
    comp, cc, out = compress(mgr, data, f"{kind} n={n}")
    c = hm.parse(comp)
    if kind == "random":
        assert c.total_bytes - hm.HEADER_BYTES > 64 * MIB          # the payload fold also takes > 1 piece per thread
    assert c.flags == hm.FLAG_CHECKSUMS
    assert c.checksum_uncomp == zlib.crc32(data)
    assert c.checksum_comp == hm.payload_crc(comp)
    dc = mgr.configure_decompression(out.ptr)
    st, back = decompress(mgr, out.ptr, dc, n, "round trip")
    assert st == 0 and back == data
    del back
    # one flipped bit in the last 64 KiB piece of the payload
    payload = c.total_bytes - hm.HEADER_BYTES
    pos = c.total_bytes - 3
    assert pos >= hm.HEADER_BYTES + (payload - 1) // 65536 * 65536
    out.xor(pos)
    st, _ = decompress(mgr, out.ptr, dc, n, "payload bit")
    assert st in (Status.ErrorBadChecksum, Status.ErrorCannotDecompress), st
    out.xor(pos)
    # one flipped bit in the stored checksum of the uncompressed buffer: only the verify-side hash of the output sees it
    out.xor(hm.OFFSET["checksum_uncomp"], 0x10)
    st, back = decompress(mgr, out.ptr, dc, n, "stored checksum bit")
    assert st == Status.ErrorBadChecksum, st
    assert back == data


# ---------------------------------------------------------------------------------------------------------------------
# C. containers assembled from CPU-encoded chunks
# ---------------------------------------------------------------------------------------------------------------------
def _deflate(s):
    z = zlib.compressobj(6, zlib.DEFLATED, -15)
    return z.compress(s) + z.flush()


# encoder(oracle, liblz4, chunk) -> stream
FOREIGN = {
    "lz4": ("LZ4", LZ4Opts(Type.CHAR), lambda o, lz4, s: o.compress("lz4", s)),
    "lz4_hc": ("LZ4", LZ4Opts(Type.CHAR), lambda o, lz4, s: lz4.compress(s, hc=12)),
    "snappy": ("Snappy", SnappyOpts(0), lambda o, lz4, s: o.compress("snappy", s)),
    "cascaded": ("Cascaded", CascadedOpts(2048, Type.UINT, 1, 1, 1),
                 lambda o, lz4, s: o.compress_typed("cascaded", s, chunk_size=2048, type=Type.UINT, num_RLEs=1,
                                                    num_deltas=1, use_bp=1)),
    "bitcomp": ("Bitcomp", BitcompOpts(1, Type.LONGLONG),
                lambda o, lz4, s: o.compress_typed("bitcomp", s, algo=1, type=Type.LONGLONG)),
    "ans": ("ANS", ANSOpts(0), lambda o, lz4, s: o.compress_typed("ans", s)),
    "deflate": ("Deflate", DeflateOpts(1), lambda o, lz4, s: _deflate(s)),
}


@pytest.mark.parametrize("checksums", [False, True])
@pytest.mark.parametrize("key", list(FOREIGN))
def test_foreign_containers(shim, oracle, request, key, checksums):
    fmt, opts, encode = FOREIGN[key]
    lz4 = request.getfixturevalue("liblz4") if key == "lz4_hc" else None
    chunk, n = 4096, 1100 * 4096 + 321
    data = _data(n, 7)
    streams = [encode(oracle, lz4, s) for s in _slices(data, chunk)]
    buf = hm.build(fmt, bytes(opts), chunk, data, streams, checksums=checksums)
    comp = Guarded(len(buf), buf)
    policy = COMPUTE_AND_VERIFY if checksums else VERIFY_IF_PRESENT
    for name, mgr in (("manager", Manager.create(shim, fmt, opts, chunk, policy)),
                      ("create_manager", Manager.from_buffer(shim, comp.ptr, policy))):
        dc = mgr.configure_decompression(comp.ptr)
        assert mgr.compressed_output_size(comp.ptr) == len(buf)
        st, back = decompress(mgr, comp.ptr, dc, n, f"{key} via {name}")
        assert st == 0 and back == data, (key, name, st)
    comp.check(0, len(buf), "container")


# ---------------------------------------------------------------------------------------------------------------------
# D. inconsistent containers
# ---------------------------------------------------------------------------------------------------------------------
D_CHUNK = 4096
D_N = 1100 * D_CHUNK + 1000                     # 1101 chunks, the last one 1000 bytes
D_K = 1050                                      # a chunk past the first 1024-chunk scan tile


def _lz4_container(oracle, edit=None, checksums=False):
    """The chunks are the oracle's LZ4 streams; edit(streams, slices) may replace some."""
    data = _data(D_N, 3)
    slices = _slices(data, D_CHUNK)
    streams = [oracle.compress("lz4", s) for s in slices]
    if edit:
        edit(streams, slices)
    return data, hm.build("LZ4", bytes(LZ4Opts(Type.CHAR)), D_CHUNK, data, streams, checksums=checksums)


def _place(buf):
    return Guarded(len(buf), buf, after=MIB + GUARD)


def _verdict(shim, buf, policy, n=D_N):
    """(configure error or None, decompress status, output) of a container under a fresh LZ4 manager."""
    comp = _place(buf)
    mgr = Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), D_CHUNK, policy)
    try:
        dc = mgr.configure_decompression(comp.ptr)
    except ShimError as e:
        return e.status, None, None
    st, back = decompress(mgr, comp.ptr, dc, n, "inconsistent container")
    comp.check(0, len(buf), "container")
    return None, st, back


@pytest.mark.parametrize("edit", ["short_nonlast", "short_last", "long_nonlast", "long_last"])
def test_chunk_decoding_to_the_wrong_length(shim, oracle, edit):
    """A chunk stream that decodes validly to one byte fewer / more than its slot."""
    i = D_K if edit.endswith("nonlast") else -1

    def resize(streams, slices):
        streams[i] = oracle.compress("lz4", slices[i][:-1] if edit.startswith("short") else slices[i] + b"x")
    _, buf = _lz4_container(oracle, resize)
    err, st, _ = _verdict(shim, buf, NO_COMPUTE_NO_VERIFY)
    assert err is None
    assert st == Status.ErrorCannotDecompress, Status(st).name


@pytest.mark.parametrize("delta", [-8, 8])
def test_total_bytes_disagreeing_with_the_table(shim, oracle, delta):
    _, buf = _lz4_container(oracle)
    buf = hm.patch(buf, "total_bytes", len(buf) + delta)
    err, st, _ = _verdict(shim, buf, NO_COMPUTE_NO_VERIFY)
    assert err == Status.ErrorInvalidValue, (err, st)


def test_table_entry_covering_bytes_past_the_stream(shim, oracle):
    """Entry D_K is 8 larger (the chunk carries 8 trailing zero bytes) and total_bytes matches."""
    def edit(streams, slices):
        streams[D_K] = streams[D_K] + bytes(8)
        assert oracle.decompress("lz4", streams[D_K], D_CHUNK) is None
    _, buf = _lz4_container(oracle, edit)
    err, st, _ = _verdict(shim, buf, NO_COMPUTE_NO_VERIFY)
    assert err is None and st == Status.ErrorCannotDecompress, (err, st)


def test_table_entry_above_the_format_bound(shim, oracle):
    """An entry larger than CompressGetMaxOutputChunkSize(chunk) is refused, even with total_bytes consistent."""
    bound = Codec("LZ4", opts=LZ4Opts(Type.CHAR)).compress_get_max_output_chunk_size(D_CHUNK)

    def edit(streams, slices):
        streams[D_K] = streams[D_K] + bytes(bound + 1 - len(streams[D_K]))
    _, buf = _lz4_container(oracle, edit)
    err, st, _ = _verdict(shim, buf, NO_COMPUTE_NO_VERIFY)
    assert err == Status.ErrorInvalidValue, (err, st)


@pytest.mark.parametrize("policy,want", [(VERIFY_IF_PRESENT, Status.ErrorBadChecksum),
                                         (COMPUTE_AND_VERIFY, Status.ErrorBadChecksum),
                                         (NO_COMPUTE_NO_VERIFY, Status.Success)])
def test_wrong_stored_checksums(shim, oracle, policy, want):
    data, buf = _lz4_container(oracle, checksums=True)
    c = hm.parse(buf)
    buf = hm.patch(hm.patch(buf, "checksum_uncomp", c.checksum_uncomp ^ 1), "checksum_comp", c.checksum_comp ^ 1)
    err, st, back = _verdict(shim, buf, policy)
    assert err is None and st == want, (err, st)
    if want == Status.Success:
        assert back == data


# ---------------------------------------------------------------------------------------------------------------------
# E. policies, scratch, alignment, construction
# ---------------------------------------------------------------------------------------------------------------------
def test_policy_matrix(shim):
    chunk, n = 4096, 3 * 4096 + 5
    data = _data(n, 11)
    for pc in range(5):
        mgr = Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), chunk, pc)
        comp, _, out = compress(mgr, data, f"policy {pc}")
        flag = hm.parse(comp).flags & hm.FLAG_CHECKSUMS
        assert bool(flag) == (pc in COMPUTES), pc
        for pd in range(5):
            dm = Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), chunk, pd)
            if pd == COMPUTE_AND_VERIFY and not flag:
                with pytest.raises(ShimError) as e:
                    dm.configure_decompression(out.ptr)
                assert e.value.status == Status.ErrorCannotVerifyChecksums
                continue
            dc = dm.configure_decompression(out.ptr)
            st, back = decompress(dm, out.ptr, dc, n, f"policy {pc} -> {pd}")
            assert st == 0 and back == data, (pc, pd, st)
            # a wrong stored checksum is seen exactly when the buffer carries checksums and the policy verifies
            out.xor(hm.OFFSET["checksum_uncomp"])
            st, back = decompress(dm, out.ptr, dc, n, f"policy {pc} -> {pd}, wrong checksum")
            out.xor(hm.OFFSET["checksum_uncomp"])
            want = Status.ErrorBadChecksum if (flag and pd in VERIFIES) else Status.Success
            assert st == want and back == data, (pc, pd, st)


def test_user_scratch(shim):
    chunk, n = 4096, 40 * 4096 + 3
    data = _data(n, 12)
    comp, _, src = compress(Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), chunk, COMPUTE_AND_VERIFY), data, "source")
    mgr = Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), chunk, COMPUTE_AND_VERIFY)
    cc = mgr.configure_compression(n)
    dc = mgr.configure_decompression(src.ptr)
    need = mgr.required_scratch()
    assert need > 0
    scratch = Guarded(need, fill=CANARY)
    mgr.set_scratch(scratch.ptr)
    inp = _dev(data)
    out = Guarded(cc.max_comp, fill=CANARY)
    mgr.compress(inp.data_ptr(), out.ptr, cc)
    assert cc.status() == 0
    total = mgr.compressed_output_size(out.ptr)
    h = out.check(0, total, "compress with user scratch")
    assert h[out.off:out.off + total].tobytes() == comp
    st, back = decompress(mgr, src.ptr, dc, n, "decompress with user scratch")
    assert st == 0 and back == data
    scratch.check(0, need, "user scratch")
    # a larger configuration no longer fits: compress refuses before anything is launched
    cc2 = mgr.configure_compression(8 * n)
    assert mgr.required_scratch() > need
    inp2, out2 = _dev(data * 8), Guarded(cc2.max_comp, fill=CANARY)
    with pytest.raises(ShimError) as e:
        mgr.compress(inp2.data_ptr(), out2.ptr, cc2)
    assert e.value.status == Status.ErrorInvalidValue
    out2.check(0, 0, "refused compress")
    scratch.check(0, need, "user scratch after the refused compress")


@pytest.mark.parametrize("misalign", [1, 4])
def test_compress_output_alignment(shim, misalign):
    mgr = Manager.create(shim, "LZ4", LZ4Opts(Type.CHAR), 4096, NO_COMPUTE_NO_VERIFY)
    inp = _dev(_data(10000, 13))
    cc = mgr.configure_compression(10000)
    out = Guarded(cc.max_comp + 8, fill=CANARY)
    with pytest.raises(ShimError) as e:
        mgr.compress(inp.data_ptr(), out.ptr + misalign, cc)
    assert e.value.status == Status.ErrorAlignment
    out.check(0, 0, "refused compress")


@pytest.mark.parametrize("chunk", [65532, 65533, 65529])
@pytest.mark.parametrize("fmt,opts", [("Cascaded", CascadedOpts(4096, Type.LONGLONG, 1, 1, 1)),
                                      ("Bitcomp", BitcompOpts(0, Type.ULONGLONG)),
                                      ("Bitcomp", BitcompOpts(1, Type.CHAR))])
def test_typed_chunk_size_refused(shim, fmt, opts, chunk):
    """The typed decoders need 8-byte aligned chunk pointers: a manager never accepts a chunk size that breaks them,
    neither at construction nor from a container's header."""
    with pytest.raises(ShimError) as e:
        Manager.create(shim, fmt, opts, chunk, NO_COMPUTE_NO_VERIFY)
    assert e.value.status == Status.ErrorInvalidValue
    mgr = Manager.create(shim, fmt, opts, chunk & ~7, NO_COMPUTE_NO_VERIFY)
    comp = _place(hm.build(fmt, bytes(opts), chunk, 0, []))
    with pytest.raises(ShimError) as e:
        Manager.from_buffer(shim, comp.ptr, NO_COMPUTE_NO_VERIFY)
    assert e.value.status == Status.ErrorInvalidValue
    with pytest.raises(ShimError) as e:
        mgr.configure_decompression(comp.ptr)
    assert e.value.status == Status.ErrorInvalidValue


# (format, writer options, reader options): the reader's own bound is below the writer's streams on random data
CROSS_OPTIONS = {
    "bitcomp_char_by_u64": ("Bitcomp", BitcompOpts(0, Type.CHAR), BitcompOpts(0, Type.ULONGLONG)),
    "cascaded_char512_by_i64": ("Cascaded", CascadedOpts(512, Type.CHAR, 1, 1, 1),
                                CascadedOpts(4096, Type.LONGLONG, 0, 0, 1)),
}


@pytest.mark.parametrize("key", list(CROSS_OPTIONS))
def test_typed_manager_decodes_containers_written_with_other_options(shim, key):
    """A typed manager's options only steer compression: the decoders read everything from the streams, and the size
    table is bounded by the options stored in the header, not by the reading manager's."""
    fmt, wopts, ropts = CROSS_OPTIONS[key]
    chunk, n = 65536, 5 * 65536 + 1000
    data = _random(n, 21)
    comp, _, out = compress(Manager.create(shim, fmt, wopts, chunk, NO_COMPUTE_NO_VERIFY), data, key)
    reader_bound = Codec(fmt, opts=ropts).compress_get_max_output_chunk_size(chunk)
    assert max(hm.parse(comp).sizes) > reader_bound, key         # the case the reader's own bound would refuse
    mgr = Manager.create(shim, fmt, ropts, chunk, NO_COMPUTE_NO_VERIFY)
    dc = mgr.configure_decompression(out.ptr)
    st, back = decompress(mgr, out.ptr, dc, n, key)
    assert st == 0 and back == data, (key, st)
