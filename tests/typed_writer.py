"""Hand-built Cascaded, Bitcomp and ANS streams (test infrastructure, CPU only).

The encoders (this library's and the oracle's) only write the streams they like: minimal bit widths, minima that are
the true minimum, partitions and segments in order, zero pads, nothing after the last byte they need.  The decoders
parse exactly the fields of the stream formats (headers of nvcomp_b200/csrc/{cascaded,bitcomp}.cu and
include/nvcomp/device/detail/ans_impl.cuh), so the writers here take explicit field values and can spell anything the
formats allow -- or, for the invalid list, break one rule at a time.  Every valid case carries the output its fields
stand for, computed here from the fields with Python integers.

VALID / INVALID: name -> Case.  A valid case must decode to `out` at capacity `cap` (and any capacity above); an invalid
case must be rejected at capacity `cap`, and must break only the oracle rules it names: with those rules skipped
(oracle_typed_skip_rules) and its `beyond` bytes placed past its end, the oracle decodes it.  Where one rule cannot be
broken alone the case names the rules it implies too, and the few whose rule-less decode would expand a run of 2^32
or more elements name none.  An invalid case with header=True is rejected by a check of the stream header alone, so
the size query answers 0 for it.  `mutate()` / `corruption_campaign()` draw seeded corruptions of real
encoder streams, aimed at one field class of the layout at a time."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

import typed_model as tm
from typed_model import ANS_L, ANS_M, ANS_MAGIC, ANS_SEG, BTC_MAGIC, CSC_MAGIC, M64, TYPE_SIZE, _r8


@dataclass
class Case:
    codec: str              # "cascaded" | "bitcomp" | "ans"
    comp: bytes
    out: bytes | None       # expected output (None: invalid)
    cap: int                # capacity the case is stated for
    header: bool = False    # invalid: rejected by the stream header alone
    rules: tuple = ()       # invalid: the oracle rules (typed_oracle.c) it breaks; it decodes with them skipped
    beyond: bytes = b""     # invalid: the bytes it lacks past its end (supplied when its rules are skipped)


def _w32(*vs: int) -> bytes:
    return b"".join((v & 0xFFFFFFFF).to_bytes(4, "little") for v in vs)


def _w64(*vs: int) -> bytes:
    return b"".join((v & M64).to_bytes(8, "little") for v in vs)


def pack_bits(vals: list[int], bits: int, nwords: int | None = None) -> bytes:
    """Value k at bits [k*bits, (k+1)*bits) of little-endian u64 words (ceil(len*bits/64) words unless given)."""
    acc = 0
    for k, v in enumerate(vals):
        acc |= (v & ((1 << bits) - 1)) << (k * bits)
    nw = tm._words(len(vals), bits) if nwords is None else nwords
    return acc.to_bytes(8 * nw, "little") if nw else b""


def _store(vals: list[int], ts: int) -> bytes:
    return b"".join((v & ((1 << (8 * ts)) - 1)).to_bytes(ts, "little") for v in vals)


# ------------------------------------------------------------------------------------------------ Cascaded
@dataclass
class Stream:
    """A packed stream: raw values (what the bits hold), the width and the minimum.  count defaults to len(raw)."""
    raw: list[int]
    bits: int
    minv: int = 0
    count: int | None = None
    nwords: int | None = None       # words written (default: the ones count * bits needs)

    def encode(self) -> bytes:
        n = len(self.raw) if self.count is None else self.count
        nw = tm._words(n, self.bits) if self.nwords is None else self.nwords
        return _w32(n, self.bits) + _w64(self.minv) + pack_bits(self.raw, self.bits, nw)

    def values(self) -> list[int]:
        mask = (1 << self.bits) - 1
        return [((r & mask) + self.minv) & M64 for r in self.raw]


@dataclass
class Part:
    """A partition payload: delta bases and element counts, run streams 0 .. R-1, the value stream."""
    runs: list[Stream]
    vals: Stream
    first: list[int] = field(default_factory=list)
    cnt_in: list[int] = field(default_factory=list)
    cnt_pad: int = 0                # the word after an odd number of element counts
    extra: bytes = b""              # bytes after the value stream inside the partition

    def encode(self) -> bytes:
        D = len(self.first)
        b = _w64(*self.first) + _w32(*self.cnt_in) + (_w32(self.cnt_pad) if D % 2 else b"")
        for s in self.runs + [self.vals]:
            b += s.encode()
        b += self.extra
        return b + bytes(_r8(len(b)) - len(b))

    def decode(self, ts: int) -> list[int]:
        """The elements the fields describe: values (raw + min, modulo 2^64), then from the last layer back the delta
        prefix sums (a zero count entering a delta layer: it saw an empty list) and the run expansion."""
        mask = (1 << (8 * ts)) - 1
        cur = [v & mask for v in self.vals.values()]
        R, D = len(self.runs), len(self.first)
        for i in range(max(R, D) - 1, -1, -1):
            if i < D and self.cnt_in[i]:
                acc, nxt = self.first[i], [self.first[i] & mask]
                for d in cur:
                    acc += d
                    nxt.append(acc & mask)
                cur = nxt
            if i < R:
                cur = [v for v, n in zip(cur, self.runs[i].values()) for _ in range(n)]
        return cur


def cascaded_chunk(type_id: int, R: int, D: int, ulen: int, parts: list[bytes], P: int = 4096, use_bp: int = 1,
                   offs: list[int] | None = None, num_parts: int | None = None, hdr_pad: int = 0,
                   tail: bytes | None = None, trailing: bytes = b"", magic: int = CSC_MAGIC) -> bytes:
    """Header, offset table, pad, the partition payloads and the tail word (the ulen % size trailing bytes, zero
    padded) when ulen is not a multiple of the element size.  offs overrides the offset table, num_parts the partition
    count the header states."""
    ts = TYPE_SIZE.get(type_id, 1)
    np_ = len(parts) if num_parts is None else num_parts
    head = _w32(magic, type_id | (R << 8) | (D << 16) | (use_bp << 24), ulen, P, np_)
    off = _r8(20 + 4 * (len(parts) + 1))
    table = [off + sum(len(q) for q in parts[:p]) for p in range(len(parts) + 1)] if offs is None else offs
    body = b"".join(parts)
    b = head + _w32(*table)
    b += _w32(hdr_pad) if len(b) % 8 else b""
    b = b[:off] + bytes(max(0, off - len(b))) + body
    if ulen % ts:
        b += tail if tail is not None else b"\x5a" * (ulen % ts) + bytes(8 - ulen % ts)
    return b + trailing


def _csc(R, D, parts, ts, type_id=4, **kw) -> tuple[bytes, bytes]:
    """A one-or-more-partition chunk and its output (the partitions' elements in order)."""
    out = b"".join(_store(p.decode(ts), ts) for p in parts)
    comp = cascaded_chunk(type_id, R, D, len(out), [p.encode() for p in parts], **kw)
    return comp, out


def _ctl_vals():
    return Stream([5, 7], 32)


def cascaded_valid() -> dict[str, Case]:
    V = {}

    def add(name, comp, out, cap=None):
        V[name] = Case("cascaded", comp, out, len(out) if cap is None else cap)

    add("csc_control", *_csc(1, 0, [Part([Stream([3, 1], 3)], _ctl_vals())], 4))
    add("csc_empty", cascaded_chunk(4, 1, 1, 0, []), b"")
    add("csc_values_0bit_min", *_csc(1, 0, [Part([Stream([3, 1], 3)], Stream([0, 0], 0, 9))], 4))
    add("csc_runs_0bit_min", *_csc(1, 0, [Part([Stream([0, 0], 0, 2)], _ctl_vals())], 4))
    add("csc_runs_wide_33bit", *_csc(1, 0, [Part([Stream([3, 1], 33)], _ctl_vals())], 4))
    add("csc_runs_wide_64bit_min", *_csc(1, 0, [Part([Stream([1, 0], 64, 1 << 1)], _ctl_vals())], 4))
    # raw + min wraps modulo 2^64 back to a small length: legal, and no minimum above the capacity may be rejected
    add("csc_run_min_wraps_2_64", *_csc(1, 0, [Part([Stream([4, 2], 3, M64)], _ctl_vals())], 4))
    add("csc_run_min_wraps_2_64_layer1", *_csc(2, 0, [Part([Stream([1, 1, 1, 1], 1), Stream([4, 2], 3, M64)],
                                                            _ctl_vals())], 4))
    add("csc_no_bp_values_min", *_csc(1, 0, [Part([Stream([3, 1], 16)], Stream([5, 7], 32, 1000))], 4, use_bp=0))
    # delta base and values above the element width (truncated on store)
    add("csc_delta_first_wide_u8", *_csc(1, 1, [Part([Stream([2, 1, 3], 2)], Stream([0x1FF, 0x301], 16),
                                                      first=[0x123456F0], cnt_in=[3])], 1, type_id=1))
    add("csc_delta_values_wide_i16", *_csc(0, 1, [Part([], Stream([0x10001, 0x7FFFF, 2], 20, 5),
                                                       first=[0xABCD0000FFFF], cnt_in=[4])], 2, type_id=2))
    add("csc_values_wide_u64_min", *_csc(1, 0, [Part([Stream([1, 2], 2)], Stream([1, 3], 2, M64 - 1))], 8,
                                         type_id=7))
    add("csc_deep_layers", *_csc(3, 2, [Part([Stream([2, 1, 1, 3, 1], 2), Stream([1, 2, 1], 2), Stream([2], 2)],
                                             Stream([4], 8), first=[9, 100], cnt_in=[5, 3])], 4))
    # partition p spans [part_off[p], part_off[p + 1]): the table chains the partitions, so they lie in order and
    # apart; what the format leaves open is slack after the streams of a partition
    full = Part([Stream([100, 28], 7)], Stream([1, 2], 2), extra=b"\x13" * 40)     # 128 INT elements
    last = Part([Stream([5], 3)], Stream([3], 2))
    add("csc_two_parts_slack", *_csc(1, 0, [full, last], 4, P=512))
    add("csc_trailing_bytes", *_csc(1, 0, [Part([Stream([3, 1], 3)], _ctl_vals())], 4, trailing=b"\xff" * 13))
    comp = cascaded_chunk(4, 1, 0, 19, [Part([Stream([3, 1], 3)], _ctl_vals()).encode()], trailing=b"\x77" * 9)
    add("csc_tail_word_and_trailing", comp, _store([5, 5, 5, 7], 4) + b"\x5a" * 3)
    add("csc_pad_nonzero", *_csc(1, 0, [Part([Stream([3, 1], 3)], _ctl_vals())], 4, hdr_pad=0xDEADBEEF))
    add("csc_partition_extra_bytes", *_csc(1, 1, [Part([Stream([3, 1], 3)], Stream([2], 32), first=[5], cnt_in=[2],
                                                       cnt_pad=0x1234, extra=b"\xee" * 24)], 4))
    return V


def cascaded_invalid() -> dict[str, Case]:
    """One case per rejection rule of oracle_cascaded_decompress.  Each is a stream that decodes with the rules it
    names (Case.rules) switched off, and the bytes it lacks past its end (Case.beyond) supplied: it breaks those
    rules and no other."""
    I = {}

    def add(name, comp, cap=16, header=False, rules=None, beyond=b""):
        I[name] = Case("cascaded", comp, None, cap, header, (name,) if rules is None else rules, beyond)

    ctl = Part([Stream([3, 1], 3)], _ctl_vals()).encode()                  # [5, 5, 5, 7] at offset 32
    n_ctl = 32 + len(ctl)

    def chunk(part=None, **kw):
        kw.setdefault("ulen", 16)
        parts = kw.pop("parts") if "parts" in kw else [part or ctl]
        return cascaded_chunk(kw.pop("type_id", 4), kw.pop("R", 1), kw.pop("D", 0), parts=parts, **kw)

    def run_part(*runs, vals=None, **kw):
        return Part(list(runs), vals or _ctl_vals(), **kw).encode()

    good = chunk()
    empty = cascaded_chunk(4, 1, 0, 0, [])
    # every stream shorter than 20 bytes is also shorter than its offset table
    add("csc_stream_shorter_than_header", empty[:19], header=True, beyond=empty[19:],
        rules=("csc_stream_shorter_than_header", "csc_offset_table_beyond_stream"))
    add("csc_magic", chunk(magic=CSC_MAGIC ^ 1), header=True)
    add("csc_type", chunk(Part([Stream([12, 4], 4)], Stream([5, 7], 8)).encode(), type_id=8), header=True)
    add("csc_R_above_7", chunk(Part([Stream([4], 3)] + [Stream([1], 1)] * 7, Stream([5], 8)).encode(), R=8),
        header=True)
    add("csc_D_above_7", chunk(Part([], Stream([], 0), first=list(range(1, 9)), cnt_in=list(range(8, 0, -1))).encode(),
                               R=0, D=8, ulen=32), cap=32, header=True)
    add("csc_part_size_below_512", chunk(P=504), header=True)
    add("csc_part_size_above_16384", chunk(P=16392), header=True)
    add("csc_part_size_not_multiple_of_8", chunk(P=4092), header=True)
    full = Part([Stream([128], 8)], Stream([9], 4)).encode()               # 128 INT elements
    add("csc_num_parts_too_small", chunk(full, P=512, ulen=528), cap=528, header=True)
    add("csc_num_parts_too_large", chunk(parts=[ctl, Part([Stream([1024], 11)], Stream([9], 4)).encode()]),
        header=True)
    add("csc_offset_table_beyond_stream", empty[:20], header=True, beyond=empty[20:])
    add("csc_n_above_capacity", good, cap=15)
    add("csc_offset_misaligned", chunk(b"\0" * 4 + ctl, offs=[36, 36 + len(ctl)]))
    # partition 1 laid out first: partition 0 runs from a later offset to an earlier one
    small = Part([Stream([3, 1], 3)], _ctl_vals()).encode()
    add("csc_offset_decreasing", cascaded_chunk(4, 1, 0, 528, [small + full], P=512, num_parts=2,
                                                offs=[32 + len(small), 32, 32 + len(small) + len(full)]), cap=528)
    add("csc_offset_beyond_stream", chunk(offs=[32, n_ctl + 8]), beyond=bytes(8))
    add("csc_part_shorter_than_delta_header",
        chunk(run_part(Stream([3, 1], 3), vals=Stream([2], 32), first=[5], cnt_in=[2]), D=1, offs=[32, 40]))
    # a stream header cut by the partition end leaves no room for its words either
    hdr_rules = ("csc_stream_header_truncated", "csc_stream_words_past_partition")
    add("csc_run_header_truncated", chunk(offs=[32, 40]), rules=hdr_rules)
    add("csc_value_header_truncated", chunk(offs=[32, 32 + 24 + 8]), rules=hdr_rules)
    add("csc_run_bits_above_64", chunk(run_part(Stream([0, 0], 65, 2, nwords=3))), rules=("csc_stream_bits_above_64",))
    add("csc_value_bits_above_64", chunk(run_part(Stream([3, 1], 3), vals=Stream([0, 0], 65, 5, nwords=3))),
        rules=("csc_stream_bits_above_64",))
    add("csc_run_words_past_partition", chunk(offs=[32, 48]), rules=("csc_stream_words_past_partition",))
    add("csc_value_words_past_partition", chunk(offs=[32, 32 + 24 + 16]), rules=("csc_stream_words_past_partition",))
    # more values than the partition holds can only expand to the wrong element count
    add("csc_value_count_above_partition", chunk(Part([], Stream([1] * 129, 1)).encode(), P=512, R=0, ulen=512),
        cap=512, rules=("csc_value_count_above_partition", "csc_total_not_partition"))
    add("csc_delta_count_zero_with_values",
        chunk(Part([], Stream([5, 5, 5, 7], 32), first=[0], cnt_in=[0]).encode(), R=0, D=1))
    add("csc_delta_count_not_values_plus_1",
        chunk(run_part(Stream([3, 1], 3), vals=Stream([2], 32), first=[5], cnt_in=[3]), D=1))
    add("csc_delta_count_above_partition",
        chunk(Part([], Stream([0] * 128, 0), first=[1], cnt_in=[129]).encode(), P=512, R=0, D=1, ulen=512), cap=512,
        rules=("csc_delta_count_above_partition", "csc_total_not_partition"))
    add("csc_run_count_not_value_count", chunk(run_part(Stream([3, 1, 0], 3))))
    add("csc_runs_total_above_partition", chunk(run_part(Stream([100, 29], 7)), P=512, ulen=512), cap=512,
        rules=("csc_runs_total_above_partition", "csc_total_not_partition"))
    add("csc_runs_total_not_partition", chunk(run_part(Stream([2, 1], 3))), rules=("csc_total_not_partition",))
    tailed = chunk(ulen=19)
    add("csc_tail_word_missing", tailed[:-8], cap=19, beyond=tailed[-8:])
    # run lengths the format forbids, each on the control chunk with only the run stream changed: zero, and lengths of
    # 2^32 and more that a 32-bit path would truncate or wrap (raw + min wraps modulo 2^64 only), at layer 0 (the fused
    # path) and at layer 1 / a wide layer 0 (the generic path).  The lengths above the capacity break the capacity rule
    # alone (csc_runs_total_above_partition shows it decodes without), but skipping that rule here would expand a run
    # of 2^32 or more elements: rules=().
    add("csc_run_zero_length", chunk(run_part(Stream([0, 4], 3))))
    add("csc_run_min_above_capacity", chunk(run_part(Stream([0, 0], 0, (1 << 32) + 2))), rules=())
    add("csc_run_length_wraps_32", chunk(run_part(Stream([M64 >> 32] * 2, 32, 3))), rules=())
    add("csc_run_min_wraps_past_capacity", chunk(run_part(Stream([2, 0], 2, M64))), rules=())
    ones = Stream([1, 1, 1, 1], 1)
    add("csc_run_zero_length_layer1", chunk(run_part(ones, Stream([0, 4], 3)), R=2), rules=("csc_run_zero_length",))
    add("csc_run_min_above_capacity_layer1", chunk(run_part(ones, Stream([1, 1], 1, (1 << 32) + 1)), R=2), rules=())
    add("csc_run_length_wraps_32_layer1", chunk(run_part(ones, Stream([M64 >> 32] * 2, 32, 3)), R=2), rules=())
    add("csc_run_zero_length_wide", chunk(run_part(Stream([0, 4], 33))), rules=("csc_run_zero_length",))
    return I

# ------------------------------------------------------------------------------------------------- Bitcomp
@dataclass
class Block:
    """algo 0: desc (bits in the low byte), the first element and the zig-zag codes of slots 0..127.
    algo 1: desc (nz | bits << 8), the 128-bit mask and the packed values (in mask order)."""
    desc: int
    head: int                       # first element (algo 0) / mask (algo 1)
    codes: list[int]
    nwords: int | None = None

    def encode(self, algo: int) -> bytes:
        if algo == 0:
            bits = self.desc & 0xFF
            return _w64(self.head) + pack_bits(self.codes, bits, 2 * bits if self.nwords is None else self.nwords)
        nz, bits = self.desc & 0xFF, self.desc >> 8
        nw = tm._words(nz, bits) if self.nwords is None else self.nwords
        return _w64(self.head & M64, self.head >> 64) + pack_bits(self.codes, bits, nw)

    def decode(self, algo: int, nv: int) -> list[int]:
        if algo == 0:
            mask = (1 << (self.desc & 0xFF)) - 1
            acc, out = self.head, []
            for z in self.codes[:nv]:
                z &= mask
                acc += (z >> 1) ^ -(z & 1)
                out.append(acc & M64)
            return out
        mask = (1 << (self.desc >> 8)) - 1
        out, rank = [], 0
        for k in range(nv):
            if (self.head >> k) & 1:
                out.append(self.codes[rank] & mask if rank < len(self.codes) else 0)
                rank += 1
            else:
                out.append(0)
        return out


def bitcomp_chunk(algo: int, type_id: int, ulen: int, blocks: list[Block], nblocks: int | None = None,
                  desc_pad: bytes | None = None, tail: bytes | None = None, trailing: bytes = b"",
                  magic: int = BTC_MAGIC, cfg_hi: int = 0) -> bytes:
    nb = len(blocks) if nblocks is None else nblocks
    b = _w32(magic, algo | (type_id << 8) | (cfg_hi << 16), ulen, nb)
    b += b"".join((blk.desc & 0xFFFF).to_bytes(2, "little") for blk in blocks)
    pad = _r8(len(b)) - len(b)
    b += (desc_pad or bytes(pad))[:pad]
    b += b"".join(blk.encode(algo) for blk in blocks)
    ts = TYPE_SIZE.get(type_id, 1)
    if ulen % ts:
        b += tail if tail is not None else b"\xa7" * (ulen % ts) + bytes(8 - ulen % ts)
    return b + trailing


def _btc(algo, type_id, blocks, ne, tail_bytes=0, **kw) -> tuple[bytes, bytes]:
    ts = TYPE_SIZE[type_id]
    vals = []
    for k, blk in enumerate(blocks):
        vals += blk.decode(algo, min(128, ne - 128 * k))
    out = _store(vals, ts) + b"\xa7" * tail_bytes
    return bitcomp_chunk(algo, type_id, len(out), blocks, **kw), out


def _zz(d: int) -> int:
    return 2 * d if d >= 0 else -2 * d - 1


def _a0(first: int, deltas: list[int], bits: int, hi: int = 0) -> Block:
    codes = [0] + [_zz(d) for d in deltas]
    return Block(bits | (hi << 8), first, codes + [0] * (128 - len(codes)))


def _a1(vals: list[int], bits: int, extra_mask: int = 0, extra: list[int] = ()) -> Block:
    """algo 1 block of vals (zero = unset slot) plus mask bits `extra_mask` set past them with values `extra`."""
    mask = sum(1 << k for k, v in enumerate(vals) if v) | extra_mask
    nzv = [v for v in vals if v] + list(extra)
    return Block(len(nzv) | (bits << 8), mask, nzv)


def bitcomp_valid() -> dict[str, Case]:
    V = {}
    rng = np.random.default_rng(11)

    def add(name, comp, out):
        V[name] = Case("bitcomp", comp, out, len(out))

    add("btc_empty", *_btc(0, 5, [], 0))
    add("btc_algo0_desc_high_byte", *_btc(0, 5, [_a0(1000, [1, -1, 3] * 42, 3, hi=0xA5)], 127))
    add("btc_algo0_64bit_deltas", *_btc(0, 7, [_a0(M64 - 5, [-(1 << 62), 1 << 62, -(1 << 63)] * 10, 64)], 31))
    add("btc_algo0_first_wider_than_type", *_btc(0, 1, [_a0(0xDEADBEEF12, [2, -3] * 10, 3)], 21))
    add("btc_algo0_zero_width", *_btc(0, 3, [_a0(0xFFFF1234, [], 0)] * 2, 200, tail_bytes=1))
    # algo 1: mask bits set past the valid elements of the last block, counted in nz (their values are not output)
    add("btc_algo1_mask_past_valid", *_btc(1, 4, [_a1([0, 3, 0, 9, 1], 4, (1 << 10) | (1 << 100), [7, 15])], 5))
    add("btc_algo1_values_wider_than_type", *_btc(1, 1, [_a1([0x1FF, 0, 0xABC, 0x100] * 32, 12)], 128))
    add("btc_algo1_zero_width_mask", *_btc(1, 5, [Block(3, 0b10101, [])], 9))
    add("btc_desc_pad_and_trailing", *_btc(0, 5, [_a0(7, [1] * 127, 2)] * 3, 300, desc_pad=b"\xff\xee",
                                            trailing=b"\x42" * 11))
    # more than 512 blocks: an offset tile of 8-byte payloads (staged) and one of 40-byte payloads (20 KB: not staged),
    # then a short tile
    blocks = []
    for k in range(1100):
        if k < 512:
            blocks.append(_a0(k * 1000, [], 0))
        elif k < 1024:
            blocks.append(_a0(k, [int(x) for x in rng.integers(-1, 2, 127)], 2))
        else:
            blocks.append(_a0(k, [int(x) for x in rng.integers(-4, 4, 127)], 4))
    add("btc_tiles_staged_and_unstaged", *_btc(0, 6, blocks, 1100 * 128 - 77))
    blocks = [_a1([int(x) for x in rng.integers(0, 3, 128)], 2) for _ in range(600)]
    add("btc_algo1_600_blocks", *_btc(1, 2, blocks, 600 * 128))
    return V


def bitcomp_invalid() -> dict[str, Case]:
    """One case per rejection rule of oracle_bitcomp_decompress (see cascaded_invalid)."""
    I = {}

    def add(name, comp, cap, header=False, rules=None, beyond=b""):
        I[name] = Case("bitcomp", comp, None, cap, header, (name,) if rules is None else rules, beyond)

    b0 = _a0(50, [1, -2] * 60, 3)
    good = bitcomp_chunk(0, 5, 512, [b0])
    empty = bitcomp_chunk(0, 5, 0, [])
    # a stream shorter than its header, or than its descriptor table, is also shorter than the first block payload
    add("btc_stream_shorter_than_header", empty[:15], 0, header=True, beyond=empty[15:],
        rules=("btc_stream_shorter_than_header", "btc_desc_table_beyond_stream"))
    add("btc_magic", bitcomp_chunk(0, 5, 512, [b0], magic=0), 512, header=True)
    add("btc_type", bitcomp_chunk(0, 9, 512, [_a0(1, [], 0)] * 4), 512, header=True)
    a1 = _a1([3, 0, 5, 1] * 32, 3)
    add("btc_algo_above_1", bitcomp_chunk(2, 5, 512, [a1]), 512, header=True)
    add("btc_nblocks_mismatch", bitcomp_chunk(0, 5, 512, [b0, b0]), 512, header=True)
    add("btc_desc_table_beyond_stream", good[:17], 512, header=True, beyond=good[17:],
        rules=("btc_desc_table_beyond_stream", "btc_payload_beyond_stream"))
    add("btc_n_above_capacity", good, 511)
    add("btc_algo0_bits_above_64", bitcomp_chunk(0, 7, 1024, [Block(65, 1, [0] * 128, nwords=130)]), 1024)
    add("btc_algo0_payload_beyond_stream", good[:-8], 512, beyond=good[-8:], rules=("btc_payload_beyond_stream",))
    g1 = bitcomp_chunk(1, 5, 512, [a1])
    add("btc_algo1_payload_beyond_stream", g1[:-8], 512, beyond=g1[-8:], rules=("btc_payload_beyond_stream",))
    # a 128-bit mask cannot hold more than 128 set bits
    add("btc_algo1_nz_above_128", bitcomp_chunk(1, 5, 512, [Block(129 | (1 << 8), (1 << 128) - 1, [1] * 129)]), 512,
        rules=("btc_algo1_nz_above_128", "btc_algo1_popcount_not_nz"))
    add("btc_algo1_bits_above_64", bitcomp_chunk(1, 5, 512, [Block(1 | (65 << 8), 1, [0], nwords=2)]), 512)
    # the extra mask bit lies past the 5 valid elements: nothing but the count check notices it
    r = _a1([3, 0, 5, 1, 2], 3)
    add("btc_algo1_popcount_not_nz", bitcomp_chunk(1, 5, 20, [Block(r.desc, r.head | (1 << 100), r.codes)]), 20)
    tailed = bitcomp_chunk(0, 5, 515, [b0])
    add("btc_tail_word_missing", tailed[:-8], 515, beyond=tailed[-8:])
    return I

# ----------------------------------------------------------------------------------------------------- ANS
def ans_chunk(n: int, mode: int = 0, nseg: int | None = None, freq: list[int] | None = None,
              segs: list[bytes] = (), offs: list[int] | None = None, trailing: bytes = b"", payload: bytes = b"",
              magic: int = ANS_MAGIC) -> bytes:
    """Mode 0: header, frequency table, segment offsets (offs overrides them) and the segments; modes 1 and 2: the
    header and `payload`."""
    ns = len(segs) if nseg is None else nseg
    b = _w32(magic, n, mode, ns)
    if mode != 0:
        return b + payload + trailing
    b += b"".join(f.to_bytes(2, "little") for f in freq)
    start = (528 + 4 * (len(segs) + 1 if offs is None else len(offs)) + 3) & ~3
    table = [start + sum(len(s) for s in segs[:k]) for k in range(len(segs) + 1)] if offs is None else offs
    b += _w32(*table)
    return b + bytes(start - len(b)) + b"".join(segs) + trailing


def ans_segment(states: list[int], words: list[int], extra_words: list[int] = (), pad: bool = True) -> bytes:
    ws = list(words) + list(extra_words)
    b = _w32(*states) + b"".join(w.to_bytes(2, "little") for w in ws)
    return b + (bytes(2) if pad and len(ws) % 2 else b"")


def _ans_segs(data: bytes, freq: list[int]) -> list[tuple[list[int], list[int]]]:
    return [tm.ans_encode_segment(data[k:k + ANS_SEG], freq) for k in range(0, len(data), ANS_SEG)]


def _sample(rng, n: int, k: int) -> bytes:
    return np.minimum(rng.geometric(0.25, n) - 1, k - 1).astype(np.uint8).tobytes()


def ans_valid() -> dict[str, Case]:
    V = {}
    rng = np.random.default_rng(13)

    def add(name, comp, out):
        V[name] = Case("ans", comp, out, len(out))

    freq = [0] * 256
    freq[0], freq[1] = 4000, 96
    add("ans_mode0_n0", ans_chunk(0, freq=freq), b"")
    data = _sample(rng, 3000, 6)
    _, f = tm.ans_freq(data)
    # symbols 200 and 201 get frequency but never occur
    f2 = list(f)
    f2[int(np.argmax(f2))] -= 7
    f2[200], f2[201] = 3, 4
    segs = [ans_segment(*s) for s in _ans_segs(data, f2)]
    add("ans_freq_without_occurrence", ans_chunk(len(data), freq=f2, segs=segs), data)
    st, ws = _ans_segs(data, f)[0]
    add("ans_one_leftover_word", ans_chunk(len(data), freq=f,
                                           segs=[ans_segment(st, ws, [0xBEEF] if len(ws) % 2 == 0 else [], pad=False)]),
        data)
    for k in range(11, 40):                     # the first alphabet whose first segment has an odd word count
        big = _sample(rng, 2 * ANS_SEG + 999, k)
        _, f = tm.ans_freq(big)
        if len(_ans_segs(big, f)[0][1]) % 2:
            break
    # segment sg spans [seg_off[sg], seg_off[sg + 1]): the table chains the segments, so they lie in order; a segment
    # before the last may still end in one leftover word (the 4-byte alignment of the next one leaves room for it
    # after an odd word count), and its content is free
    segs = [ans_segment(st, ws, [0x5A5A] if len(ws) % 2 else [], pad=False) for st, ws in _ans_segs(big, f)]
    assert any(len(ws) % 2 for _, ws in _ans_segs(big, f))
    add("ans_segments_leftover_words", ans_chunk(len(big), freq=f, segs=segs), big)
    add("ans_trailing_bytes", ans_chunk(len(data), freq=tm.ans_freq(data)[1],
                                        segs=[ans_segment(*s) for s in _ans_segs(data, tm.ans_freq(data)[1])],
                                        trailing=b"\x99" * 10), data)
    add("ans_mode1_nseg", ans_chunk(5, mode=1, nseg=77, payload=b"hello", trailing=b"!!"), b"hello")
    add("ans_mode2_nseg", ans_chunk(1000, mode=2, nseg=3, payload=b"\x07", trailing=b"\x01\x02"), b"\x07" * 1000)
    add("ans_mode1_empty", ans_chunk(0, mode=1), b"")
    return V


def ans_invalid() -> dict[str, Case]:
    """One case per rejection rule of oracle_ans_decompress (see cascaded_invalid)."""
    I = {}
    rng = np.random.default_rng(17)

    def add(name, comp, cap, header=False, rules=None, beyond=b""):
        I[name] = Case("ans", comp, None, cap, header, (name,) if rules is None else rules, beyond)

    for k in range(9, 40):                      # the first alphabet whose segment has an even word count (no pad)
        data = _sample(rng, 2000, k)
        _, f = tm.ans_freq(data)
        (st, ws), = _ans_segs(data, f)
        if len(ws) % 2 == 0:
            break
    seg = ans_segment(st, ws)
    good = ans_chunk(len(data), freq=f, segs=[seg])
    n = len(data)
    o0 = (528 + 8 + 3) & ~3                     # the segment of a one-segment stream
    stored0 = ans_chunk(0, mode=1)
    # 15 bytes are too short for any mode: the empty stored stream is the shortest stream there is
    add("ans_stream_shorter_than_header", stored0[:15], 0, header=True, beyond=stored0[15:],
        rules=("ans_stream_shorter_than_header", "ans_mode1_short"))
    add("ans_magic", ans_chunk(n, freq=f, segs=[seg], magic=ANS_MAGIC + 1), n, header=True)
    add("ans_mode_above_2", ans_chunk(n, mode=3, nseg=1, payload=good[16:]), n, header=True)
    add("ans_mode1_short", ans_chunk(n, mode=1, payload=data[:-1]), n, header=True, beyond=data[-1:])
    add("ans_mode2_short", ans_chunk(n, mode=2), n, header=True, beyond=b"\x07")
    # a second segment of 16384 symbols, which the rule-less decoder writes past n
    seg2 = ans_segment(*tm.ans_encode_segment((data * 9)[:ANS_SEG], f))
    add("ans_nseg_mismatch", ans_chunk(n, freq=f, segs=[seg, seg2]), n, header=True)
    empty0 = ans_chunk(0, freq=f)
    add("ans_header_beyond_stream", empty0[:530], 0, header=True, beyond=empty0[530:])
    add("ans_n_above_capacity", good, n - 1)
    f3 = list(f)
    f3[int(np.argmax(f3))] -= 1                 # the table sums to 4095; the segment is coded with it
    add("ans_freq_sum_not_4096", ans_chunk(n, freq=f3, segs=[ans_segment(*_ans_segs(data, f3)[0])]), n)
    f4 = [0] * 256
    f4[3] = ANS_M                               # one symbol: states stay at 2^16, no words
    add("ans_single_freq_4096", ans_chunk(100, freq=f4, segs=[ans_segment([ANS_L] * 32, [])]), 100)
    add("ans_seg_offset_misaligned", ans_chunk(n, freq=f, segs=[bytes(2) + seg], offs=[o0 + 2, o0 + 2 + len(seg)]), n)
    # segment 1 laid out first: segment 0 runs from a later offset to an earlier one, which also leaves both word
    # counts wrong
    big = _sample(rng, ANS_SEG + 500, 9)
    _, fb = tm.ans_freq(big)
    s0, s1 = (ans_segment(*s) for s in _ans_segs(big, fb))
    b0 = (528 + 12 + 3) & ~3
    add("ans_seg_offset_decreasing", ans_chunk(len(big), nseg=2, freq=fb, segs=[s1 + s0],
                                               offs=[b0 + len(s1), b0, b0 + len(s1) + len(s0)]), len(big),
        rules=("ans_seg_offset_decreasing", "ans_two_leftover_words"))
    add("ans_seg_offset_past_end", ans_chunk(n, freq=f, segs=[seg], offs=[o0, o0 + len(seg) + 2]), n, beyond=bytes(2))
    # a segment shorter than its 128 bytes of states has a negative word count
    add("ans_seg_shorter_than_128", ans_chunk(n, freq=f, segs=[seg], offs=[o0, o0 + 124]), n,
        rules=("ans_seg_shorter_than_128", "ans_two_leftover_words"))
    # the last word lies just past the segment end; reading it leaves the word count negative
    add("ans_words_exhausted", ans_chunk(n, freq=f, segs=[seg], offs=[o0, o0 + len(seg) - 2]), n,
        rules=("ans_words_exhausted", "ans_two_leftover_words"))
    add("ans_two_leftover_words", ans_chunk(n, freq=f, segs=[ans_segment(st, ws, [1, 2], pad=False)]), n)
    st2, ws2 = tm.ans_encode_segment(data, f, start=[ANS_L + 1] + [ANS_L] * 31)
    add("ans_final_state_not_L", ans_chunk(n, freq=f, segs=[ans_segment(st2, ws2)]), n)
    return I

def valid_cases() -> dict[str, Case]:
    return {**cascaded_valid(), **bitcomp_valid(), **ans_valid()}


def invalid_cases() -> dict[str, Case]:
    return {**cascaded_invalid(), **bitcomp_invalid(), **ans_invalid()}


VALID = valid_cases()
INVALID = invalid_cases()


# ------------------------------------------------------------------------------------------------ faithfulness
def cascaded_from_fields(data: bytes, type_id: int, part: int, R: int, D: int, use_bp: int) -> bytes:
    """The stream an encoder writes for `data`, built by this writer from the fields typed_model predicts."""
    ts = TYPE_SIZE[type_id]
    per = part // ts
    ev = tm.elements(data, ts)
    parts = []
    for p in range(0, len(ev), per):
        first, cnt_in, run_lists, cur = tm.cascaded_layers(ev[p:p + per], ts, R, D)
        runs = []
        for ls in run_lists:
            c, bits, mn = tm._stream_hdr(ls, bool(use_bp), False, 2, 16)
            runs.append(Stream([(v - mn) & M64 for v in ls], bits, mn))
        signed = D > 0 or type_id in tm.SIGNED
        c, bits, mn = tm._stream_hdr(cur, bool(use_bp), signed, ts, 8 * ts)
        xs = [tm._signed(v, ts) if signed and use_bp else v for v in cur]
        parts.append(Part(runs, Stream([(x - mn) & M64 for x in xs], bits, mn), first, cnt_in).encode())
    tail = len(data) % ts
    return cascaded_chunk(type_id, R, D, len(data), parts, P=part, use_bp=use_bp,
                          tail=data[len(data) - tail:] + bytes(8 - tail) if tail else None)


def bitcomp_from_fields(data: bytes, algo: int, type_id: int) -> bytes:
    ts = TYPE_SIZE[type_id]
    mask = (1 << (8 * ts)) - 1
    ev = tm.elements(data, ts)
    descs = tm.bitcomp_model(data, algo, type_id)["descs"]
    blocks = []
    for k, desc in enumerate(descs):
        blk = ev[128 * k:128 * k + 128]
        if algo == 0:
            codes = [0] + [tm._zigzag((b - a) & mask, ts) for a, b in zip(blk, blk[1:])]
            blocks.append(Block(desc, blk[0], codes + [0] * (128 - len(codes))))
        else:
            blocks.append(Block(desc, sum(1 << i for i, v in enumerate(blk) if v), [v for v in blk if v]))
    tail = len(data) % ts
    return bitcomp_chunk(algo, type_id, len(data), blocks,
                         tail=data[len(data) - tail:] + bytes(8 - tail) if tail else None)


def ans_from_fields(data: bytes) -> bytes:
    m = tm.ans_model(data)
    _, n, mode, _ = m["header"]
    if mode == 2:
        return ans_chunk(n, mode=2, payload=bytes([m["symbol"]]))
    if mode == 1:
        return ans_chunk(n, mode=1, payload=data)
    return ans_chunk(n, freq=m["freq"], segs=[ans_segment(*s) for s in _ans_segs(data, m["freq"])])


# ------------------------------------------------------------------------------------------------ corruption
CLASSES = {"cascaded": ["header", "table", "stream_header", "payload", "trunc", "extend", "swap"],
           "bitcomp": ["header", "table", "stream_header", "payload", "trunc", "extend"],
           "ans": ["header", "freq", "table", "stream_header", "payload", "trunc", "extend", "swap"]}


def layout(codec: str, b: bytes) -> dict[str, list[tuple[int, int]]]:
    """Byte spans of each field class of a well-formed stream: header words, the offset / descriptor table, the stream
    headers (Cascaded delta bases, counts and packed-stream headers; Bitcomp first elements and masks; ANS states), the
    frequency table (ANS) and the packed payload."""
    spans = {k: [] for k in ("header", "table", "stream_header", "freq", "payload")}
    if codec == "cascaded":
        spans["header"].append((0, 20))
        if len(b) < 20:
            return spans
        m = tm.parse_cascaded(b)
        _, cfg, _, _, npart = m["header"]
        R, D = (cfg >> 8) & 0xFF, (cfg >> 16) & 0xFF
        spans["table"].append((20, 20 + 4 * (npart + 1)))
        for o, pm in zip(m["part_off"], m["parts"]):
            q = o + 8 * D + _r8(4 * D)
            spans["stream_header"].append((o, q))
            for c, bits, _ in pm["runs"] + [pm["vals"]]:
                spans["stream_header"].append((q, q + 16))
                w = 8 * tm._words(c, bits)
                if w:
                    spans["payload"].append((q + 16, q + 16 + w))
                q += 16 + w
        return spans
    if codec == "bitcomp":
        m = tm.parse_bitcomp(b)
        spans["header"].append((0, 16))
        nb = m["header"][3]
        algo = m["header"][1] & 0xFF
        spans["table"].append((16, 16 + 2 * nb))
        q = _r8(16 + 2 * nb)
        for d in m["descs"]:
            h = 8 if algo == 0 else 16
            sz = tm.bitcomp_block_bytes(algo, d)
            spans["stream_header"].append((q, q + h))
            if sz > h:
                spans["payload"].append((q + h, q + sz))
            q += sz
        return spans
    m = tm.parse_ans(b)
    spans["header"].append((0, 16))
    if m["header"][2] != 0:
        if len(b) > 16:
            spans["payload"].append((16, len(b)))
        return spans
    spans["freq"].append((16, 528))
    nseg = m["header"][3]
    spans["table"].append((528, 528 + 4 * (nseg + 1)))
    for o0, o1 in zip(m["seg_off"], m["seg_off"][1:]):
        spans["stream_header"].append((o0, o0 + 128))
        if o1 > o0 + 128:
            spans["payload"].append((o0 + 128, o1))
    return spans


def mutate(rng, codec: str, comp: bytes) -> tuple[str, bytes]:
    """One seeded corruption of a valid stream, aimed at one field class: bit flips inside the header words, the offset
    / descriptor table, the stream headers, the ANS frequency table or the payload; a truncation; appended bytes; or two
    partition / segment offsets swapped.  A class the stream does not have falls back to a payload flip."""
    kind = CLASSES[codec][int(rng.integers(0, len(CLASSES[codec])))]
    b = bytearray(comp)
    spans = layout(codec, comp)
    if kind == "trunc":
        return kind, bytes(b[:int(rng.integers(0, len(b)))])
    if kind == "extend":
        return kind, bytes(b) + rng.integers(0, 256, int(rng.integers(1, 17)), dtype=np.uint8).tobytes()
    if kind == "swap":
        lo, hi = spans["table"][0] if spans["table"] else (0, 0)
        ne = (hi - lo) // 4
        if ne >= 3:
            i, j = (int(x) for x in rng.choice(ne, 2, replace=False))
            a, c = b[lo + 4 * i:lo + 4 * i + 4], b[lo + 4 * j:lo + 4 * j + 4]
            b[lo + 4 * i:lo + 4 * i + 4], b[lo + 4 * j:lo + 4 * j + 4] = c, a
            return kind, bytes(b)
        kind = "header"
    sp = [(s, min(e, len(b))) for s, e in spans[kind] if min(e, len(b)) > s]
    if not sp:
        kind = "payload"
        sp = [(s, min(e, len(b))) for s, e in spans["payload"] if min(e, len(b)) > s] or [(0, len(b))]
    for _ in range(int(rng.integers(1, 4))):
        s, e = sp[int(rng.integers(0, len(sp)))]
        i = int(rng.integers(s, e))
        b[i] ^= 1 << int(rng.integers(0, 8))
    return kind, bytes(b)


def campaign_sources(seed: int = 0) -> dict[str, list[tuple[str, bytes, bytes]]]:
    """Per codec: (config, raw chunk, oracle-encoder stream) over several configurations and the edge inputs of
    typed_model.  The oracle's streams are the encoders' streams (test_typed_sweep_gpu pins the GPU encoder to them)."""
    from conftest import Oracle
    o = Oracle()
    out = {"cascaded": [], "bitcomp": [], "ans": []}
    for type_id, part, R, D, bp in ((4, 4096, 1, 0, 1), (6, 4096, 1, 1, 1), (1, 512, 2, 1, 1), (3, 1024, 0, 2, 1),
                                    (5, 2048, 3, 2, 0), (7, 8192, 1, 1, 0)):
        for name, raw in tm.edge_chunks(type_id, part, seed):
            cfg = f"t{type_id}_p{part}_R{R}D{D}bp{bp}"
            out["cascaded"].append((f"{cfg}/{name}", raw, o.compress_typed(
                "cascaded", raw, chunk_size=part, type=type_id, num_RLEs=R, num_deltas=D, use_bp=bp)))
    for algo, type_id in ((0, 1), (0, 6), (1, 4), (1, 3)):
        for name, raw in tm.bitcomp_edge_chunks(type_id, seed):
            out["bitcomp"].append((f"a{algo}_t{type_id}/{name}", raw,
                                   o.compress_typed("bitcomp", raw, algo=algo, type=type_id)))
    for name, raw in tm.ans_edge_chunks(seed, big=False):
        out["ans"].append((name, raw, o.compress_typed("ans", raw)))
    return out


def corruption_campaign(sources, codec: str, n: int = 3000, seed: int = 5) -> list[tuple[str, str, bytes, int]]:
    """n seeded corruptions of `codec`'s source streams: (source name, field class, stream, raw length)."""
    rng = np.random.default_rng(seed)
    src = sources[codec]
    out = []
    for i in range(n):
        name, raw, comp = src[int(rng.integers(0, len(src)))]
        kind, bad = mutate(rng, codec, comp)
        out.append((name, kind, bad, len(raw)))
    return out
