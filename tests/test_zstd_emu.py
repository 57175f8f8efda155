"""CPU: the warp-level Zstandard decoder of nvcomp_b200/csrc (zstd_decode.cuh) executed in the host warp emulator
(tests/emu: 32 fibers, rendezvous at every warp intrinsic, bounds-checked shared and vector accesses, guard pages
around the global buffers), with libzstd as the oracle.  The hand-built streams of tests/zstd_writer.py are pinned to
libzstd first, so every verdict here is libzstd's."""
import ctypes as C
import os
import subprocess

import pytest

import zstd_writer as W
from conftest import ROOT, sample_inputs

INPUTS = sample_inputs()
BAD, FAULT, CHECKSUM = -1, -2, -3
VERDICT = {"bad": BAD, "checksum": CHECKSUM}
# bound on the documented difference (W.four_stream_end_mismatch) per 500 corruptions; about 11 are seen
MAX_EXEMPT_PER_500 = 25


class Emu:
    def __init__(self):
        subprocess.run(["make", "-C", ROOT, "tests/emu/libemu_lz.so"], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "libemu_lz.so"))
        self.lib.emu_zstd.restype = C.c_long
        self.lib.emu_zstd.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint, C.c_uint,
                                      C.c_int, C.c_char_p, C.c_size_t]

    def run(self, comp: bytes, cap: int, count_only=False, in_mis=0, out_mis=0, reps=1):
        """bytes on success, else BAD / CHECKSUM (count_only: the decoded length or BAD)."""
        out = C.create_string_buffer(max(cap, 1))
        msg = C.create_string_buffer(256)
        r = self.lib.emu_zstd(int(count_only), comp, len(comp), out, cap, in_mis, out_mis, reps, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        if r < 0 or count_only:
            return r
        return out.raw[:r]


@pytest.fixture(scope="module")
def emu():
    return Emu()


@pytest.fixture(scope="module")
def zs():
    z = W.libzstd_or_none()
    if z is None:
        pytest.skip("libzstd 1.5.5 (libzstd.so.1) not available: the verdicts are pinned to that release")
    return z


def pyarrow_zstd(data: bytes, level):
    pa = pytest.importorskip("pyarrow")
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def check(emu, zs, comp, cap, size_query=True, **kw):
    """The emulated decoder's verdict and bytes equal libzstd's; the size query agrees with it.  Returns libzstd's
    verdict, or "exempt" for the one documented difference (W.four_stream_end_mismatch)."""
    verdict, want = zs.expect(comp, cap)
    got = emu.run(comp, cap, **kw)
    if got == BAD and verdict != "bad" and W.four_stream_end_mismatch(comp):
        return "exempt"
    if verdict == "ok":
        assert got == want
    else:
        assert got == VERDICT[verdict], (verdict, got if isinstance(got, int) else len(got))
    if size_query:
        n = emu.run(comp, 0, count_only=True)
        v_unlimited, w_unlimited = zs.expect(comp, 1 << 25)
        if v_unlimited == "ok":
            assert n == len(w_unlimited)
        elif v_unlimited == "bad":
            assert n == BAD
        else:
            assert n != BAD
    return verdict


def corpus(zs, names=None, small=False):
    """(label, raw, stream) for libzstd at several levels / strategies / options and pyarrow's encoder."""
    out = []
    for name in (names or sorted(INPUTS)):
        data = INPUTS[name]
        combos = [(-5, None, 17, False, True), (1, None, 17, True, True), (3, None, 10, False, False),
                  (9, None, 17, True, False), (19, None, 17, False, True), (22, None, 10, True, True)]
        if not small:
            combos += [(l, s, wl, s % 2 == 0, s % 3 != 0) for l, s, wl in
                       ((1, 1, 17), (3, 2, 10), (5, 3, 17), (6, 4, 17), (7, 5, 10), (9, 6, 17), (12, 7, 17),
                        (16, 8, 10), (19, 9, 17))]
        for level, strategy, wl, ck, cs in combos:
            out.append((f"{name}/l{level}/s{strategy}/w{wl}/ck{int(ck)}/cs{int(cs)}", data,
                        zs.compress(data, level, strategy, wl, ck, cs)))
        for level in (1, 3, 19):
            out.append((f"{name}/pyarrow{level}", data, pyarrow_zstd(data, level)))
    return out


# 1. the writer is pinned to libzstd
def test_writer_valid_streams_pinned_to_libzstd(zs):
    for name, s, want in W.valid_streams(zs, INPUTS):
        assert zs.expect(s, len(want)) == ("ok", want), name


def test_writer_mutations_pinned_to_libzstd(zs):
    for rule, s, verdict in W.mutations(zs, INPUTS):
        assert zs.expect(s, 1 << 20)[0] == verdict, rule


def test_xxh64_matches_libzstd_checksums(zs):
    for name in ("empty", "one", "short13", "text", "random_777", "zeros_64k", "ragged_40001"):
        data = INPUTS[name]
        s = zs.compress(data, 3, checksum=True)
        assert int.from_bytes(s[-4:], "little") == W.xxh64(data) & 0xFFFFFFFF, name
    assert W.xxh64(b"") == 0xEF46DB3751D8E999


def test_coverage_of_the_stream_features(zs):
    """Across the corpus and the writer's streams, the parser sees every block type, literal mode (1 and 4 streams),
    Number_of_Sequences form, symbol-compression mode per table, and repeat-offset case."""
    seen = set()
    for _, _, s in corpus(zs, small=True):
        seen |= W.features(s)
    for _, s, _ in W.valid_streams(zs, INPUTS):
        seen |= W.features(s)
    for _, s in long_sequence_streams(zs):
        seen |= W.features(s)
    want = {("block", t) for t in ("raw", "rle", "compressed")}
    want |= {("lit", "raw", 0), ("lit", "rle", 0), ("lit", "huffman", 1), ("lit", "huffman", 4),
             ("lit", "treeless", 1), ("lit", "treeless", 4)}
    want |= {("nseq_form", k) for k in (1, 2, 3)} | {("nseq_ge_7f00",), ("nseq_zero_2byte",)}
    want |= {("mode", t, m) for t in ("LL", "OF", "ML") for m in ("predefined", "rle", "fse", "repeat")}
    want |= {("rep", r, ll0) for r in (1, 2, 3) for ll0 in (False, True)}
    assert not want - seen, sorted(want - seen)


def long_sequence_streams(zs):
    """Blocks with 0x7F00 or more sequences (the 3-byte Number_of_Sequences form)."""
    import random
    rng = random.Random(5)
    words = [bytes(rng.randrange(97, 123) for _ in range(rng.randint(3, 5))) for _ in range(64)]
    data = b"".join(rng.choice(words) for _ in range(40000))[:1 << 17]
    return [("words_128k", zs.compress(data, 1, window_log=17)), ("words_128k_l3", zs.compress(data, 3))]


# 2. hand-built and mutated streams
def test_emulated_decoder_on_hand_built_streams(emu, zs):
    for name, s, want in W.valid_streams(zs, INPUTS):
        assert emu.run(s, len(want)) == want, name
        assert emu.run(s, 0, count_only=True) == len(want), name


def test_emulated_decoder_on_mutations(emu, zs):
    for rule, s, verdict in W.mutations(zs, INPUTS):
        got = emu.run(s, 1 << 20)
        assert got == VERDICT.get(verdict, got), rule
        if verdict == "ok":
            assert got == zs.expect(s, 1 << 20)[1], rule


# 3. libzstd's and pyarrow's streams
@pytest.mark.parametrize("name", sorted(INPUTS))
def test_emulated_decoder_matches_libzstd(emu, zs, name):
    for label, data, s in corpus(zs, [name]):
        assert check(emu, zs, s, len(data)) == "ok", label


def test_emulated_decoder_long_sequence_blocks(emu, zs):
    for name, s in long_sequence_streams(zs):
        v, want = zs.expect(s, 1 << 17)
        assert v == "ok" and emu.run(s, len(want)) == want, name


def test_emulated_decoder_multi_block_1mb(emu, zs):
    from nvcomp_b200 import datagen
    data = datagen.tabular_f32(16, seed=3).tobytes()[:1 << 20]
    for level, ck in ((1, True), (3, False), (19, True)):
        s = zs.compress(data, level, checksum=ck)
        assert len(W.describe(s)[0]["blocks"]) > 1
        assert emu.run(s, len(data)) == data, level


# 4. capacity, alignment, repeated use of one warp
def test_emulated_decoder_capacity(emu, zs):
    for name in ("one", "text", "zeros_64k", "random_64k", "sensor", "ragged_40001", "period600"):
        data = INPUTS[name]
        for level in (1, 19):
            s = zs.compress(data, level, checksum=level == 1)
            for cap in (len(data), max(len(data) - 1, 0), 0, len(data) + 100):
                check(emu, zs, s, cap, size_query=False)


@pytest.mark.parametrize("mis", range(16))
def test_emulated_decoder_misaligned_buffers(emu, zs, mis):
    for name in ("text", "price_walk", "period7", "random_777"):
        data = INPUTS[name]
        s = zs.compress(data, 3, checksum=True)
        assert emu.run(s, len(data), in_mis=mis, out_mis=(mis * 5) % 16) == data
        assert emu.run(s, len(data), in_mis=(mis * 3) % 16, out_mis=mis) == data


def test_emulated_decoder_tables_reset_between_chunks(emu, zs):
    for name in ("text", "lowcard", "price_walk"):
        data = INPUTS[name]
        s = zs.compress(data, 19)
        assert emu.run(s, len(data), reps=3) == data


# 5. corruption campaign
def campaign_streams(zs):
    out = []
    for name in ("text", "price_walk", "lowentropy", "clustered", "period33", "short13", "runlength_i32"):
        data = INPUTS[name]
        for level, ck, cs in ((1, True, True), (3, False, False), (19, True, False), (-5, False, True)):
            out.append(zs.compress(data, level, checksum=ck, content_size=cs))
    return out


@pytest.mark.parametrize("part", range(6))
def test_emulated_decoder_corruption_campaign(emu, zs, part):
    """3000 seeded corruptions: the emulated decoder's verdict and bytes equal libzstd's, and nothing is written past
    the decoded bytes (checked inside the emulator).  The one exception: a 4-stream Huffman literal stream that does
    not end exactly on its first bit is rejected where libzstd may decode it (W.four_stream_end_mismatch); those
    cases are counted and must stay rare."""
    streams = campaign_streams(zs)
    exempt = 0
    for seed in range(part * 500, (part + 1) * 500):
        base = streams[seed % len(streams)]
        s = W.corrupt(base, seed)
        exempt += check(emu, zs, s, 1 << 16, size_query=seed % 4 == 0) == "exempt"
    print(f"corruption seeds {part * 500}..{(part + 1) * 500 - 1}: {exempt} four-stream end mismatches")
    assert exempt <= MAX_EXEMPT_PER_500, exempt


def test_size_query_past_a_bad_checksum(emu, zs):
    """The size query cannot see a content checksum: in a chunk whose first frame has a wrong checksum and whose
    second frame is malformed, the decode stops at the checksum (libzstd's first error) and the size query reports 0
    for the malformed frame (include/nvcomp/zstd.h)."""
    text = INPUTS["text"]
    good = zs.compress(text, 3, checksum=True)
    bad_ck = good[:-1] + bytes([good[-1] ^ 1])
    malformed = zs.compress(text, 3)[:40]
    s = bad_ck + malformed
    assert zs.expect(s, 1 << 20)[0] == "checksum"
    assert emu.run(s, 1 << 20) == CHECKSUM
    assert emu.run(s, 0, count_only=True) == BAD
    # without the malformed frame the size query reports the decoded length
    assert emu.run(bad_ck + good, 0, count_only=True) == 2 * len(text)
