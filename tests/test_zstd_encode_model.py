"""CPU: the warp-level Zstd encoder (include/nvcomp/device/detail/zstd_encode.cuh), run in the host warp emulator, held
to the stream-rules model of tests/zstd_encode_model.py.

For every input of the shared corpus, the model must rebuild the emulated frame byte for byte from the matcher's own
parse.  Independent checks then read the frame back without the model's rules: the parse obeys the matcher's limits
and is maximal; the frame's sequences and literals are the block-split parse; every match that can use a repeat code
does; the Huffman code is length-limited optimal; every block type, literal mode, weight form and table mode is the
cheapest with the stated ties; every normalised count table sums to 2^log and round-trips.  The corpus must reach each
boundary of the rules (header sizes, stream counts, sequence counts, bodies one byte either side of their block)."""
import itertools

import pytest

import lz_encode_model as LZ
import zstd_encode_model as M
import zstd_writer as W
from test_deflate_encode_emu import check_lengths, huffman_cost
from zstd_encode_corpus import EmuZstdEncoder, corpus

INPUTS = corpus()
NAMES = sorted(INPUTS)
_CASES = {}


@pytest.fixture(scope="module")
def enc():
    return EmuZstdEncoder()


@pytest.fixture
def case(enc, name):
    return _case(enc, name)


def _case(enc, name):
    """(data, parse, frame, plan, frame read back) of one corpus input, computed once."""
    if name not in _CASES:
        data = INPUTS[name]
        parse = enc.parse(data)
        frame = enc.compress(data)
        _CASES[name] = (data, parse, frame, M.plan(data, parse), M.parse_frame(frame))
    return _CASES[name]


def _first_min(sizes: dict, order):
    """The first of `order` whose size is the smallest: the tie rule."""
    present = [k for k in order if k in sizes]
    best = min(sizes[k] for k in present)
    return next(k for k in present if sizes[k] == best)


@pytest.mark.parametrize("name", NAMES)
def test_model_rebuilds_frame(name, case):
    data, parse, frame, _, _ = case
    assert M.encode(data, parse) == frame


@pytest.mark.parametrize("name", NAMES)
def test_parse_obeys_matcher_rules(name, case):
    """Offsets in [1, min(pos, 65535)], matches >= 4 bytes equal to their source, starting before n - 4, maximal."""
    data, parse, _, _, _ = case
    LZ.check_sequences(data, parse, 4, 0)


@pytest.mark.parametrize("name", NAMES)
def test_frame_is_the_block_split_parse(name, case):
    data, parse, frame, _, fr = case
    n = len(data)
    assert fr["content"] == data and fr["n"] == n
    assert fr["header"] == (6 if n <= 255 else 7)
    assert [(b["start"], b["end"]) for b in fr["blocks"]] == \
        [(s, min(s + M.BLOCK, n)) for s in range(0, max(n, 1), M.BLOCK)]
    # the matches of the parse, cut at block ends, pieces under 4 bytes dropped to literals
    matches, pos = [], 0
    for ll, off, ml in parse[:-1]:
        p = pos + ll
        for s in range(p, p + ml):
            if s == p or s % M.BLOCK == 0:
                end = min(p + ml, (s // M.BLOCK + 1) * M.BLOCK)
                if end - s >= M.MIN_MATCH:
                    matches.append((s, off, end - s))
        pos = p + ml
    got = []
    for b in fr["blocks"]:
        if b["type"] != "compressed":
            continue
        pos = b["start"]
        want_lits = bytearray()
        for s in b["sequences"]:
            want_lits += data[pos:pos + s["ll"]]
            pos += s["ll"]
            got.append((pos, s["off"], s["ml"]))
            pos += s["ml"]
        want_lits += data[pos:b["end"]]
        assert b["literals"] == want_lits
    in_compressed = [m for m in matches
                     if next(b for b in fr["blocks"] if b["start"] <= m[0] < b["end"])["type"] == "compressed"]
    assert got == in_compressed


@pytest.mark.parametrize("name", NAMES)
def test_every_repeatable_match_uses_a_repeat_code(name, case):
    _, _, _, _, fr = case
    for b in fr["blocks"]:
        for s in b.get("sequences", ()):
            rep, off = s["rep"], s["off"]
            usable = rep if s["ll"] else rep[1:]
            if off in usable:
                assert s["ov"] <= 3, s
                # the first slot that holds the offset
                assert s["ov"] == usable.index(off) + 1, s
            else:
                assert s["ov"] == off + 3, s


@pytest.mark.parametrize("name", NAMES)
def test_huffman_literals(name, case):
    _, _, _, plan, fr = case
    for b, p in zip(fr["blocks"], plan):
        if b.get("lit_mode") != "huffman":
            continue
        lits, L = b["literals"], b["L"]
        hist = [0] * 256
        for c in lits:
            hist[c] += 1
        lens = b["huf_lens"] + [0] * (256 - len(b["huf_lens"]))
        assert all((lens[s] > 0) == (hist[s] > 0) for s in range(256))
        check_lengths(hist, lens, M.HUF_LIMIT)
        assert sum(2.0 ** -x for x in lens if x) == 1.0
        assert b["huf_log"] == max(lens)
        if max(lens) < M.HUF_LIMIT:
            assert sum(h * x for h, x in zip(hist, lens)) == huffman_cost(hist)
        # one stream below 256 literals, four otherwise
        assert b["lit_streams"] == (1 if L < 256 else 4)
        # the weight form: direct (maxsym < 128) unless the FSE form is strictly smaller
        maxsym = max(s for s in range(256) if hist[s])
        direct_sz = (maxsym + 1) // 2 if maxsym < 128 else None
        fse = M.fse_weights(b["tree"]["weights"])
        assert len(b["tree"]["weights"]) == maxsym
        if b["tree"]["form"] == "direct":
            assert direct_sz is not None and (fse is None or direct_sz <= len(fse))
            assert b["tree"]["size"] == 1 + direct_sz
        else:
            assert fse is not None and (direct_sz is None or len(fse) < direct_sz)
            assert b["tree"]["size"] == 1 + len(fse)
            _check_counts(b["tree"]["norm"], b["tree"]["log"], b["tree"]["ncount"], set(b["tree"]["weights"]), 6)
        # the smallest Size_Format
        assert b["lit_header"] == M.huf_lit_header_size(L, b["csz"], L < 256)


@pytest.mark.parametrize("name", NAMES)
def test_block_and_literal_modes_are_cheapest(name, case):
    data, _, _, plan, fr = case
    assert len(plan) == len(fr["blocks"])
    for b, p in zip(fr["blocks"], plan):
        blk = data[b["start"]:b["end"]]
        sizes = {"raw": len(blk)}
        if len(blk) >= 2 and blk.count(blk[0]) == len(blk):
            sizes["rle"] = 1
        if "compressed" in p["sizes"]:
            sizes["compressed"] = p["sizes"]["compressed"]
        assert b["type"] == _first_min(sizes, ("raw", "rle", "compressed")), sizes
        if b["type"] != "compressed":
            continue
        assert b["size"] == sizes["compressed"] < len(blk)
        L = b["L"]
        lsizes = dict(p["lit"]["sizes"])
        lh_raw = 1 if L <= 31 else 2 if L <= 4095 else 3
        assert lsizes["raw"] == lh_raw + L
        assert ("rle" in lsizes) == (len(set(b["literals"])) == 1)
        assert b["lit_mode"] == _first_min(lsizes, ("raw", "rle", "huffman")), lsizes
        assert b["lit_section"] == lsizes[b["lit_mode"]]
        if b["lit_mode"] != "huffman":
            assert b["lit_header"] == lh_raw


def _check_counts(norm, log, ncount, used, max_log):
    assert 5 <= log <= max_log
    assert sum(abs(c) for c in norm) == 1 << log
    for s, c in enumerate(norm):
        assert (c >= 1) if s in used else (c == 0), (s, c)
    assert all(s < len(norm) for s in used)
    assert M.ncount_bytes(norm, len(norm) - 1, log) == ncount
    assert W._read_ncount(ncount + bytes(8), len(norm) - 1) == (norm, log, len(ncount))


@pytest.mark.parametrize("name", NAMES)
def test_sequence_tables(name, case):
    _, _, _, plan, fr = case
    for b, p in zip(fr["blocks"], plan):
        if b["type"] != "compressed":
            continue
        nseq = b["nseq"]
        assert b["nseq_bytes"] == (1 if nseq < 128 else 2)
        if not nseq:
            continue
        for i, t in enumerate(M.NAMES):
            codes = [s["codes"][i] for s in b["sequences"]]
            used = set(codes)
            tp = p["seq"]["tables"][t]
            # predefined cost, recomputed from the predefined distribution
            pnorm, plog, max_log = M.PREDEFINED[t]
            pcost = sum(M.cost(max(pnorm[c], 1), plog) for c in codes)
            assert tp["pcost"] == pcost
            costs = {"predefined": pcost, "fse": tp["fcost"]}
            if len(used) == 1:
                costs["rle"] = 8 << 8
            mode = b["tables"][t]["mode"]
            assert mode == _first_min(costs, ("predefined", "rle", "fse")), (t, costs)
            if mode == "rle":
                assert b["tables"][t]["symbol"] == codes[0]
            if mode == "fse":
                tb = b["tables"][t]
                _check_counts(tb["norm"], tb["log"], tb["ncount"], used, max_log)
                assert len(tb["norm"]) == max(used) + 1
                assert tb["log"] == M.table_log(max_log, nseq, max(used))
                assert tp["fcost"] == sum(M.cost(tb["norm"][c], tb["log"]) for c in codes) + (len(tb["ncount"]) << 11)


def test_boundaries_reached(enc):
    """The corpus reaches every boundary of the header and section rules."""
    seen = set()
    for name in NAMES:
        _, _, _, plan, fr = _case(enc, name)
        prev = None
        for b, p in zip(fr["blocks"], plan):
            if b["type"] == "compressed":
                L = b["L"]
                if b["lit_mode"] == "raw":
                    seen.add(("raw_lits", b["lit_header"], L))
                    if p["lit"]["sizes"].get("rle") == p["lit"]["sizes"]["raw"]:
                        seen.add(("raw_rle_tie",))
                if b["lit_mode"] == "huffman":
                    seen.add(("huf_header", b["lit_header"]))
                    seen.add(("huf_L", L, b["lit_streams"]))
                    seen.add(("weights", b["tree"]["form"]))
                    fse = p["lit"]["fse_weights"]
                    if fse is not None and len(fse) == p["lit"]["direct_sz"]:
                        seen.add(("weights_tie", b["tree"]["form"]))
                seen.add(("nseq", b["nseq"], b["nseq_bytes"]))
                for t in M.NAMES:
                    tb = b["tables"].get(t, {})
                    if tb.get("mode") == "fse" and b["nseq"] <= 4:
                        seen.add(("fse_below_5_sequences", tb["log"]))
                    if tb:
                        tp = p["seq"]["tables"][t]
                        if tp["fcost"] == min(c for c in (tp["pcost"], tp["rle_cost"]) if c is not None):
                            seen.add(("table_cost_tie", tb["mode"]))
                if prev is not None and prev[0]["type"] == "raw" and prev[1]["seqs"] and \
                        any(s["ov"] <= 3 for s in b["sequences"]):
                    seen.add(("raw_then_repeat",))
            c = p["sizes"].get("compressed")
            if c is not None and c >= len(INPUTS[name][b["start"]:b["end"]]) - 1:
                seen.add(("body_minus_block", b["end"] - b["start"] - c, b["type"]))
            prev = (b, p)
    want = {("raw_lits", 1, 31), ("raw_lits", 2, 32), ("raw_lits", 2, 4095), ("raw_lits", 3, 4096),
            ("huf_header", 3), ("huf_header", 4), ("huf_header", 5), ("huf_L", 255, 1), ("huf_L", 256, 4),
            ("huf_L", 16384, 4), ("weights", "direct"), ("weights", "fse"), ("nseq", 127, 1), ("nseq", 128, 2),
            ("body_minus_block", 1, "compressed"), ("body_minus_block", 0, "raw"), ("raw_then_repeat",),
            ("fse_below_5_sequences", 5), ("raw_rle_tie",), ("weights_tie", "direct"),
            ("table_cost_tie", "predefined")}
    assert want <= seen, sorted(want - seen)


def test_small_table_log_decides_the_mode():
    """Below 5 sequences the accuracy log is 5, not libzstd's maximum, and that decides modes: 4 sequences with OF
    codes 0, 0, 0, 1 cost 20 bits Predefined, 19.5 bits FSE at log 5 (2 header bytes) and 27.5 bits at log 8 (3)."""
    codes = (0, 0, 0, 1)
    hist = [3, 1] + [0] * 62
    costs = {}
    for log in (5, 8):
        norm = M.normalize(hist, 1, 4, log)
        costs[log] = sum(M.cost(norm[c], log) for c in codes) + (len(M.ncount_bytes(norm, 1, log)) << 11)
    pcost = sum(M.cost(M.PREDEFINED["OF"][0][c], 5) for c in codes)
    assert M.table_log(8, 4, 1) == 5 and costs[5] < pcost < costs[8]
    assert M.plan_table("OF", list(codes), 4)["mode"] == "fse"


def test_no_fse_weights_below_five_weights():
    """With at most 4 weights the direct form takes at most 2 bytes and the FSE form at least 2, a tie that goes
    direct: every weight vector is tried, so the weights' accuracy log below 5 weights never reaches a frame."""
    for nw in range(2, 5):
        for w in itertools.product(range(12), repeat=nw):
            fse = M.fse_weights(list(w))
            assert fse is None or len(fse) >= (nw + 1) // 2
