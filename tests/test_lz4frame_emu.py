"""CPU: the warp-level LZ4 frame decoder (include/nvcomp/device/detail/lz4frame_decode.cuh, with the LZ4 block bodies
and their bulk-copy staging) run in the host warp emulator and held to liblz4 1.9.4's LZ4F_decompress: status, size
and bytes on the hand-built frames of tests/lz4frame_writer.py, on frames from pyarrow and LZ4F_compressFrame, on a
seeded corruption campaign (where liblz4 accepts an offset-0 match, which the LZ4 block grammar does not have, the
decoder must reject the chunk), at capacities exact, exact - 1 and 0, and at input / output misalignments 0-15 with
guard pages around both buffers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lz4frame_writer as F
from conftest import ROOT, sample_inputs

SUCCESS, CANNOT, BAD_CHECKSUM = F.SUCCESS, F.CANNOT, F.BAD_CHECKSUM


class FrameEmu:
    def __init__(self):
        subprocess.run(["make", "-C", ROOT, "tests/emu/libemu_lz.so"], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "libemu_lz.so"))
        f = self.lib.emu_lz4frame
        f.restype = C.c_long
        f.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint, C.c_uint, C.c_int,
                      C.c_char_p, C.c_size_t]

    def decode(self, chunk: bytes, cap: int, in_mis=0, out_mis=0, reps=1):
        """(status, bytes or None) as nvcompBatchedLZ4FrameDecompressAsync reports them."""
        out = C.create_string_buffer(max(cap, 1))
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz4frame(0, chunk, len(chunk), out, cap, in_mis, out_mis, reps, msg, 256)
        assert r != -2, f"emulator fault: {msg.value.decode()}"
        if r == -1:
            return CANNOT, None
        if r == -3:
            return BAD_CHECKSUM, None
        return SUCCESS, out.raw[:r]

    def size(self, chunk: bytes, in_mis=0) -> int:
        msg = C.create_string_buffer(256)
        r = self.lib.emu_lz4frame(1, chunk, len(chunk), None, 0, in_mis, 0, 1, msg, 256)
        assert r != -2, f"emulator fault: {msg.value.decode()}"
        return max(r, 0)


@pytest.fixture(scope="module")
def emu():
    return FrameEmu()


@pytest.fixture(scope="module")
def lz4f():
    try:
        return F.LibLZ4F()
    except OSError:
        pytest.skip("liblz4.so.1 not available")


def _caps(lz4f, chunk):
    err, out = lz4f.decode(chunk)
    n = len(out) if err is None else len(out) + 1024
    return sorted({n, max(n - 1, 0), 0})


def check(emu, lz4f, chunk, name, caps=None, **mis):
    for cap in caps if caps is not None else _caps(lz4f, chunk):
        want = lz4f.verdict(chunk, cap)
        got = emu.decode(chunk, cap, **mis)
        assert got[0] == want[0], (name, cap, got[0], want[0])
        assert got[1] == want[1], (name, cap)
    assert emu.size(chunk, mis.get("in_mis", 0)) == lz4f.size_verdict(chunk), name


# ---- the writer's corpus, each frame pinned to liblz4 first ----------------------------------------------------------
PINNED = {
    "reach_before_frame_start": "ERROR_decompressionFailed",
    "reach_prev_block_independent": "ERROR_decompressionFailed",
    "mut_bad_magic": "ERROR_frameType_unknown", "mut_legacy_magic": "ERROR_frameType_unknown",
    "mut_version_0": "ERROR_headerVersion_wrong", "mut_version_2": "ERROR_headerVersion_wrong",
    "mut_flg_reserved": "ERROR_reservedFlag_set", "mut_bd_reserved_low": "ERROR_reservedFlag_set",
    "mut_bd_reserved_high": "ERROR_reservedFlag_set",
    **{f"mut_bsid_{i}": "ERROR_maxBlockSize_invalid" for i in range(4)},
    "mut_wrong_hc": "ERROR_headerChecksum_invalid",
    "mut_compressed_over_max": "ERROR_maxBlockSize_invalid", "mut_raw_over_max": "ERROR_maxBlockSize_invalid",
    "mut_decoded_over_max": "ERROR_decompressionFailed",
    "mut_block_sum_flipped": "ERROR_blockChecksum_invalid", "mut_raw_block_sum_flipped": "ERROR_blockChecksum_invalid",
    "mut_content_sum_flipped": "ERROR_contentChecksum_invalid",
    "mut_content_size_plus1": "ERROR_frameSize_wrong", "mut_content_size_minus1": "ERROR_frameSize_wrong",
    "mut_trailing_byte": "truncated", "mut_trailing_magic": "truncated", "mut_truncated_skippable": "truncated",
}


@pytest.fixture(scope="module")
def corpus(lz4f):
    return F.corpus(lz4f)


def test_corpus_pinned_to_liblz4(lz4f, corpus):
    for name, chunk in corpus.items():
        err, _ = lz4f.decode(chunk)
        want = PINNED.get(name, "truncated" if name.startswith("mut_truncated") else None)
        assert err == want, (name, err)
    # the reach frames: exactly to the frame start and into the previous block (linked) decode
    for name in ("reach_to_frame_start", "reach_prev_block_linked", "reach_own_block_independent"):
        assert lz4f.decode(corpus[name])[0] is None


def test_corpus(emu, lz4f, corpus):
    for name, chunk in corpus.items():
        check(emu, lz4f, chunk, name)


def test_chunk_loop_carries_the_region(emu, lz4f, corpus):
    """Three decodes of one chunk by one warp, one region and one mbarrier phase (the batched kernel's chunk loop)."""
    for name in ("b4_L000", "b4_I111", "compressFrame_l9_L", "mut_block_sum_flipped", "three_frames"):
        chunk = corpus[name]
        err, out = lz4f.decode(chunk)
        cap = len(out) + 100
        assert emu.decode(chunk, cap, reps=3) == lz4f.verdict(chunk, cap), name


# ---- frames from liblz4 and pyarrow ---------------------------------------------------------------------------------
def producer_inputs():
    from nvcomp_b200 import datagen
    inputs = dict(sample_inputs())
    gdir = os.path.join(ROOT, "tests", "golden")
    for fn in sorted(os.listdir(gdir)):
        if fn.endswith(".raw"):
            inputs["golden_" + fn[:-4]] = open(os.path.join(gdir, fn), "rb").read()[:1 << 17]
    inputs["dg_runlength"] = datagen.runlength_i32(2, seed=21).tobytes()
    inputs["dg_tabular"] = datagen.tabular_f32(2, seed=22).tobytes()
    inputs["dg_lowentropy"] = datagen.lowentropy_bytes(1, seed=23).tobytes()
    return inputs


PREFS = [dict(bsid=b, linked=lk, content_sum=cs, block_sum=bs, content_size=sz, level=lv)
         for b in (4, 5) for lk in (True, False) for cs in (False, True) for bs in (False, True)
         for sz in (False, True) for lv in (0, 12)]


def producer_frames(lz4f, inputs, prefs=PREFS):
    import pyarrow as pa
    out = {}
    codec = pa.Codec("lz4")
    for name, data in inputs.items():
        out[f"{name}/pyarrow"] = codec.compress(data).to_pybytes()
        for k, p in enumerate(prefs):
            out[f"{name}/pref{k}"] = lz4f.compress_frame(data, **p)
        # the largest block sizes on one preference each (their frames equal 64 KB ones below 64 KB)
        out[f"{name}/bsid7"] = lz4f.compress_frame(data, 7, True, True, True, True)
    return out


def test_producer_frames(emu, lz4f):
    inputs = producer_inputs()
    frames = producer_frames(lz4f, inputs)
    for name, chunk in frames.items():
        data = inputs[name.split("/")[0]]
        assert lz4f.decode(chunk) == (None, data), name
        caps = [len(data), max(len(data) - 1, 0), 0] if "pref0" in name or "pyarrow" in name else [len(data)]
        check(emu, lz4f, chunk, name, caps=caps)


@pytest.mark.parametrize("mis", [(i, (7 * i + 3) % 16) for i in range(16)])
def test_misaligned_buffers(emu, lz4f, corpus, mis):
    inputs = sample_inputs()
    chunks = {"pyarrow_price": lz4f.compress_frame(inputs["price_walk"], 4, True, True, True),
              "independent_text": lz4f.compress_frame(inputs["text"] * 3, 4, False, True, True, True),
              "uncompressed": corpus["uncompressed_only"], "three_frames": corpus["three_frames"],
              "reach": corpus["reach_to_frame_start"], "bad_block_sum": corpus["mut_block_sum_flipped"]}
    for name, chunk in chunks.items():
        err, out = lz4f.decode(chunk)
        check(emu, lz4f, chunk, name, caps=[len(out) + (0 if err is None else 64)], in_mis=mis[0], out_mis=mis[1])


# ---- seeded corruption campaign -------------------------------------------------------------------------------------
def mutate(rng, chunk: bytes):
    b = bytearray(chunk)
    kind = int(rng.integers(0, 4))
    if kind == 0 and b:                                # bit flips
        for _ in range(int(rng.integers(1, 4))):
            i = int(rng.integers(0, len(b)))
            b[i] ^= 1 << int(rng.integers(0, 8))
    elif kind == 1 and b:                              # truncation
        del b[int(rng.integers(0, len(b))):]
    elif kind == 2:                                    # insertion
        i = int(rng.integers(0, len(b) + 1))
        b[i:i] = rng.integers(0, 256, int(rng.integers(1, 5)), dtype=np.uint8).tobytes()
    else:                                              # a byte set to an extreme value
        if b:
            b[int(rng.integers(0, len(b)))] = int(rng.choice([0, 0xff, 0x80, 0x7f]))
    return bytes(b)


def campaign_seeds(lz4f):
    inputs = sample_inputs()
    small = {k: v[:6000] for k, v in inputs.items() if k in ("text", "price_walk", "runlength_i32", "period7",
                                                               "lowcard", "sorted_i64", "random_777")}
    return producer_frames(lz4f, small, prefs=[PREFS[0], PREFS[5], PREFS[11], PREFS[23], PREFS[30]])


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_corruption_campaign(emu, lz4f, corpus, seed):
    rng = np.random.default_rng(seed)
    seeds = list(campaign_seeds(lz4f).values()) + [c for k, c in corpus.items()
                                                     if len(c) < 20000 and not k.startswith("mut_")]
    statuses = {SUCCESS: 0, CANNOT: 0, BAD_CHECKSUM: 0}
    offset0 = 0
    for i in range(600):
        chunk = mutate(rng, seeds[int(rng.integers(0, len(seeds)))])
        err, out = lz4f.decode(chunk)
        cap = len(out) + int(rng.integers(0, 64)) if err is None or i % 2 else len(out) + 1024
        want = lz4f.verdict(chunk, cap)
        got = emu.decode(chunk, cap)
        size = emu.size(chunk)
        if got != want and F.has_offset0_match(chunk):
            # liblz4 accepts an offset-0 match (it copies the destination's own bytes); the block grammar rejects it
            assert got == (CANNOT, None) and size == 0, (seed, i)
            offset0 += 1
            continue
        assert got == want, (seed, i, chunk.hex()[:200], cap, got[0], want[0])
        assert size == lz4f.size_verdict(chunk), (seed, i)
        statuses[want[0]] += 1
    assert all(statuses.values()), statuses
    assert offset0 < 10, offset0
