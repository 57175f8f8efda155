"""CPU: the run-length steps of the direct Snappy loop (snappy_decode_chunk, what the light kernel runs) in the host
warp emulator, held to the oracle.  A step decodes up to 32 literals of 1..8 bytes and copy-1 / copy-2 elements with
offset 1..8 at once; every other element, and every element that fails a check, goes to the serial element code.
The streams here are hand-built (lz_writer) around exactly those edges: every literal length against every offset,
periods that reach into the run before (pyarrow's shape) or stay inside the literal (the oracle's), runs across step
and window boundaries, serial elements inside a step, and each rejection rule.  Every stream runs at all 16 input and
16 output misalignments, with guard pages around both buffers."""
import numpy as np
import pytest

import lz_writer as W
from test_lz_writer import SeqEmu

MIS = [(i, (7 * i + 3) % 16) for i in range(16)]      # every input and every output misalignment


@pytest.fixture(scope="module")
def emu():
    return SeqEmu()


def _rand(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _check(emu, oracle, case, mis=MIS, what=""):
    want = oracle.decompress("snappy", case.comp, case.cap)
    if case.out is not None:
        assert want == case.out, ("writer and oracle disagree", what)
    for im, om in mis:
        got = emu.decode("snappy", case.comp, case.cap, "direct", in_mis=im, out_mis=om)
        assert got == want, (what, im, om, None if want is None else len(want), None if got is None else len(got))


def _run_soup(rng, n_elems, stop_rate=0.0, start=8):
    """A valid stream of run elements (and, at stop_rate, elements the steps leave to the serial code)."""
    s = W.Snappy().lit(_rand(rng, start))
    for _ in range(n_elems):
        r = rng.random()
        if r < stop_rate:
            k = int(rng.integers(0, 4))
            if k == 0:
                s.lit(_rand(rng, int(rng.choice([9, 17, 60, 61, 200]))))
            elif k == 1:
                s.copy2(int(rng.integers(9, min(len(s.out), 3000) + 1)) if len(s.out) >= 9 else 1,
                        int(rng.integers(1, 65)))
            elif k == 2:
                s.copy4(int(rng.integers(1, min(len(s.out), 40) + 1)), int(rng.integers(1, 65)))
            else:
                s.copy1(int(rng.integers(9, min(len(s.out), 2047) + 1)) if len(s.out) >= 9 else 1,
                        int(rng.integers(4, 12)))
        elif r < 0.35:
            s.lit(_rand(rng, int(rng.integers(1, 9))))
        elif r < 0.6:
            s.copy1(int(rng.integers(1, 9)), int(rng.integers(4, 12)))
        else:
            s.copy2(int(rng.integers(1, 9)), int(rng.choice([64, int(rng.integers(1, 65))])))
    return s


def test_every_literal_length_and_offset(emu, oracle):
    """Literals of 1..8 bytes followed by copy-1 and copy-2 elements at every offset 1..8: off <= literal length (the
    period inside the literal) and off > literal length (the period reaching into the run before)."""
    rng = np.random.default_rng(1)
    for ll in range(1, 9):
        s = W.Snappy().lit(_rand(rng, 8))
        for off in range(1, 9):
            s.lit(_rand(rng, ll)).copy1(off, int(rng.integers(4, 12))).copy2(off, 64).copy2(off, 64)
            s.copy2(off, int(rng.integers(1, 64))).copy1(off, 4).copy2(off, 1)
        _check(emu, oracle, s.case(), what=("ll", ll))


def test_first_elements_of_a_chunk(emu, oracle):
    """Copies right at the start: off == op (valid) and off == op + 1 (invalid) for every op < 9."""
    rng = np.random.default_rng(2)
    for ll in range(1, 9):
        for off in range(1, 9):
            for kind in ("copy1", "copy2"):
                s = W.Snappy().lit(_rand(rng, ll))
                getattr(s, kind)(off, 4 if kind == "copy1" else 5)
                s.lit(_rand(rng, 3)).copy2(min(off, ll + 8), 64)
                _check(emu, oracle, s.case(), mis=MIS[:4], what=(kind, ll, off))


@pytest.mark.parametrize("n_elems", list(range(1, 80)) + [95, 96, 97, 127, 128, 129, 300])
def test_runs_across_step_boundaries(emu, oracle, n_elems):
    """Every stream length from 1 to 80 run elements and around multiples of 32: steps that end at the 32nd element, at
    the window's last byte, mid-element at the window's end, and exactly at the end of the input."""
    rng = np.random.default_rng(100 + n_elems)
    for trial in range(3):
        s = _run_soup(rng, n_elems, start=int(rng.integers(1, 9)))
        _check(emu, oracle, s.case(), mis=MIS if trial == 0 else MIS[::5], what=(n_elems, trial))


def test_serial_elements_inside_steps(emu, oracle):
    """Long literals, copies with offset > 8 and copy-4 elements (also with offset <= 8) between run elements."""
    rng = np.random.default_rng(3)
    for trial in range(40):
        s = _run_soup(rng, int(rng.integers(20, 200)), stop_rate=float(rng.choice([0.02, 0.1, 0.4])))
        _check(emu, oracle, s.case(), mis=MIS[trial % 16:trial % 16 + 2], what=trial)


def test_rejections_inside_steps(emu, oracle):
    """Each rejection rule hit by an element deep inside a step of valid run elements: off == 0, off == op + 1, a copy
    that overruns the output by one byte, a literal past the end of the input, an element truncated at the end, and
    a final length short of the preamble's."""
    rng = np.random.default_rng(4)
    for trial in range(24):
        base = _run_soup(rng, int(rng.integers(0, 70)), start=int(rng.integers(1, 9)))
        comp, out = bytes(base.body), bytes(base.out)
        n = len(out)
        cases = []
        # off == 0 (copy-1 / copy-2)
        cases.append(W.varint(n + 8) + comp + bytes([1 | (4 << 2), 0]))
        cases.append(W.varint(n + 8) + comp + bytes([2 | (7 << 2), 0, 0]))
        # off == op + 1, on the very first copy of a chunk
        cases.append(W.varint(9) + bytes([0 << 2, 0x41]) + bytes([2 | (7 << 2), 2, 0]))
        # copy overrunning the output by one byte
        cases.append(W.varint(n + 7) + comp + bytes([2 | (7 << 2), 1, 0]))
        cases.append(W.varint(n + 4) + comp + bytes([1 | (1 << 2), 3]))
        # literal past the end of the input; element truncated at the end of the input
        cases.append(W.varint(n + 6) + comp + bytes([5 << 2]) + b"abc")
        cases.append(W.varint(n + 64) + comp + bytes([2 | (63 << 2), 4]))
        cases.append(W.varint(n + 5) + comp + bytes([1 | (1 << 2)]))
        # the stream ends short of the preamble's length
        cases.append(W.varint(n + 1) + comp)
        for k, c in enumerate(cases):
            # valid elements behind the rejected one must not change the verdict
            tail = bytes([0 << 2, 0x55, 2 | (63 << 2), 1, 0]) if k < 5 else b""
            _check(emu, oracle, W.Case("snappy", c + tail, None, n + 70), mis=MIS[k % 16:k % 16 + 1],
                   what=(trial, k))


def _clustered(n):
    from nvcomp_b200 import datagen
    return [r.tobytes() for r in datagen.tabular_f32(n, column=2)]


def test_clustered_column_both_producers(emu, oracle):
    """The benchmark's run-length column, compressed by the oracle (4-byte literals, period inside the literal) and by
    pyarrow (3-byte literals, period reaching into the run before)."""
    import pyarrow as pa
    snap = pa.Codec("snappy")
    for i, raw in enumerate(_clustered(3)):
        for comp in (oracle.compress("snappy", raw), snap.compress(raw).to_pybytes()):
            _check(emu, oracle, W.Case("snappy", comp, raw, len(raw)), mis=MIS[i::3], what=i)


def test_mutation_campaign(emu, oracle):
    """Seeded corruptions of clustered-column streams from both producers and of run-element soups: the verdict,
    the length and the bytes equal the oracle's, and nothing outside the buffers is touched."""
    import pyarrow as pa
    snap = pa.Codec("snappy")
    rng = np.random.default_rng(9)
    raws = [r[:int(n)] for r, n in zip(_clustered(2), (65536, 20000))]
    streams = [oracle.compress("snappy", r) for r in raws] + [snap.compress(r).to_pybytes() for r in raws]
    streams += [_run_soup(rng, 150, stop_rate=0.05).case().comp for _ in range(4)]
    for i in range(400):
        comp = streams[i % len(streams)]
        kind, bad = W.mutate(rng, "snappy", comp)
        n = oracle.size("snappy", comp)
        cap = W.corpus_cap(i, bad, n)
        _check(emu, oracle, W.Case("snappy", bad, None, cap), mis=MIS[i % 16:i % 16 + 1], what=(i, kind))
