"""CPU: the warp-level Deflate encoder of nvcomp_b200/csrc (deflate_compress.cuh) executed in the host warp emulator
(tests/emu: 32 fibers, rendezvous at every warp intrinsic, guard pages around the global buffers).  Every stream must
inflate under zlib, fit the maximum output size, and equal byte for byte what the stream rules of
tests/deflate_encode_model.py build from the encoder's own parse."""
import ctypes as C
import heapq
import os
import subprocess
import zlib

import numpy as np
import pytest

import deflate_encode_model as M
from conftest import ROOT, sample_inputs
from nvcomp_b200 import datagen

ALGOS = (0, 1, 2)
FAULT = -2


class Emu:
    def __init__(self):
        subprocess.run(["make", "-C", ROOT, "tests/emu/libemu_lz.so"], check=True, stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(os.path.join(ROOT, "tests", "emu", "libemu_lz.so"))
        self.lib.emu_deflate.restype = C.c_int
        self.lib.emu_deflate.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_uint, C.c_char_p, C.c_size_t,
                                         C.c_char_p, C.c_size_t]
        self.lib.emu_deflate_parse.restype = C.c_int
        self.lib.emu_deflate_parse.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint32), C.c_size_t,
                                               C.c_char_p, C.c_size_t]

    def compress(self, algo: int, data: bytes, in_mis: int = 0) -> bytes:
        cap = M.max_output_size(len(data))
        out = C.create_string_buffer(cap)
        msg = C.create_string_buffer(256)
        r = self.lib.emu_deflate(algo, data, len(data), in_mis, out, cap, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        return out.raw[:r]

    def parse(self, algo: int, data: bytes) -> list:
        cap = 3 * (len(data) + 1)
        t = (C.c_uint32 * cap)()
        msg = C.create_string_buffer(256)
        r = self.lib.emu_deflate_parse(algo, data, len(data), t, cap, msg, 256)
        assert r != FAULT, f"emulator fault: {msg.value.decode()}"
        return M.tokens_from_parse(data, [tuple(t[i:i + 3]) for i in range(0, r, 3)])


@pytest.fixture(scope="module")
def emu():
    return Emu()


def _fibonacci_bytes(n=65536, seed=5):
    """Literal frequencies in Fibonacci proportion over 22 symbols: an unlimited Huffman code would be 21 bits deep."""
    fib = [1, 1]
    while len(fib) < 22:
        fib.append(fib[-1] + fib[-2])
    scale = n / sum(fib)
    counts = [max(1, int(f * scale)) for f in fib]
    counts[-1] += n - sum(counts)
    data = np.repeat(np.arange(22, dtype=np.uint8) * 11, counts)
    np.random.default_rng(seed).shuffle(data)
    return data.tobytes()


def dataset_inputs():
    """A 64 KB slice of every datagen dataset."""
    out = {
        "snappy_synth": datagen.snappy_synth(1, 3, seed=21)[0],
        "runlength_i32": datagen.runlength_i32(1, seed=22)[0],
        "sorted_i64": datagen.sorted_i64(1, seed=23)[0],
        "lowentropy_bytes": datagen.lowentropy_bytes(1, seed=24)[0],
        "random_bytes": datagen.random_bytes(1, seed=25)[0],
        "zeros": datagen.zeros(1)[0],
        "lz4_mixed": datagen.lz4_mixed(1, seed=26)[0],
    }
    for col in range(4):
        out[f"tabular_f32_col{col}"] = datagen.tabular_f32(1, seed=27, column=col)[0]
    return {k: v.tobytes()[:65536] for k, v in out.items()}


def edge_inputs():
    rng = np.random.default_rng(99)
    text = (b"It was the best of times, it was the worst of times, it was the age of wisdom. " * 1000)
    x32768 = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    x32769 = rng.integers(0, 256, 32769, dtype=np.uint8).tobytes()
    out = {f"len{n}": text[:n] for n in range(6)}
    out.update({
        "len65535": text[:65535],
        "len65536": text[:65536],
        "random65536": rng.integers(0, 256, 65536, dtype=np.uint8).tobytes(),
        "zeros65536": bytes(65536),
        "period1": b"\x07" * 50000,
        "period2": b"\x01\x02" * 25000,
        "period4": bytes(range(4)) * 12500,
        "period8": bytes(range(100, 108)) * 6250,
        "repeat_at_32768": x32768 + x32768[:20000],
        "repeat_at_32769": x32769 + x32769[:20000],
        "fibonacci": _fibonacci_bytes(),
        "single_byte": b"Q",
        "fixed_9bit_literals": bytes([0xB8, 0x52]),        # a fixed block with 9-bit and 8-bit literal codes
        "fixed_all_code_lengths": bytes([200, 150, 255, 144, 143, 0, 7, 0xB8]) * 3,
    })
    return out


INPUTS = {**{f"sample:{k}": v for k, v in sample_inputs().items()},
          **{f"data:{k}": v for k, v in dataset_inputs().items()},
          **{f"edge:{k}": v for k, v in edge_inputs().items()}}


def zlib_raw(data: bytes, level: int) -> bytes:
    z = zlib.compressobj(level, zlib.DEFLATED, -15)
    return z.compress(data) + z.flush()


def huffman_cost(freq) -> int:
    """Bit cost of an unlimited-depth Huffman code: a lower bound for any length limit."""
    h = [f for f in freq if f]
    if len(h) <= 1:
        return sum(h)
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        cost += a + b
        heapq.heappush(h, a + b)
    return cost


def check_lengths(freq, lens, limit):
    used = [s for s in range(len(freq)) if freq[s]]
    assert all(lens[s] for s in used) and all(x <= limit for x in lens)
    if len(used) >= 2:
        assert sum(2.0 ** -x for x in lens if x) <= 1.0
        cost = sum(f * x for f, x in zip(freq, lens))
        assert cost >= huffman_cost(freq)
        if max(lens) < limit:       # the limit did not bind: package-merge gives a Huffman code
            assert cost == huffman_cost(freq)


def check_stream(emu, algo, data, stream):
    # 1. zlib reads it to the end
    z = zlib.decompressobj(-15)
    assert z.decompress(stream) == data and z.eof and not z.unused_data
    # 2. size bound (the emulator also checks that nothing past the stream was written)
    assert len(stream) <= M.max_output_size(len(data))
    # 3. the model rebuilds the same bytes from the encoder's parse
    items = emu.parse(algo, data)
    plan = M.plan(data, items)
    assert M.encode(data, items) == stream
    blocks = M.parse_stream(stream)
    if plan["kind"] == "stored":
        assert [b["kind"] for b in blocks] == ["stored"] * max(1, -(-len(data) // 65535))
    else:
        assert len(blocks) == 1 and blocks[0]["kind"] == plan["kind"] and blocks[0]["items"] == items
    # 4. the dynamic code is package-merge optimal and the chosen block is the cheapest of the three
    check_lengths(plan["lit"], plan["lit_lens"], 15)
    check_lengths(plan["dist"], plan["dist_lens"], 15)
    check_lengths(plan["cfreq"], plan["clen_lens"], 7)
    costs = {"stored": plan["stored_bits"], "fixed": plan["fixed_bits"], "dynamic": plan["dyn_bits"]}
    assert costs[plan["kind"]] == min(costs.values())
    assert len(stream) == (costs[plan["kind"]] + 7) // 8
    if plan["kind"] == "dynamic":
        assert blocks[0]["lit_lens"] == plan["lit_lens"] and blocks[0]["seq"] == plan["seq"]
    # 5. window and parse mode
    matches = [it for it in items if not isinstance(it, int)]
    assert all(1 <= d <= 32768 and 4 <= n <= 258 for n, d in matches)
    if algo == 2:
        assert not matches
    return plan, matches


@pytest.mark.parametrize("name", sorted(INPUTS))
def test_emulated_encoder(emu, name):
    data = INPUTS[name]
    for algo in ALGOS:
        stream = emu.compress(algo, data)
        plan, matches = check_stream(emu, algo, data, stream)
        for mis in range(1, 16):
            assert emu.compress(algo, data, in_mis=mis) == stream, (algo, mis)
        if name == "edge:random65536":
            assert plan["kind"] == "stored" and len(stream) == 65536 + 10
        if name == "edge:zeros65536" and algo != 2:
            assert any(n == 258 for n, _ in matches)
        if name == "edge:fibonacci" and algo == 2:
            assert max(plan["lit_lens"]) == 15 and plan["kind"] == "dynamic"
        if name == "edge:repeat_at_32769" and algo != 2:
            assert all(d != 32769 for _, d in matches)


def test_emulated_encoder_uses_the_full_window(emu):
    """A repeat exactly 32 768 bytes back is found (the high-compression table keeps it)."""
    items = emu.parse(1, INPUTS["edge:repeat_at_32768"])
    assert any(not isinstance(it, int) and it[1] == 32768 for it in items)


def test_high_compression_is_no_larger(emu):
    """Summed over each dataset (8 chunks), algo 1's output is no larger than algo 0's; ratios beside zlib 1 and 6."""
    sets = {
        "tabular_f32": datagen.tabular_f32(8, seed=31),
        "runlength_i32": datagen.runlength_i32(8, seed=32),
        "sorted_i64": datagen.sorted_i64(8, seed=33),
        "lowentropy_bytes": datagen.lowentropy_bytes(8, seed=34),
        "snappy_synth": datagen.snappy_synth(8, 3, seed=35),
        "lz4_mixed": datagen.lz4_mixed(8, seed=36),
        "random_bytes": datagen.random_bytes(8, seed=37),
    }
    print()
    for name, arr in sets.items():
        chunks = [arr[i].tobytes() for i in range(arr.shape[0])]
        raw = sum(len(c) for c in chunks)
        sizes = {a: sum(len(emu.compress(a, c)) for c in chunks) for a in ALGOS}
        zl = {lv: sum(len(zlib_raw(c, lv)) for c in chunks) for lv in (1, 6)}
        print(f"{name:18s} ratio algo0 {raw / sizes[0]:6.2f}  algo1 {raw / sizes[1]:6.2f}  algo2 {raw / sizes[2]:6.2f}"
              f"  zlib1 {raw / zl[1]:6.2f}  zlib6 {raw / zl[6]:6.2f}")
        assert sizes[1] <= sizes[0], name
