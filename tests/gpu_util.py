"""Helpers shared by the -m gpu parity tests (all calls go through the C ABI via nvcomp_b200.batched).

Output buffers are guarded: every output chunk sits in its own region, pre-filled with FILL, with at least GUARD bytes
of CANARY in front and behind.  A compressed chunk may use [ptr, ptr + CompressGetMaxOutputChunkSize), a decompressed
one [ptr, ptr + cap).  After every call the canaries must be intact, and a successful decode must have written exactly
`actual` bytes: [actual, cap) still holds FILL."""
import numpy as np
import torch

from nvcomp_b200.batched import Batch, Codec, make_batch

GUARD = 64
FILL = 0xA5
CANARY = 0x3C


def _guarded_batch(lens, misalign=0):
    """Output batch whose chunk i may use lens[i] bytes at a 16-byte aligned address + misalign.  Returns the batch and
    the host mask of the bytes the chunks may write."""
    slots = [(n + misalign + 15) // 16 * 16 + GUARD for n in lens]       # each chunk its own slot: one huge chunk
    offsets = GUARD + misalign + np.cumsum([0] + slots[:-1], dtype=np.int64)[:len(lens)]
    total = GUARD + max(sum(slots), 1)
    host = np.full(total, CANARY, dtype=np.uint8)
    allowed = np.zeros(total, dtype=bool)
    for o, n in zip(offsets, lens):
        host[o:o + n] = FILL
        allowed[o:o + n] = True
    slab = torch.from_numpy(host).cuda()
    ptrs = torch.from_numpy(offsets + slab.data_ptr()).cuda()
    sizes = torch.tensor(list(lens), dtype=torch.int64, device="cuda")
    return Batch(slab, ptrs, sizes, offsets), allowed


def _check_canaries(host, allowed, offsets, what):
    bad = np.flatnonzero((host != CANARY) & ~allowed)
    if bad.size:
        i = int(np.searchsorted(offsets, bad[0], side="right")) - 1
        raise AssertionError(f"{what}: byte written outside its chunk at slab offset {int(bad[0])} "
                             f"({int(bad[0] - offsets[max(i, 0)])} from chunk {max(i, 0)}), {bad.size} bytes in all")


def guarded_decompress(launch, what: str, comp_chunks, caps, in_misalign=0, out_misalign=0):
    """Run a decoder into guarded outputs and check them.  launch(comp batch, out batch, max capacity) enqueues the
    decode and returns its (actual, status) tensors (either may be None).  Inputs sit at 16-byte aligned addresses +
    in_misalign, outputs + out_misalign.  Returns (outputs, actual, status, out batch)."""
    caps = [int(c) for c in caps]
    comp = make_batch(comp_chunks, misalign=in_misalign)
    out, allowed = _guarded_batch(caps, out_misalign)
    actual, status = launch(comp, out, max(caps + [1]))
    torch.cuda.synchronize()
    a = actual.cpu().numpy()[:len(caps)] if actual is not None else None
    s = status.cpu().numpy()[:len(caps)] if status is not None else None
    host = out.slab.cpu().numpy()
    _check_canaries(host, allowed, out.offsets, what)
    if a is not None and s is not None:
        for i, (o, cap) in enumerate(zip(out.offsets, caps)):
            if s[i] == 0:
                assert a[i] <= cap, (what, i, a[i], cap)
                rest = host[o + int(a[i]):o + cap]
                assert (rest == FILL).all(), f"{what}: chunk {i} wrote past actual={int(a[i])} (cap {cap})"
    sizes = np.maximum(a, 0) if a is not None else np.asarray(caps)
    return out.to_host(sizes), a, s, out


def gpu_decompress(codec: Codec, comp_chunks, caps, misalign=0, want_actual=True, want_status=True, in_misalign=None,
                   out_misalign=None):
    """comp_chunks: list of bytes; caps: list of output capacities, through the codec's DecompressAsync.  Inputs sit at
    16-byte aligned addresses + in_misalign, outputs + out_misalign (both default to misalign).  Returns (outputs,
    actual, status, out batch)."""
    def launch(comp, out, max_chunk):
        return codec.decompress(comp, out, max_chunk=max_chunk, want_actual=want_actual, want_status=want_status)
    return guarded_decompress(launch, f"{codec.fmt} decompress", comp_chunks, caps,
                              misalign if in_misalign is None else in_misalign,
                              misalign if out_misalign is None else out_misalign)


def gpu_compress(codec: Codec, raw_chunks, misalign=0, out_misalign=0):
    """Compress raw_chunks (inputs at 16-byte aligned addresses + misalign, outputs + out_misalign).  Every stream
    must fit in CompressGetMaxOutputChunkSize.  Returns (streams, out batch with sizes = compressed bytes)."""
    inp = make_batch(raw_chunks, misalign=misalign)
    n = len(raw_chunks)
    max_chunk = max([len(c) for c in raw_chunks] + [1])
    max_out = codec.compress_get_max_output_chunk_size(max_chunk)
    tb = codec.compress_get_temp_size(n, max_chunk)
    temp = torch.empty(max(tb, 1), dtype=torch.uint8, device="cuda")
    out, allowed = _guarded_batch([max_out] * n, out_misalign)
    codec.compress_async(inp.ptrs.data_ptr(), inp.sizes.data_ptr(), max_chunk, n, temp.data_ptr(), tb,
                         out.ptrs.data_ptr(), out.sizes.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    sizes = out.sizes.cpu().numpy()
    assert (sizes <= max_out).all(), (codec.fmt, int(sizes.max()), max_out)
    _check_canaries(out.slab.cpu().numpy(), allowed, out.offsets, f"{codec.fmt} compress")
    return out.to_host(sizes), out
