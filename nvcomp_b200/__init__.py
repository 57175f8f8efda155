"""nvcomp_b200 -- H100-native batched lossless codecs behind nvCOMP's C API.

The product is ``nvcomp_b200/lib/libnvcomp.so`` (hand-written sm_90a CUDA behind
the ``nvcompBatched*`` C ABI declared in ``include/nvcomp/*.h``).  This Python
package is the host-side mirror used by the tests and ``bench.py``: it loads the
shared library with ctypes and passes raw device pointers; torch is only used
for device memory, streams and ``torch.distributed`` plumbing.

There is no CPU fallback: importing :mod:`nvcomp_b200.batched` (or calling
:func:`nvcomp_b200.load`) raises if the CUDA library has not been built.
"""
from ._lib import load, lib_path, FORMATS, DECODE_ONLY_FORMATS, Status, Type  # noqa: F401

__all__ = ["load", "lib_path", "FORMATS", "DECODE_ONLY_FORMATS", "Status", "Type"]
