"""The eight warp-level device headers (include/nvcomp/device/*.cuh) are included by users' own .cu files, often by
several in one program.  `make` links two translation units that both include all eight and both call every Deflate,
Gzip and Zstd device function into one library, once from plain objects and once with relocatable device code
(tests/cpp/device_headers_link.cu); a header function with external, non-inline linkage fails either link with a
multiple definition.  Here both libraries must exist and carry the symbols of both translation units."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", ["libdevice_headers_link.so", "libdevice_headers_link_rdc.so"])
def test_two_translation_units_link(name):
    path = os.path.join(ROOT, "build", "tests", name)
    assert os.path.exists(path), f"{path} is missing: `make` builds it, and a failed link leaves it missing"
    lib = C.CDLL(path)
    assert lib.device_headers_link_tu1() == 1
    assert lib.device_headers_link_tu2() == 2
