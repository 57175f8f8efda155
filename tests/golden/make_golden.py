#!/usr/bin/env python3
"""Generate the golden vectors in this directory.

Compressed streams come from the independent CPU codecs the reference links or names:
liblz4 1.9.4 (LZ4_compress_default and LZ4_compress_HC level 12, as in the reference's
examples/lz4_cpu_compression.cu:61-66) and pyarrow's bundled snappy.  Raw inputs are
small slices of the deterministic generators in nvcomp_b200/datagen.py plus one column
of the reference's own sample table (benchmarks/ExampleTable.txt column 5, as in the
usage text of benchmarks/text_to_binary.py:66-67) when its path is given; without it the
ref_table_* vectors already in the manifest are kept as they are.
Run from the repo root: python tests/golden/make_golden.py [path/to/nvcomp/benchmarks/ExampleTable.txt]
"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from conftest import LibLZ4, sample_inputs  # noqa: E402


def main():
    import pyarrow as pa
    lz4 = LibLZ4()
    snappy = pa.Codec("snappy")
    inputs = sample_inputs()
    keep = ["short13", "text", "period3", "period33", "period600", "runlength_i32", "price_walk",
            "lowcard", "clustered", "sorted_i64", "gen_data3", "zeros_1000", "random_777"]
    raws = {k: inputs[k][:16384] for k in keep}
    ref_table = sys.argv[1] if len(sys.argv) > 1 else None
    if ref_table:
        col = np.genfromtxt(ref_table, dtype="int64", usecols=(5,), delimiter="|")
        raws["ref_table_col5_i64"] = col.tobytes()[:16384]
        col = np.genfromtxt(ref_table, dtype="int32", usecols=(9,), delimiter="|")
        raws["ref_table_col9_i32"] = col.tobytes()[:16384]
    vectors = []
    for name, raw in sorted(raws.items()):
        open(os.path.join(HERE, name + ".raw"), "wb").write(raw)
        for tag, comp in (("lz4", lz4.compress(raw)), ("lz4hc", lz4.compress(raw, 12)),
                          ("snappy", snappy.compress(raw).to_pybytes())):
            fn = f"{name}.{tag}"
            open(os.path.join(HERE, fn), "wb").write(comp)
            vectors.append({"codec": "lz4" if tag.startswith("lz4") else "snappy", "comp": fn,
                            "raw": name + ".raw", "producer": tag})
    if not ref_table:
        # the table is needed to regenerate these vectors, not to keep testing with them
        old = json.load(open(os.path.join(HERE, "manifest.json")))["vectors"]
        vectors += [v for v in old if v["raw"].startswith("ref_table_")]
        vectors.sort(key=lambda v: v["raw"])
    json.dump({"vectors": vectors, "liblz4": lz4.lib.LZ4_versionNumber(), "pyarrow": pa.__version__},
              open(os.path.join(HERE, "manifest.json"), "w"), indent=1)
    print(len(vectors), "vectors")


if __name__ == "__main__":
    main()
