#!/usr/bin/env python3
"""Generate the Zstd golden vectors in this directory: every *.raw input of manifest.json compressed by libzstd at
levels 3 and 19 with the content checksum on, listed in zstd_manifest.json (kept apart from manifest.json, which
other tests read).  smoke() decodes these on the GPU, so it needs no host Zstd library.
Run from the repo root: python tests/golden/make_golden_zstd.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from zstd_writer import LibZstd  # noqa: E402


def main():
    zs = LibZstd()
    with open(os.path.join(HERE, "manifest.json")) as f:
        raws = sorted({v["raw"] for v in json.load(f)["vectors"]})
    vectors = []
    for raw in raws:
        with open(os.path.join(HERE, raw), "rb") as f:
            data = f.read()
        for level in (3, 19):
            name = f"{raw[:-4]}.l{level}.zst"
            comp = zs.compress(data, level, checksum=True)
            assert zs.expect(comp, len(data)) == ("ok", data)
            with open(os.path.join(HERE, name), "wb") as f:
                f.write(comp)
            vectors.append({"codec": "zstd", "comp": name, "raw": raw, "producer": f"libzstd {zs.version} level "
                            f"{level} checksum"})
    with open(os.path.join(HERE, "zstd_manifest.json"), "w") as f:
        json.dump({"vectors": vectors}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
