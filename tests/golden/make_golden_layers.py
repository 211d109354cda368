#!/usr/bin/env python3
"""Generate tests/golden/layers_digests.json from the reference's OWN layer-copy bodies (oracle/_ref/libitw_ref_layers.so, built by
oracle/build_ref_layers.py from IntelPlugin.h and IntelPlugin.cpp: CopyLayersIntoMipMaps, CopyFromLayerChannelIntoImage,
FillLayerDataToWhite).

Run where the reference tree exists:   python tests/golden/make_golden_layers.py
The inputs are the seeded generators of tests/test_mips_from_layers.py (its GRID on a 13 x 7 document)."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import ctypes  # noqa: E402

import build_ref_layers  # noqa: E402
import test_mips_from_layers as L  # noqa: E402


def main():
    lib = ctypes.CDLL(build_ref_layers.build(verbose=False))
    lib.ref_copy_layers_into_mips.restype = ctypes.c_int
    levels = {}
    for case in L.GRID:
        fmt, depth, channels, alpha, has_alpha, count = case
        layers, before = L.grid_case(*case)
        out = L.ref_do_write_dds(lib, fmt, depth, L.W, L.H, before, layers, has_alpha)
        levels[":".join(str(int(x) if isinstance(x, bool) else x) for x in case)] = L.grid_digest(*case, out)
    path = os.path.join(HERE, "layers_digests.json")
    with open(path, "w") as f:
        json.dump({"document": [L.W, L.H], "levels": levels}, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(levels)} digests to {path}")


if __name__ == "__main__":
    main()
