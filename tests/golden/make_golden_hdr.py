#!/usr/bin/env python3
"""Generate tests/golden/hdr_digests.json: SHA-256 digests of what the reference's own code computes on the HDR corpus of
tests/hdr_corpus.py, so that the oracle stays pinned to the reference where the reference is not present.

  inputs     the corpus surfaces and planes themselves (a changed generator shows up here first)
  convert32  oracle/_ref/libitw_ref_frontend.so ref_convert_pixels, BC6H, 32-bit planes of every pinned family, 1-4 planes,
             every flag set of test_frontend.flag_sets
  convert16  the same at depth 16 over every value 0 ... 65535
  chain_f16  ref_mip_chain_f16 (the reference's _Generate2DMipsBoxFilter / _Generate2DMipsLinearFilter) of every pinned family
             at test_mips_f16.SIZES + hdr_corpus.EXTRA_CHAIN_SHAPES
  bc6h       oracle/_ref/libitw_ref.so's BC6H blocks of every padded level of the hdr_corpus.BC6H_CHAINS chains, all five presets

Run where the reference is present:   python tests/golden/make_golden_hdr.py      (a few seconds)
Running it again gives a byte-identical file."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
import hdr_corpus as H  # noqa: E402
import itw_testlib as T  # noqa: E402
import test_frontend as F  # noqa: E402
import test_mips_f16 as M  # noqa: E402


def main():
    fe, ref = T.ref_frontend(), T.ref()
    assert fe is not None and ref is not None, "needs /root/reference (or prebuilt oracle/_ref libraries)"
    out = {"generator": "tests/golden/make_golden_hdr.py", "produced_by": "oracle/_ref (the reference's own function bodies and sources)",
           "inputs": {}, "convert32": {}, "convert16": {}, "chain_f16": {}, "bc6h": {}}
    h, w = H.CONVERT_SHAPE
    for fam in H.FAMILIES:
        px = H.family_planes(fam, h, w)
        out["inputs"][H.key("planes", fam, h, w)] = H.sha(px)
        for planes in (1, 2, 3, 4):
            sub = np.ascontiguousarray(px[..., :planes])
            for flags in F.flag_sets("BC6H", 32, planes):
                out["convert32"][H.key(fam, planes, flags)] = H.sha(F.ref_convert(fe, "BC6H", sub, flags))
    for planes in (1, 2, 3, 4):
        px = H.sixteen_bit_planes(planes)
        out["inputs"][H.key("u16", planes)] = H.sha(px)
        for flags in F.flag_sets("BC6H", 16, planes):
            out["convert16"][H.key(planes, flags)] = H.sha(F.ref_convert(fe, "BC6H", px, flags))
    for fam in H.FAMILIES:
        for sh, sw in M.SIZES + H.EXTRA_CHAIN_SHAPES:
            img = H.family(fam, sh, sw)
            out["inputs"][H.key(fam, sh, sw)] = H.sha(img)
            chain = M.chain_with(fe.ref_mip_chain_f16, img, M.full_levels(sw, sh))
            out["chain_f16"][H.key(fam, sh, sw)] = H.sha(np.concatenate([l.reshape(-1) for l in chain]))
    for fam, sh, sw in H.BC6H_CHAINS:
        img = H.family(fam, sh, sw)
        out["inputs"][H.key(fam, sh, sw)] = H.sha(img)
        chain = M.chain_with(fe.ref_mip_chain_f16, img, M.full_levels(sw, sh))
        for preset in T.binding.BC6H_PROFILES:
            s = ref.profile(preset)
            blocks = [ref.encode("BC6H", np.ascontiguousarray(M.pad4(l)), s) for l in chain]
            out["bc6h"][H.key(fam, sh, sw, preset)] = H.sha(np.concatenate(blocks))
    path = os.path.join(HERE, "hdr_digests.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path, {k: len(v) for k, v in out.items() if isinstance(v, dict)})


if __name__ == "__main__":
    main()
