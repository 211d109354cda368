"""The full two-subset phase of the BC7 encoder walks the 64 two-subset shapes in the order of itw_order2.cuh.  The table must
be what tools/gen_mask_tables.py generates: a permutation of the 64 shapes in non-decreasing popcount of subset 0 (taken
from the oracle's own shape table, independent of the generator), so that the lanes of a step walk loops of similar length.
The results are keyed by shape id, so the order cannot change them; the emulation and GPU parity tests check that."""
import importlib.util
import os
import re

import itw_testlib as T

ORDER2 = os.path.join(T.ROOT, "intel-texture-works-plugin_b200", "csrc", "itw_order2.cuh")


def subset0_popcounts():
    src = open(os.path.join(T.ROOT, "oracle", "itw_oracle.cpp")).read()
    body = re.search(r"kShape2\[64\]\s*=\s*\{(.*?)\};", src, re.S).group(1)
    sets = [int(x, 0) for x in re.findall(r"0x[0-9A-Fa-f]+|\b\d+\b", body)]          # bit k set: texel k is in subset 1
    assert len(sets) == 64
    return [16 - bin(m).count("1") for m in sets]


def test_shape2_order_is_generated_and_sorted():
    spec = importlib.util.spec_from_file_location("gen_mask_tables", os.path.join(T.ROOT, "tools", "gen_mask_tables.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    text = gen.order2(gen.shape_masks())
    src = open(ORDER2).read()
    assert text == src, "itw_order2.cuh is not what tools/gen_mask_tables.py generates"

    order = [int(x) for x in re.findall(r"\b\d+\b", src[src.index("ITW_TABLE_INIT_shape2_order") + len("ITW_TABLE_INIT_shape2_order"):])]
    assert sorted(order) == list(range(64))
    counts = subset0_popcounts()
    walked = [counts[s] for s in order]
    assert walked == sorted(walked)
    # 8 shapes per step of 32 lanes (4 blocks): the longest subset-0 walk plus the longest subset-1 walk of a step
    steps = [walked[i:i + 8] for i in range(0, 64, 8)]
    assert sum(max(s) + 16 - min(s) for s in steps) == 135
