"""The BC7 three-subset shape phases fit and search two subset masks of a block per lane: masks 2i and 2i + 1 of
itw_masks3.cuh (bc7_fit_masks2, bc7_masks_error2).  Compiled for the CPU like the emulation, both routines must equal the
per-mask routines for all 70 lane pairs, on random blocks and on blocks with ties and flat subsets.  The table itself must
be what tools/gen_mask_tables.py generates, pair masks as the phases assume, and describe every three-subset shape."""
import ctypes
import importlib.util
import os
import re
import subprocess

import itw_testlib as T
import test_bc7_pair_fit as pair_fit

SRC = os.path.join(T.ROOT, "tests", "emu", "mask3_pair_check.cpp")
MASKS3 = os.path.join(T.ROOT, "intel-texture-works-plugin_b200", "csrc", "itw_masks3.cuh")


def popcount(m):
    return bin(m).count("1")


def committed_table():
    src = open(MASKS3).read()
    count = int(re.search(r"#define ITW_MASK3_COUNT (\d+)", src).group(1))
    first = int(re.search(r"#define ITW_MASK3_FIRST (\d+)", src).group(1))
    masks_src = src[src.index("ITW_TABLE_INIT_mask3_unique"):src.index("ITW_TABLE_INIT_shape3_mask_id")]
    ids_src = src[src.index("ITW_TABLE_INIT_shape3_mask_id") + len("ITW_TABLE_INIT_shape3_mask_id"):]
    masks = [int(x, 16) for x in re.findall(r"0x([0-9A-Fa-f]+)", masks_src)]
    ids = [int(x) for x in re.findall(r"\b\d+\b", ids_src)]
    assert len(masks) == count and len(ids) == 64 * 3
    return masks, first, ids


def three_subset_masks():
    """Subset masks of the 64 three-subset shapes, from the oracle's own pattern table (independent of the generator)."""
    src = open(os.path.join(T.ROOT, "oracle", "itw_oracle.cpp")).read()
    body = re.search(r"kShape3\[64\]\s*=\s*\{(.*?)\};", src, re.S).group(1)
    pats = [int(x, 0) for x in re.findall(r"0x[0-9A-Fa-f]+|\b\d+\b", body)]
    assert len(pats) == 64
    return [[sum(1 << k for k in range(16) if ((p >> (2 * k)) & 3) == j) for j in range(3)] for p in pats]


def test_mask3_table_is_generated_and_paired():
    spec = importlib.util.spec_from_file_location("gen_mask_tables", os.path.join(T.ROOT, "tools", "gen_mask_tables.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    text, _, _ = gen.masks3(gen.shape_masks())
    assert text == open(MASKS3).read(), "itw_masks3.cuh is not what tools/gen_mask_tables.py generates"

    masks, first, ids = committed_table()
    assert len(set(masks)) == len(masks)
    assert first % 2 == 0 and len(masks) % 2 == 0                    # no lane pair straddles the mode-0 boundary
    for lo, hi in ((0, first), (first, len(masks))):
        group = masks[lo:hi]
        odd_classes = sum(1 for pc in {popcount(m) for m in group} if sum(popcount(m) == pc for m in group) % 2)
        unequal = sum(1 for i in range(0, len(group), 2) if popcount(group[i]) != popcount(group[i + 1]))
        assert unequal == odd_classes // 2, f"masks [{lo}, {hi}): {unequal} lane pairs of unequal popcount"

    shapes = three_subset_masks()
    for n in range(64):
        assert [masks[u] for u in ids[3 * n:3 * n + 3]] == shapes[n], f"shape {64 + n}"
        if n < 16:
            assert max(ids[3 * n:3 * n + 3]) < first                     # mode 0 only stores the first group's endpoints
    assert {m for row in shapes for m in row} == set(masks)
    assert {m for row in shapes[:16] for m in row} == set(masks[:first])


def test_mask_pair_routines_equal_per_mask_routines(tmp_path):
    lib = str(tmp_path / "mask3_pair_check.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fwrapv",
                           "-mfpmath=sse", "-msse2", "-Wno-unknown-pragmas", SRC, "-o", lib])
    dll = ctypes.CDLL(lib)
    assert dll.mask3_pair_count() == 70
    check = dll.mask3_pair_check
    check.restype = ctypes.c_int
    tex = pair_fit.blocks()
    what = ctypes.create_string_buffer(256)
    bad = check(tex.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(tex)), what, ctypes.c_int(len(what)))
    assert bad == 0, f"{bad} mismatches, first: {what.value.decode()}"
