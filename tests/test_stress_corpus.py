"""The structured stress corpus (tests/stress_corpus.py) on the CPU: the generator still makes the surfaces whose reference
digests are recorded (tests/golden/stress_digests.json), the oracle run over whole surfaces equals those digests, the corpus
reaches every encoder decision it is built to reach (checked from the block headers, not assumed), and the emulated kernels
equal the digests for every case on every 16th chunk of 16 block rows.

Runtime: about 55 s on 8 cores (the oracle on four whole surfaces, the emulation on 2 of 17 chunks for 24 cases)."""
import hashlib
import importlib.util
import json
import os
import time
from collections import Counter
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import bcn_decode as D
import itw_testlib as T
import stress_corpus as S

_spec = importlib.util.spec_from_file_location("make_golden_stress", os.path.join(os.path.dirname(__file__), "golden", "make_golden_stress.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "stress_digests.json")))
CASES = G.cases()
ROWS = G.CHUNK_BLOCK_ROWS
LAYOUTS = D.bc6_layouts(open(os.path.join(T.ROOT, "oracle", "itw_oracle.cpp")).read())


# ---- surfaces, chunked encodes --------------------------------------------------------------------------------------------
_SURFACES = {}


def surface(fmt):
    if fmt not in _SURFACES:
        _SURFACES[fmt] = np.ascontiguousarray(G.surface(fmt))
    return _SURFACES[fmt]


def chunk_rows(fmt, j):
    """texel rows of chunk j (16 block rows; the last chunk is shorter)"""
    h = surface(fmt).shape[0]
    return 4 * ROWS * j, min(4 * ROWS * (j + 1), h)


def encode_chunks(api, case, chunks, threads=None):
    """{chunk index: blocks} for the given chunks of the case's surface, one chunk per thread (blocks are independent, so a
    chunk encoded as a surface of its own gives the chunk's bytes)."""
    fmt = CASES[case][0]
    img = surface(fmt)

    def work(j):
        y0, y1 = chunk_rows(fmt, j)
        return j, api.encode(fmt, np.ascontiguousarray(img[y0:y1]), G.settings(api, case))
    with ThreadPoolExecutor(threads or len(os.sched_getaffinity(0))) as ex:
        return dict(ex.map(work, chunks))


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def nchunks(fmt):
    return -(-surface(fmt).shape[0] // (4 * ROWS))


# ---- block header reader --------------------------------------------------------------------------------------------------
BC6_FIELD = {0: 0, 1: 1, 2: 2, 6: 3, 10: 4, 14: 5, 18: 6, 22: 7, 26: 8, 30: 9, 3: 10, 7: 11, 11: 12, 15: 13}


def bc7_header(blk):
    """-> (mode, partition or None, rotation or None, index selection or None) of one BC7 block"""
    v = int.from_bytes(bytes(blk[:8]), "little")
    mode = (v & -v).bit_length() - 1
    v >>= mode + 1
    if mode == 0:
        return 0, v & 15, None, None
    if mode in (1, 2, 3, 7):
        return mode, v & 63, None, None
    if mode == 4:
        return 4, None, v & 3, (v >> 2) & 1
    if mode == 5:
        return 5, None, v & 3, None
    return mode, None, None, None


def bc6h_header(blk):
    """-> (mode 0-13, partition or None) of one BC6H block; the two-region modes end their header with 5 partition bits at
    bit 77"""
    v = int.from_bytes(bytes(blk), "little")
    mode = BC6_FIELD[v & 3 if (v & 3) < 2 else v & 31]
    return mode, ((v >> 77) & 31) if mode < 10 else None


def reach_cells(fmt, blocks):
    """cell -> block count.  BC7 cells: ("mode", m), ("mode m partition", p), ("mode 4 rotation, isel", (r, i)),
    ("mode 5 rotation", r).  BC6H cells: ("mode", m), ("mode m partition", p) for the two-region modes."""
    c = Counter()
    for blk in blocks.reshape(-1, 16):
        if fmt == "BC7":
            m, p, r, i = bc7_header(blk)
            c[("mode", m)] += 1
            if p is not None:
                c[(f"mode {m} partition", p)] += 1
            if m == 4:
                c[("mode 4 rotation, isel", (r, i))] += 1
            if m == 5:
                c[("mode 5 rotation", r)] += 1
        else:
            m, p = bc6h_header(blk)
            c[("mode", m)] += 1
            if p is not None:
                c[(f"mode {m} partition", p)] += 1
    return c


def wanted_cells(fmt):
    if fmt == "BC7":
        cells = [("mode", m) for m in range(8)]
        cells += [("mode 0 partition", p) for p in range(16)]
        cells += [(f"mode {m} partition", p) for m in (1, 2, 3, 7) for p in range(64)]
        cells += [("mode 4 rotation, isel", (r, i)) for r in range(4) for i in range(2)]
        return cells + [("mode 5 rotation", r) for r in range(4)]
    return [("mode", m) for m in range(14)] + [(f"mode {m} partition", p) for m in range(10) for p in range(32)]


# Cells a profile cannot produce, whatever the content: the opaque profiles (channels = 3) never evaluate mode 7
# (fastSkipTreshold_mode7 = 0) and run the mode 4 / 5 rotation loop over the colour channels only, so the stored rotation 0
# (alpha kept in its own channel) never comes out of them.
UNREACHABLE = {
    "slow": {("mode", 7): "mode 7 is not evaluated with channels = 3"}
    | {("mode 7 partition", p): "mode 7 is not evaluated with channels = 3" for p in range(64)}
    | {("mode 4 rotation, isel", (0, i)): "rotation 0 is outside the channels = 3 rotation loop" for i in range(2)}
    | {("mode 5 rotation", 0): "rotation 0 is outside the channels = 3 rotation loop"},
    "alpha_slow": {},
    "bc6h_slow": {},
    "bc6h_veryslow": {},
}
MIN_BLOCKS = 4


# ---- tests ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["BC7", "BC6H"])
def test_generator_reproduces_the_recorded_inputs(fmt):
    img = surface(fmt)
    assert img.shape == (GOLDEN["height"], GOLDEN["width"], 4) == (S.HEIGHT, S.WIDTH, 4)
    for case, (f, _, _) in CASES.items():
        if f == fmt:
            assert sha(img) == GOLDEN["cases"][case]["input_sha256"], f"{case}: the generator drifted from the recorded corpus"
    one = S.block_rgba16f if fmt == "BC6H" else S.block_rgba8
    for i in (0, 1, 4095, 33791, 66559):                    # any block regenerates from its index alone
        by, bx = divmod(i, S.BLOCKS_X)
        assert np.array_equal(img[4 * by:4 * by + 4, 4 * bx:4 * bx + 4], one(i)), i


def test_every_case_is_recorded_with_its_settings_bytes():
    assert sorted(GOLDEN["cases"]) == sorted(CASES)
    for case, (fmt, preset, _) in CASES.items():
        want = GOLDEN["cases"][case]
        assert (want["format"], want["preset"], want["chunk_block_rows"]) == (fmt, preset, ROWS)
        assert len(want["chunks"]) == nchunks(fmt)
        for tag, api in (("oracle", T.oracle()), ("emulation", T.emu())):
            assert G.settings_hex(G.settings(api, case)) == want["settings_hex"], (case, tag)


def test_header_reader_agrees_with_the_decoder():
    """The reader used for the reach table, against the independent decoders' mode on a sample of blocks of three profiles."""
    rng = np.random.default_rng(0)
    for fmt, prof in (("BC7", "alpha_slow"), ("BC7", "slow"), ("BC6H", "bc6h_slow")):
        blocks = encode_chunks(T.oracle(), prof, [3])[3].reshape(-1, 16)
        for k in rng.choice(len(blocks), 300, replace=False):
            if fmt == "BC7":
                _, mode = D.decode_bc7_block(blocks[k])
                assert bc7_header(blocks[k])[0] == mode
            else:
                _, mode = D.decode_bc6h_block(blocks[k], LAYOUTS)
                assert bc6h_header(blocks[k])[0] == mode


@pytest.mark.parametrize("prof", ["slow", "alpha_slow", "bc6h_slow", "bc6h_veryslow"])
def test_oracle_on_the_whole_surface_equals_the_reference_and_reaches_every_cell(prof, capsys):
    t0 = time.time()
    fmt = CASES[prof][0]
    want = GOLDEN["cases"][prof]
    got = encode_chunks(T.oracle(), prof, range(nchunks(fmt)))
    bad = [j for j in range(nchunks(fmt)) if sha(got[j]) != want["chunks"][j]]
    assert not bad, f"{prof}: chunks of 16 block rows where the oracle differs from the reference build: {bad}"
    blocks = np.concatenate([got[j] for j in range(nchunks(fmt))])
    assert sha(blocks) == want["sha256"]
    cells = reach_cells(fmt, blocks)
    skip = UNREACHABLE[prof]
    short = [(c, cells[c]) for c in wanted_cells(fmt) if c not in skip and cells[c] < MIN_BLOCKS]
    with capsys.disabled():
        print(f"\n[reach] {fmt} {prof}: {blocks.size // 16} blocks, {time.time() - t0:.1f} s")
        groups = {}
        for c in wanted_cells(fmt):
            groups.setdefault(c[0], []).append(c)
        for g, cs in groups.items():
            counts = [cells[c] for c in cs if c not in skip]
            line = "  ".join(f"{c[1]}:{cells[c]}" for c in cs if c not in skip) if len(cs) <= 16 else \
                f"{len(counts)} cells, min {min(counts)}, max {max(counts)}" if counts else ""
            print(f"  {g}: {line}" + (f"  (unreachable: {sum(c in skip for c in cs)})" if any(c in skip for c in cs) else ""))
    assert not short, f"{prof}: cells with fewer than {MIN_BLOCKS} blocks: {short[:20]}"
    for c, why in skip.items():                              # and what is listed as unreachable really does not occur
        assert cells[c] == 0, (c, why)


@pytest.mark.parametrize("case", list(CASES))
def test_emulated_kernels_equal_the_reference_every_16th_chunk(case):
    fmt = CASES[case][0]
    chunks = list(range(0, nchunks(fmt), 16))
    got = encode_chunks(T.emu(), case, chunks, threads=len(chunks))
    for j in chunks:
        assert sha(got[j]) == GOLDEN["cases"][case]["chunks"][j], f"{case}: chunk {j} of the emulated kernels differs from the reference"
