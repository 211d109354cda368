#!/usr/bin/env python3
"""Generate tests/golden/stress_digests.json: SHA-256 of the reference-source build's output (oracle/_ref: kernel.ispc +
ispc_texcomp.cpp compiled scalar by oracle/build_ref.py) on the structured corpus of tests/stress_corpus.py, for every BC7 and
BC6H preset and for a fixed list of non-preset settings (CUSTOM below).

Run where the reference is present:   python tests/golden/make_golden_stress.py      (about a minute on 8 cores)

Each case stores the settings struct's bytes, the SHA-256 of the input surface, of the whole packed output and of every chunk
of 16 block rows (256 x 16 = 4 096 blocks; the last chunk of the 260 block rows has 4), so that a mismatch can be localised
to a chunk and the reference re-run on that chunk alone.  Row bands are encoded on threads; blocks are independent, so the
bytes do not depend on the thread count.  Running the script again gives a byte-identical file."""
import ctypes
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import itw_testlib as T  # noqa: E402
import stress_corpus as S  # noqa: E402
from make_golden_full import encode_mt  # noqa: E402

CHUNK_BLOCK_ROWS = 16

# name -> (format, preset the struct starts from, fields overwritten).  The non-preset settings cover short two-subset lists
# next to full and empty ones, both ends of the mode-7 list, no and extra refinement, every mode45_channel0 the presets do
# not use (1, 2, 4), skip_mode2 on the slow path, partial mode selections, and the BC6H slow / fast combinations with
# short, medium and full partition lists.
CUSTOM = {
    "bc7_t64_t9_norefine": ("BC7", "slow", {"fastSkipTreshold_mode1": 64, "fastSkipTreshold_mode3": 9, "refineIterations": [0] * 8}),
    "bc7_t7_t64_t7_5_ch1": ("BC7", "alpha_slow", {"fastSkipTreshold_mode1": 7, "fastSkipTreshold_mode3": 64, "fastSkipTreshold_mode7": 5,
                                                 "mode45_channel0": 1, "refineIterations": [3] * 8}),
    "bc7_t0_t64_t7_64_ch2_skip2": ("BC7", "alpha_slow", {"fastSkipTreshold_mode1": 0, "fastSkipTreshold_mode3": 64, "fastSkipTreshold_mode7": 64,
                                                        "mode45_channel0": 2, "skip_mode2": True}),
    "bc7_partial_selection_ch3_refine3": ("BC7", "alpha_slow", {"mode_selection": [True, True, False, False], "mode45_channel0": 3,
                                                               "fastSkipTreshold_mode7": 5, "refineIterations": [3] * 8,
                                                               "refineIterations_channel": 3}),
    "bc7_ch4_no_rotations": ("BC7", "alpha_basic", {"mode45_channel0": 4, "fastSkipTreshold_mode7": 64, "refineIterations_channel": 0}),
    "bc7_rgb_partial_selection_skip2_ch1": ("BC7", "slow", {"mode_selection": [False, True, True, False], "skip_mode2": True,
                                                           "mode45_channel0": 1, "refineIterations": [0, 1, 2, 3, 0, 1, 2, 0]}),
    "bc6h_slow_skip1": ("BC6H", "bc6h_slow", {"slow_mode": True, "fast_mode": False, "fastSkipTreshold": 1, "refineIterations_1p": 0,
                                              "refineIterations_2p": 3}),
    "bc6h_fast_skip17": ("BC6H", "bc6h_basic", {"slow_mode": False, "fast_mode": True, "fastSkipTreshold": 17, "refineIterations_1p": 3,
                                                "refineIterations_2p": 0}),
    "bc6h_slow_fast_skip32": ("BC6H", "bc6h_basic", {"slow_mode": True, "fast_mode": True, "fastSkipTreshold": 32, "refineIterations_1p": 1,
                                                     "refineIterations_2p": 1}),
}


def cases():
    """name -> (format, preset, overrides): every preset, then the non-preset settings"""
    out = {p: ("BC7", p, {}) for p in T.binding.BC7_PROFILES}
    out.update({p: ("BC6H", p, {}) for p in T.binding.BC6H_PROFILES})
    out.update(CUSTOM)
    return out


def settings(api, case):
    _, preset, over = cases()[case]
    s = api.profile(preset)
    for field, value in over.items():
        if isinstance(value, list):
            arr = getattr(s, field)
            for i, v in enumerate(value):
                arr[i] = v
        else:
            setattr(s, field, value)
    return s


def settings_hex(s):
    return bytes(ctypes.string_at(ctypes.addressof(s), ctypes.sizeof(s))).hex()


def surface(fmt):
    return S.structured_rgba16f() if fmt == "BC6H" else S.structured_rgba8()


def digest_entry(fmt, img, out):
    """make_golden_full.digest_entry with chunks of 16 block rows"""
    h, w = img.shape[:2]
    row = (w // 4) * T.binding.FORMATS[fmt][1]
    chunks = [hashlib.sha256(out[r * row:(r + CHUNK_BLOCK_ROWS) * row].tobytes()).hexdigest() for r in range(0, h // 4, CHUNK_BLOCK_ROWS)]
    return {"sha256": hashlib.sha256(out.tobytes()).hexdigest(), "bytes": int(out.size), "input_sha256": hashlib.sha256(img.tobytes()).hexdigest(),
            "chunk_block_rows": CHUNK_BLOCK_ROWS, "chunks": chunks}


def main():
    ref = T.ref()
    assert ref is not None, "needs /root/reference (or a prebuilt oracle/_ref/libitw_ref.so)"
    threads = len(os.sched_getaffinity(0))
    imgs = {fmt: np.ascontiguousarray(surface(fmt)) for fmt in ("BC7", "BC6H")}
    out = {"generator": "tests/golden/make_golden_stress.py", "produced_by": "oracle/_ref (reference-source build)",
           "height": S.HEIGHT, "width": S.WIDTH, "cases": {}}
    for name, (fmt, preset, over) in cases().items():
        t0 = time.time()
        s = settings(ref, name)
        entry = digest_entry(fmt, imgs[fmt], encode_mt(ref, fmt, imgs[fmt], s, threads))
        entry.update({"format": fmt, "preset": preset, "settings_hex": settings_hex(s)})
        out["cases"][name] = entry
        print(name, fmt, f"{time.time() - t0:.1f}s", flush=True)
    path = os.path.join(HERE, "stress_digests.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
