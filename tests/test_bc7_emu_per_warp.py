"""The BC7 warp program at every blocks-per-warp count the kernel deals (16 in a full round; 1, 2, 4, 8 or 16 in the last one),
in all three lane orders, on the tie-heavy two-colour and flat blocks of test_bc7_two_subset_lists.py: both two-subset lists
full (t1 = t3 = 64, winners by (error, key) without a ranking), mode 7's full list (t7 = 64), and a short list next to a full
one (ranked).  Driven on the CPU through tests/emu/bc7_rounds.cpp."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import itw_testlib as T
from test_bc7_two_subset_lists import images, settings

SRC = os.path.join(T.ROOT, "tests", "emu", "bc7_rounds.cpp")
CASES = [(3, 64, 64, None), (4, 64, 64, 64), (3, 64, 9, None), (4, 7, 64, 64), (4, 64, 64, 5)]


@pytest.fixture(scope="module")
def rounds(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("bc7_rounds") / "bc7_rounds.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fwrapv",
                           "-mfpmath=sse", "-msse2", "-Wno-unknown-pragmas", SRC, "-o", lib])
    f = ctypes.CDLL(lib).bc7_rounds_encode
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    return f


def encode(rounds, img, s, per_warp, order):
    h, w = img.shape[:2]
    img = np.ascontiguousarray(img)
    out = np.zeros((h // 4) * (w // 4) * 16, np.uint8)
    surf = T.binding.RgbaSurface(img.ctypes.data, w, h, w * 4)
    assert rounds(ctypes.addressof(surf), out.ctypes.data, ctypes.addressof(s), per_warp, order) == 0
    return out


@pytest.mark.parametrize("per_warp", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("channels,t1,t3,t7", CASES)
def test_every_blocks_per_warp_and_lane_order(rounds, channels, t1, t3, t7, per_warp):
    oracle = T.oracle()
    s = settings(oracle, channels, t1, t3)
    if t7 is not None:
        s.fastSkipTreshold_mode7 = t7
    for img in images(channels):
        want = oracle.encode("BC7", img, s).reshape(-1)
        for order in (0, 1, 2):
            assert np.array_equal(encode(rounds, img, s, per_warp, order), want), (channels, t1, t3, t7, per_warp, order)

