"""The BC7 warp program at every blocks-per-warp count the kernel deals (16 in a full round; 1, 2, 4, 8 or 16 in the last one),
in all three lane orders, on the tie-heavy two-colour and flat blocks of test_bc7_two_subset_lists.py: both two-subset lists
full (t1 = t3 = 64, winners by (error, key) without a ranking), mode 7's full list (t7 = 64), and a short list next to a full
one (ranked).  Driven on the CPU through the emulation (tests/emu)."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
from test_bc7_two_subset_lists import images, settings

CASES = [(3, 64, 64, None), (4, 64, 64, 64), (3, 64, 9, None), (4, 7, 64, 64), (4, 64, 64, 5)]


@pytest.fixture
def emu():
    """The emulation, with its blocks per warp and lane order restored afterwards."""
    emu = T.emu()
    emu.lib.emu_set_bc7_per_warp.argtypes = [ctypes.c_int]
    emu.lib.emu_set_bc7_per_warp.restype = ctypes.c_int
    emu.lib.emu_set_lane_order.argtypes = [ctypes.c_int]
    emu.lib.emu_set_lane_order.restype = None
    try:
        yield emu
    finally:
        emu.lib.emu_set_bc7_per_warp(16)
        emu.lib.emu_set_lane_order(0)


def test_other_blocks_per_warp_counts_are_rejected(emu):
    for n in (0, 3, 32, -1):
        assert emu.lib.emu_set_bc7_per_warp(n) == -1


@pytest.mark.parametrize("per_warp", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("channels,t1,t3,t7", CASES)
def test_every_blocks_per_warp_and_lane_order(emu, channels, t1, t3, t7, per_warp):
    oracle = T.oracle()
    s = settings(oracle, channels, t1, t3)
    if t7 is not None:
        s.fastSkipTreshold_mode7 = t7
    assert emu.lib.emu_set_bc7_per_warp(per_warp) == 0
    for img in images(channels):
        want = oracle.encode("BC7", img, s).reshape(-1)
        for order in (0, 1, 2):
            emu.lib.emu_set_lane_order(order)
            assert np.array_equal(emu.encode("BC7", img, s).reshape(-1), want), (channels, t1, t3, t7, per_warp, order)
