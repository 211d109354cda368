"""The BC7 chain phase runs the roles of modes 4 and 5 at one rotation (mode 4 with index swap 0 and 1, mode 5) as one unit:
one fit, shared texel walks, the three refinements side by side, and the unit's best candidate merged under its own role
number.  Driven on the CPU through the emulation (tests/emu) with only the one-subset modes selected, every profile must give
the oracle's bytes: from each first rotation on and with all rotations, with mode 6 beside them, with unequal refinement
counts for modes 4 and 5, and at every number of blocks per warp the last round of a launch can deal (1, 2, 4, 8, 16)."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
from test_bc7_one_subset_chains import PROFILES, images


def selections(api, prof):
    """(label, settings) with only modes 4/5 (and 6) of the profile selected."""
    base = api.profile(prof)
    out = []

    def only(mode6):
        s = api.profile(prof)
        s.mode_selection[0] = s.mode_selection[1] = 0
        s.mode_selection[2] = 1
        s.mode_selection[3] = 1 if mode6 else 0
        return s

    for ch0 in range(base.channels):                       # rotations ch0 .. channels - 1; the last is one rotation alone
        s = only(False)
        s.mode45_channel0 = ch0
        out.append((f"modes 4/5 from rotation {ch0}", s))
    out.append(("modes 4/5/6", only(True)))
    for r4, r5, rch in ((1, 3, 0), (3, 0, 1), (0, 2, 2)):    # the roles of a unit refine a different number of times
        s = only(base.mode_selection[3])
        s.refineIterations[4], s.refineIterations[5], s.refineIterations_channel = r4, r5, rch
        out.append((f"refine 4/5/channel = {r4}/{r5}/{rch}", s))
    return out


@pytest.fixture
def emu():
    emu = T.emu()
    emu.lib.emu_set_bc7_per_warp.argtypes = [ctypes.c_int]
    emu.lib.emu_set_bc7_per_warp.restype = ctypes.c_int
    try:
        yield emu
    finally:
        emu.lib.emu_set_bc7_per_warp(16)


@pytest.mark.parametrize("per_warp", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("prof", PROFILES)
def test_rotation_units_emulated(emu, prof, per_warp):
    oracle = T.oracle()
    assert emu.lib.emu_set_bc7_per_warp(per_warp) == 0
    for label, s in selections(emu, prof):
        for n, img in enumerate(images()):
            want = oracle.encode("BC7", img, s)
            got = emu.encode("BC7", img, s)
            assert np.array_equal(got, want), (prof, label, per_warp, n, T.differing_blocks(got, want, 16))
