"""The BC7 chain phase runs the one-subset roles (mode 4 by rotation and index swap, mode 5 by rotation, mode 6) through their
own routine, with two-bit searches by thresholds and in a run order that is not the reference's.  Driven on the CPU through
the emulation (tests/emu) with only those modes selected, every profile's one-subset settings must give the oracle's bytes:
each rotation alone and all of them together, at one and at sixteen blocks per warp (one pass per block, and two roles per
pass), on tie-heavy blocks (few distinct values, grey), flat blocks (coincident endpoints: the quotient is 0/0 and the
thresholds out of reach), near-flat and random blocks."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T

PROFILES = ["ultrafast", "veryfast", "fast", "basic", "slow",
            "alpha_ultrafast", "alpha_veryfast", "alpha_fast", "alpha_basic", "alpha_slow"]


def images():
    rng = np.random.default_rng(31)
    n = 32
    out = [rng.integers(0, 256, (n, n, 4))]                                          # random
    out.append(rng.integers(0, 3, (n, n, 4)) * 127)                                 # three levels per channel: ties
    out.append(np.repeat(np.repeat(rng.integers(0, 256, (n // 4, n // 4, 4)), 4, 0), 4, 1))     # flat blocks
    out.append(rng.integers(100, 103, (n, n, 4)))                                   # spans below one unit
    out.append(np.repeat(rng.integers(0, 256, (n, n, 1)), 4, axis=2))               # r = g = b = a
    two = np.where(rng.random((n, n, 1)) < 0.5, (250, 10, 30, 255), (20, 200, 90, 128))
    out.append(two)                                                                  # two colours
    return [np.ascontiguousarray(x.astype(np.uint8)) for x in out]


def selections(api, prof):
    """(label, settings) with only the one-subset modes of the profile selected."""
    base = api.profile(prof)
    out = []
    if base.mode_selection[2]:
        for ch0 in range(base.mode45_channel0, base.channels):                       # one rotation at a time
            s = api.profile(prof)
            s.mode_selection[0] = s.mode_selection[1] = s.mode_selection[3] = 0
            s.mode45_channel0 = ch0
            out.append((f"modes 4/5 rotation {ch0}", s))
    if base.mode_selection[3]:
        s = api.profile(prof)
        s.mode_selection[0] = s.mode_selection[1] = s.mode_selection[2] = 0
        out.append(("mode 6", s))
    s = api.profile(prof)
    s.mode_selection[0] = s.mode_selection[1] = 0
    out.append(("modes 4/5/6", s))
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


@pytest.mark.parametrize("per_warp", [1, 16])
@pytest.mark.parametrize("prof", PROFILES)
def test_one_subset_roles_emulated(emu, prof, per_warp):
    oracle = T.oracle()
    assert emu.lib.emu_set_bc7_per_warp(per_warp) == 0
    for label, s in selections(emu, prof):
        for n, img in enumerate(images()):
            want = oracle.encode("BC7", img, s)
            got = emu.encode("BC7", img, s)
            assert np.array_equal(got, want), (prof, label, per_warp, n, T.differing_blocks(got, want, 16))
