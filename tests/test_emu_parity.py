"""The product's kernel logic, executed lane by lane on the CPU (tests/emu), against the oracle.
This covers the warp program (phases, lane<->task maps, winner selection, bit packing) without a
GPU; the GPU's own float instructions are covered by the -m gpu tests."""
import numpy as np
import pytest

import itw_testlib as T


@pytest.mark.parametrize("fmt,prof", T.ALL_CASES, ids=[f"{f}-{p}" for f, p in T.ALL_CASES])
def test_emulated_kernels_bit_exact(fmt, prof):
    bpb = T.binding.FORMATS[fmt][1]
    for name, img in T.corpus_for(fmt, 32).items():
        got = T.run(T.emu(), fmt, img, prof)
        want = T.run(T.oracle(), fmt, img, prof)
        assert T.differing_blocks(got, want, bpb) == 0, f"{fmt}/{prof}/{name}"


@pytest.mark.parametrize("fmt,prof", [("BC7", "alpha_basic"), ("BC6H", "bc6h_basic"), ("BC3", None)])
def test_ragged_batches_and_strides(fmt, prof):
    """Block counts that are not multiples of the per-warp batch, non-square surfaces, padded strides."""
    rng = np.random.default_rng(5)
    dt = np.uint16 if fmt == "BC6H" else np.uint8
    hi = 0x7C00 if fmt == "BC6H" else 256
    for h, w, pad in ((4, 4, 0), (4, 12, 3), (12, 20, 5), (8, 4, 1)):
        buf = rng.integers(0, hi, (h, w + pad, 4)).astype(dt)
        img = buf[:, :w]                       # row stride larger than the row
        got = T.run(T.emu(), fmt, img, prof)
        want = T.run(T.oracle(), fmt, np.ascontiguousarray(img), prof)
        assert np.array_equal(got, want), (h, w, pad)


@pytest.mark.parametrize("per_warp", [8, 16])
@pytest.mark.parametrize("prof", ["slow", "alpha_slow", "alpha_fast", "veryfast"])
def test_bc7_round_sizes(prof, per_warp):
    """The BC7 warp program in rounds of 16 blocks (two halves, one chain phase: every full round) and of 8 (one half: a last
    round), with every ragged remainder 1..17 of the surface's last round, equals the oracle (test_bc7_emu_per_warp.py runs
    every count on tie-heavy blocks)."""
    import ctypes
    emu = T.emu()
    setter = emu.lib.emu_set_bc7_per_warp
    setter.argtypes = [ctypes.c_int]
    setter.restype = None
    rng = np.random.default_rng(11)
    try:
        setter(per_warp)
        for nblocks in (1, 7, 8, 9, 15, 16, 17, 33):
            img = rng.integers(0, 256, (4, 4 * nblocks, 4)).astype(np.uint8)
            img[:, : 4 * (nblocks // 2), 3] = 255                # opaque and translucent blocks side by side
            got = T.run(emu, "BC7", img, prof)
            want = T.run(T.oracle(), "BC7", img, prof)
            assert np.array_equal(got, want), (prof, per_warp, nblocks)
    finally:
        setter(16)


@pytest.mark.parametrize("order", [1, 2], ids=["descending", "shuffled"])
@pytest.mark.parametrize("fmt,prof", [("BC7", "slow"), ("BC7", "alpha_basic"), ("BC7", "alpha_veryfast"), ("BC6H", "bc6h_slow"),
                                      ("BC6H", "bc6h_veryfast")])
def test_phases_do_not_depend_on_lane_order(fmt, prof, order):
    """On the GPU the lanes of a phase run concurrently; the emulation runs them one after the other.  A phase that read what
    another lane of the same phase writes would give order-dependent output: descending and shuffled lane orders must equal
    the oracle too (13 i + 7 mod 32 is a permutation of the lanes)."""
    import ctypes
    emu = T.emu()
    setter = emu.lib.emu_set_lane_order
    setter.argtypes = [ctypes.c_int]
    setter.restype = None
    bpb = T.binding.FORMATS[fmt][1]
    try:
        setter(order)
        for name, img in T.corpus_for(fmt, 32).items():
            got = T.run(emu, fmt, img, prof)
            want = T.run(T.oracle(), fmt, img, prof)
            assert T.differing_blocks(got, want, bpb) == 0, f"{fmt}/{prof}/{name}/order {order}"
    finally:
        setter(0)
