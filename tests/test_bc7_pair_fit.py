"""The BC7 shape phases fit both subsets of a two-subset shape in one routine (bc7_fit_pair) and score both of its mode-1 and
mode-3 searches in one texel walk (bc7_pair_error).  Compiled for the CPU like the emulation, every output must equal the
per-subset routines -- bc7_fit, a split bound written out in the driver and the key of the ranking, bc7_assign -- over all
64 shapes, on random blocks and on blocks with ties and flat subsets."""
import ctypes
import os

import numpy as np

import itw_testlib as T

SRC = os.path.join(T.ROOT, "tests", "emu", "bc7_pair_check.cpp")


def check_lib(tmp_path):
    """tests/emu/bc7_pair_check.cpp, compiled for the CPU like the emulation."""
    return ctypes.CDLL(T.build_emu().compile_cpu(SRC, str(tmp_path / "bc7_pair_check.so")))


def blocks():
    rng = np.random.default_rng(7)
    out = [rng.integers(0, 256, (64, 16, 4))]                                   # random
    out.append(rng.integers(0, 3, (64, 16, 4)) * 127)                           # three levels per channel: ties
    flat = np.repeat(rng.integers(0, 256, (32, 1, 4)), 16, axis=1)              # one colour: every subset flat
    out.append(flat)
    masks = rng.integers(0, 2, (64, 16, 1)).astype(bool)                        # two colours over a random split
    two = np.where(masks, rng.integers(0, 256, (64, 1, 4)), rng.integers(0, 256, (64, 1, 4)))
    out.append(two)
    near = rng.integers(100, 104, (32, 16, 4))                                  # spans below one unit after projection
    out.append(near)
    grey = np.repeat(rng.integers(0, 256, (32, 16, 1)), 4, axis=2)              # r = g = b = a
    out.append(grey)
    b = np.concatenate(out).astype(np.uint32)
    return np.ascontiguousarray(b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16) | (b[..., 3] << 24))


def test_pair_fit_equals_per_subset_routines(tmp_path):
    check = check_lib(tmp_path).pair_fit_check
    check.restype = ctypes.c_int
    tex = blocks()
    what = ctypes.create_string_buffer(256)
    bad = check(tex.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(tex)), what, ctypes.c_int(len(what)))
    assert bad == 0, f"{bad} mismatches, first: {what.value.decode()}"
