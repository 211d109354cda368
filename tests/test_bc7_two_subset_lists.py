"""BC7 modes 1 and 3 take one of two paths: when the longer of their two candidate lists holds all 64 two-subset shapes, every
subset mask is fitted and searched and the errors are read back in ranked order; otherwise only the top t ranked shapes are
evaluated.  A full list next to a short (or empty) one, in both orders, must still give the first minimum of each list in
ranked order -- on blocks with many tied errors, where that order decides."""
import os
import re

import numpy as np
import pytest

import itw_testlib as T

LISTS = [(64, 0), (64, 1), (64, 9), (0, 64), (7, 64), (63, 64)]


def settings(api, channels, t1, t3):
    s = api.profile("slow" if channels == 3 else "alpha_slow")
    s.fastSkipTreshold_mode1 = t1
    s.fastSkipTreshold_mode3 = t3
    return s


def shape_masks():
    src = open(os.path.join(T.ROOT, "intel-texture-works-plugin_b200", "csrc", "itw_tables.cuh")).read()
    body = re.search(r"#define ITW_TABLE_INIT_shape_mask01 \\\n(.*?)\n\n", src, re.S).group(1)
    return [int(x.rstrip("u"), 16) & 0xFFFF for x in re.findall(r"0x[0-9A-Fa-f]+u?", body)][:64]


def images(channels):
    """Blocks of two colours split along a random two-subset shape (modes 1 and 3 win many of them), with a little noise or with
    few distinct values (tied shape errors)."""
    rng = np.random.default_rng(23)
    masks = shape_masks()
    out = []
    for noise in (4, 0):
        img = np.zeros((8, 32, 4), np.uint8)
        for by in range(2):
            for bx in range(8):
                m = masks[int(rng.integers(0, 64))]
                c = (rng.integers(0, 3, (2, 4)) * 120 if noise == 0 else rng.integers(0, 252, (2, 4))).astype(np.int64)
                for k in range(16):
                    v = c[0 if (m >> k) & 1 else 1] + rng.integers(0, noise + 1, 4)
                    img[4 * by + k // 4, 4 * bx + k % 4] = np.clip(v, 0, 255)
        if channels == 3:
            img[..., 3] = 255
        out.append(img)
    return out


@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("t1,t3", LISTS)
def test_full_and_short_two_subset_lists_emulated(t1, t3, channels):
    emu, oracle = T.emu(), T.oracle()
    for img in images(channels):
        got = emu.encode("BC7", img, settings(emu, channels, t1, t3))
        assert np.array_equal(got, oracle.encode("BC7", img, settings(oracle, channels, t1, t3))), (t1, t3, channels)


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("t1,t3", LISTS)
def test_full_and_short_two_subset_lists_gpu(t1, t3, channels):
    lib, oracle = T.product(), T.oracle()
    for img in images(channels):
        got = lib.encode("BC7", img, settings(lib, channels, t1, t3))
        assert np.array_equal(got, oracle.encode("BC7", img, settings(oracle, channels, t1, t3))), (t1, t3, channels)
