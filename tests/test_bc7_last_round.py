"""BC7's last round: the blocks left after the full rounds (16 blocks per warp on every warp of the grid) are dealt over all
warps of the grid, 1, 2, 4, 8 or 16 blocks per warp.  One surface per per-warp count, sized from the device's SM count, with a
ragged last warp, plus surfaces smaller than one round; every block of the last round and a fixed sample of the full round
against the oracle."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import itw_testlib as T

pytestmark = pytest.mark.gpu

WARPS_PER_CTA, FULL_PER_WARP = 16, 16


def _oracle_blocks(img, idx, prof):
    """Oracle encode of the blocks `idx` of a one-block-row surface: blocks are independent, so they are packed into strips of
    their own and encoded on several threads."""
    oracle = T.oracle()
    blocks = img.reshape(4, -1, 4, 4).transpose(1, 0, 2, 3)[idx]          # (n, 4 rows, 4 texels, 4 channels)
    chunks = np.array_split(np.arange(len(idx)), max(1, min(16, len(idx) // 64)))

    def work(c):
        strip = np.ascontiguousarray(blocks[c].transpose(1, 0, 2, 3).reshape(4, 4 * len(c), 4))
        return T.run(oracle, "BC7", strip, prof).reshape(-1, 16)

    with ThreadPoolExecutor(len(chunks)) as ex:
        return np.concatenate(list(ex.map(work, chunks)))


def _surfaces(sms):
    warps = sms * WARPS_PER_CTA
    wave = warps * FULL_PER_WARP
    out = []
    # remainder r takes p blocks per warp when ceil(r / (p / 2)) > warps >= ceil(r / p); an odd r leaves the last warp ragged
    for p, rem in ((1, warps - 5), (2, warps + 3), (4, 2 * warps + 3), (8, 4 * warps + 5), (16, 8 * warps + 7)):
        assert -(-rem // p) <= warps and (p == 1 or -(-rem // (p // 2)) > warps)
        out.append((f"p{p}", wave + rem, wave))
    out.append(("small100", 100, 0))                  # fewer blocks than SMs x 16: one CTA per 16 blocks, one block per warp
    out.append(("small3001", 3001, 0))                # one round of two blocks per warp, no full round
    return out


@pytest.mark.parametrize("prof", ["basic", "slow"])
def test_last_round_every_blocks_per_warp(prof):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lib = T.product()
    rng = np.random.default_rng(23)
    for name, nblocks, last_first in _surfaces(sms):
        img = rng.integers(0, 256, (4, 4 * nblocks, 4)).astype(np.uint8)
        img[:, : 4 * (nblocks // 3), 3] = 255                                 # opaque and translucent blocks
        got = T.run(lib, "BC7", img, prof).reshape(-1, 16)
        idx = np.arange(last_first, nblocks)
        if last_first > 0:
            idx = np.concatenate([np.sort(rng.choice(last_first, 256, replace=False)), idx])
        want = _oracle_blocks(img, idx, prof)
        bad = np.flatnonzero((got[idx] != want).any(1))
        assert bad.size == 0, f"{prof}/{name}: {bad.size} of {idx.size} checked blocks differ, first at block {idx[bad[0]]}"
