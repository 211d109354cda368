"""The display decompressor's per-block logic (csrc/display.cuh, run on the CPU) against the reference's own DirectX::Decompress
(oracle/build_ref_preview.py) for every (source, target) pair, and its sRGB tables against the oracle's sRGB functions."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import preview_lib as P

needs_ref = pytest.mark.skipif(P.ref() is None, reason="oracle/_ref/libitw_ref_preview.so unavailable")


def streams(src):
    profiles = {"BC7": ("ultrafast", "basic", "alpha_basic"), "BC6H": ("bc6h_veryfast", "bc6h_basic")}.get(P.NAME[src], (None,))
    yield from P.encoded_streams(src, profiles)
    yield "random", P.random_blocks(src, 64 * 72, seed=src), 256, 288


@needs_ref
@pytest.mark.parametrize("pair", sorted(P.PAIRS), ids=lambda p: f"{p[0]}-to-{p[1]}")
def test_display_logic_equals_directxtex(pair):
    src, target = pair
    for tag, blocks, w, h in streams(src):
        got, want = P.emu_decompress(src, blocks, w, h, target), P.ref_decompress(src, blocks, w, h, target)
        bad = np.argwhere((got.view(np.uint8).reshape(h, w, -1) != want.view(np.uint8).reshape(h, w, -1)).any(-1))
        assert bad.size == 0, f"{pair} {tag}: {len(bad)} texels differ, first {bad[:4].tolist()}"


@needs_ref
@pytest.mark.parametrize("pair", sorted(P.PAIRS), ids=lambda p: f"{p[0]}-to-{p[1]}")
def test_display_logic_ragged_sizes(pair):
    src, target = pair
    for w in range(1, 10):
        for h in range(1, 10):
            blocks = P.random_blocks(src, P.nblocks(w, h), seed=100 * w + h)
            got, want = P.emu_decompress(src, blocks, w, h, target), P.ref_decompress(src, blocks, w, h, target)
            assert got.tobytes() == want.tobytes(), f"{pair} {w}x{h}"


def _bc1_floats():
    out = set()
    for bits in (5, 6):
        e = np.arange(1 << bits, dtype=np.float32) * np.float32(1.0 / ((1 << bits) - 1))
        f0, f1 = [a.ravel() for a in np.meshgrid(e, e, indexing="ij")]
        out.update(e.tolist())
        for t in (np.float32(1.0 / 3.0), np.float32(2.0 / 3.0), np.float32(0.5)):
            out.update(((f1 - f0) * t + f0).astype(np.float32).tolist())
    return np.array(sorted(out), np.float32)


def _store8(x):
    x = np.clip(np.float32(x), np.float32(0), np.float32(1))
    return int(x * np.float32(255) + np.float32(0.5))


def test_bc1_srgb_thresholds_exhaustive():
    """Every float the BC1 / BC3 colour decoder can hand over (every 5- and 6-bit endpoint pair x every weight), both directions,
    plus both sides of every threshold of the SRGB-in table."""
    o, e = T.oracle().lib, P.emu()
    o.oracle_srgb_to_linear.restype = ctypes.c_float
    o.oracle_srgb_to_linear.argtypes = [ctypes.c_float]
    o.oracle_linear_to_srgb8.restype = ctypes.c_int
    o.oracle_linear_to_srgb8.argtypes = [ctypes.c_float]
    for f in _bc1_floats():
        f = float(f)
        assert e.emu_srgb_in_store(f) == _store8(o.oracle_srgb_to_linear(f)), f
        assert e.emu_srgb_out_store(f) == o.oracle_linear_to_srgb8(f), f
    import re
    text = open(T.ROOT + "/intel-texture-works-plugin_b200/csrc/display_tables.cuh").read()
    block = text.split("ITW_TABLE_INIT_srgb_in_threshold")[1].split("#define")[0]
    thresholds = [int(v, 16) for v in re.findall(r"0x([0-9A-F]{8})u", block)]
    assert len(thresholds) == 255
    for k, t in enumerate(thresholds, 1):
        at, below = np.array([t, t - 1], np.uint32).view(np.float32)
        assert _store8(o.oracle_srgb_to_linear(float(at))) >= k > _store8(o.oracle_srgb_to_linear(float(below)))
        assert e.emu_srgb_in_store(float(at)) == k and e.emu_srgb_in_store(float(below)) == k - 1


@needs_ref
@pytest.mark.parametrize("target", [28, 29])
def test_bc4_shows_grey(target):
    """BC4 is an R format: DirectX::Decompress copies red into green and blue for an RGB target (DirectXTexConvert.cpp:3445-3457)."""
    blocks = np.array([200, 200, 0, 0, 0, 0, 0, 0, 17, 90, 0x49, 0x92, 0x24, 0x49, 0x92, 0x24], np.uint8)    # constant + a ramp
    for got in (P.ref_decompress(80, blocks, 8, 4, target), P.emu_decompress(80, blocks, 8, 4, target)):
        assert (got[..., 0] > 0).all() and (got[..., 1] == got[..., 0]).all() and (got[..., 2] == got[..., 0]).all()
        assert (got[..., 3] == 255).all()
    assert P.emu_decompress(80, blocks, 8, 4, target).tobytes() == P.ref_decompress(80, blocks, 8, 4, target).tobytes()


@pytest.mark.parametrize("fmt", [71, 99, 95])
@pytest.mark.parametrize("flags", [0, T.binding.FRONT_FLIP_X | T.binding.FRONT_FLIP_Y])
def test_preview_oracle_cross_layout(fmt, flags):
    """The preview oracle's cross before encoding: face i lands in cell CROSS[i] of the 4w x 3h image, and every other cell holds
    the zero texel (alpha 0) after the normal-map flips."""
    faces = [P.document(5, 3, 4, 8 if fmt != 95 else 16, seed=i) for i in range(6)]
    img = P.oracle_cross(fmt, faces, flags)
    assert img.shape == (9, 20, 4)
    o = T.oracle()
    covered = np.zeros((9, 20), bool)
    for face, (cx, cy) in zip(faces, P.CROSS):
        want = o.convert_pixels(P.NAME[fmt], face, flags, pad=False)
        assert np.array_equal(img[3 * cy:3 * cy + 3, 5 * cx:5 * cx + 5], want), (cx, cy)
        covered[3 * cy:3 * cy + 3, 5 * cx:5 * cx + 5] = True
    flip = flags != 0
    if fmt == 95:
        blank = [0x3C00, 0x3C00, 0, 0] if flip else [0, 0, 0, 0]        # half(1 - 0) = 1.0
    else:
        blank = [255, 255, 0, 0] if flip else [0, 0, 0, 0]
    assert (img[~covered] == np.array(blank, img.dtype)).all()
    assert np.array_equal(P.oracle_cross(fmt, [faces[4]], flags), o.convert_pixels(P.NAME[fmt], faces[4], flags, pad=False))
