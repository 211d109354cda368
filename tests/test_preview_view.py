"""The preview dialog's view of a pane (include/itw_bcn.h section 11, itw_preview_view): FetchPreviewRGB on the GPU.

CPU: the kernel's per-texel routines (view_channels / view_texel in csrc/view.cuh, run through tests/emu/view_emu.cpp) against the
reference's own channel table and sampling loops (IntelPlugin.cpp:585-739, cut by oracle/build_ref_view.py), byte for byte, over
every channel mask, every source kind (documents of depth 8 / 16 / 32 with 1-4 planes, both panes), zooms the dialog passes, mip
levels 0-3, offsets before, at and past the source, several matte colours, and the float specials at depth 32.  Argument
rejections, which happen before any CUDA call.  tests/test_preview_view_gpu.py runs the same matrix on the GPU."""
import ctypes
import functools
import os
import sys

import numpy as np
import pytest

import itw_testlib as T

B = T.binding
MASKS = [m << 2 for m in range(16)]                     # every combination of ITW_VIEW_RED / GREEN / BLUE / ALPHA, 0 = RGB
# (depth or DXGI format the plug-in switches on, planes, depth of the itw_pixel_source): the document, then the two panes
KINDS = [(d, p, d) for d in (8, 16, 32) for p in (1, 2, 3, 4)] + [(28, 4, 8), (2, 4, 32)]
# 1.f / previewZoom for zoom steps of the dialog and values that are not exact in binary
ZOOMS = [float(np.float32(1) / np.float32(z)) for z in (0.01, 0.1, 0.3, 0.7, 1.0, 1.7, 3.0, 4.0)] + [1 / 3, 0.45]
MATTES = (0x000000, 0xFF8040, 0x123456)
SPECIALS32 = np.array([np.nan, -np.nan, np.inf, -np.inf, -0.0, 0.0, -1.5, -1e-30, 1.0, 1.0000001, 7.5, 1e30, 1e-45, 1e-40, 1.1754942e-38,
                       0.99999994, 0.5, 1 / 255, 0.003921568], np.float32)
SRC_W, SRC_H = 37, 23
VIEW_W, VIEW_H = 29, 17


def source(kind, seed):
    """H x W x planes elements of the kind's depth; panes carry a row pitch wider than the texels."""
    fmt, planes, depth = kind
    rng = np.random.default_rng(seed)
    if depth == 8:
        a = rng.integers(0, 256, (SRC_H, SRC_W, planes), dtype=np.uint8)
    elif depth == 16:
        a = rng.integers(0, 32769, (SRC_H, SRC_W, planes), dtype=np.uint16)
        a.reshape(-1)[:6] = [32768, 32767, 40000, 65535, 0, 129]
    else:
        a = (rng.random((SRC_H, SRC_W, planes), dtype=np.float32) * 1.4 - 0.2).astype(np.float32)
        a.reshape(-1)[:SPECIALS32.size] = SPECIALS32
        a.reshape(-1)[-SPECIALS32.size:] = SPECIALS32[::-1]
    return a


def row_pitch(kind):
    """Bytes between rows: tight for documents, a wider display stride for the panes."""
    fmt, planes, depth = kind
    tight = SRC_W * planes * depth // 8
    return tight + (48 if fmt in (2, 28) else 0)


def with_pitch(a, pitch):
    """`a` in a buffer whose rows are `pitch` bytes apart (as an H x pitch uint8 array)."""
    h = a.shape[0]
    buf = np.zeros((h, pitch), np.uint8)
    raw = a.reshape(h, -1).view(np.uint8)
    buf[:, :raw.shape[1]] = raw
    return buf


def views():
    """(x, y, zoom, mip, matte) covering offsets before, at and past the source, every zoom and mip level."""
    out = []
    offsets = [(0, 0), (-1, -1), (-7, 3), (5, -2), (SRC_W - 3, SRC_H - 2), (SRC_W + 4, 0), (-40, -30), (2000, 9)]
    i = 0
    for z in ZOOMS:
        for mip in range(4):
            x, y = offsets[i % len(offsets)]
            out.append((x, y, z, mip, MATTES[i % len(MATTES)]))
            i += 1
    for x, y in offsets:                                         # every offset at zoom 1/4.f, where (-1 + xt) * 0.25 lands on 0
        out.append((x, y, ZOOMS[-3], 0, MATTES[1]))
    return out


@functools.lru_cache(None)
def ref_view():
    """oracle/_ref/libitw_ref_view.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_view
        try:
            path = build_ref_view.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_fetch_preview_rgb.restype = None
    lib.ref_fetch_preview_rgb.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int,
                                          ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_int]
    return lib


def ref_fetch(kind, buf, pitch, w, h, x, y, zoom, mip, mask, matte):
    """FetchPreviewRGB of the reference cut into an h x w x 3 buffer."""
    fmt, planes, depth = kind
    out = np.zeros((h, w, 3), np.uint8)
    ref_view().ref_fetch_preview_rgb(out.ctypes.data, w, h, x, y, zoom, mask, matte, buf.ctypes.data, SRC_W, SRC_H, planes, fmt, pitch, mip)
    return out


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_view_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_view.restype = None
    lib.emu_view.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                             ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_uint, ctypes.c_uint, ctypes.c_void_p]
    return lib


def emu_fetch(kind, buf, pitch, w, h, x, y, zoom, mip, mask, matte):
    fmt, planes, depth = kind
    out = np.zeros((h, w, 3), np.uint8)
    emu().emu_view(buf.ctypes.data, SRC_W, SRC_H, planes, depth, pitch, w, h, x, y, zoom, mip, mask, matte, out.ctypes.data)
    return out


@pytest.fixture(scope="module")
def ref_lib():
    if ref_view() is None:
        pytest.skip("reference view not built (no reference tree and no prebuilt oracle/_ref)")
    return ref_view()


@pytest.mark.parametrize("kind", KINDS, ids=lambda k: f"fmt{k[0]}-p{k[1]}")
def test_emulated_view_matches_reference(ref_lib, kind):
    buf_src = source(kind, seed=kind[0] * 10 + kind[1])
    pitch = row_pitch(kind)
    buf = with_pitch(buf_src, pitch)
    shown_matte = 0
    for mask in MASKS:
        for x, y, zoom, mip, matte in views():
            want = ref_fetch(kind, buf, pitch, VIEW_W, VIEW_H, x, y, zoom, mip, mask, matte)
            got = emu_fetch(kind, buf, pitch, VIEW_W, VIEW_H, x, y, zoom, mip, mask, matte)
            assert np.array_equal(got, want), (mask, x, y, zoom, mip, matte)
            shown_matte += int((want == np.array([matte & 255, (matte >> 8) & 255, matte >> 16], np.uint8)).all(-1).sum())
    assert shown_matte > 0                                       # the matrix reaches the out-of-bounds texels


def test_specials_reach_every_byte_rule(ref_lib):
    """At depth 32 the specials land in the view: NaN, infinities, negatives, values above 1 and denormals each give their byte."""
    kind = (32, 1, 32)
    a = np.zeros((SRC_H, SRC_W, 1), np.float32)
    a.reshape(-1)[:SPECIALS32.size] = SPECIALS32
    buf = with_pitch(a, row_pitch(kind))
    want = ref_fetch(kind, buf, row_pitch(kind), SRC_W, SRC_H, 0, 0, 1.0, 0, B.VIEW_RED, 0)
    got = emu_fetch(kind, buf, row_pitch(kind), SRC_W, SRC_H, 0, 0, 1.0, 0, B.VIEW_RED, 0)
    assert np.array_equal(got, want)
    first = want[0, :SPECIALS32.size, 0].tolist()
    assert first[:4] == [0, 0, 255, 0] and first[8] == 255 and first[11] == 255 and first[12] == 0


def reject_cases(p):
    """(description, source, view, dst) triples that itw_preview_view must refuse."""
    a = np.zeros((8, 8, 4), np.uint8)
    good_src = B.PixelSource(a.ctypes.data, 8, 8, 4, 8, 0)
    good_view = B.View(6, 5, 0, 0, 1.0, 0, 0, 0)
    dst = np.full((5, 6, 3), 0xAB, np.uint8)

    def src(**kw):
        s = B.PixelSource(a.ctypes.data, 8, 8, 4, 8, 0)
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def view(**kw):
        v = B.View(6, 5, 0, 0, 1.0, 0, 0, 0)
        for k, val in kw.items():
            setattr(v, k, val)
        return v
    cases = [("null source", None, good_view), ("null data", src(data=None), good_view), ("null view", good_src, None),
             ("depth 24", src(depth=24), good_view), ("planes 0", src(planes=0), good_view), ("planes 5", src(planes=5), good_view),
             ("short row_bytes", src(row_bytes=31), good_view), ("source width 0", src(width=0), good_view),
             ("source height -1", src(height=-1), good_view), ("view width 0", good_src, view(width=0)),
             ("view height -3", good_src, view(height=-3)), ("zoom 0", good_src, view(zoom=0.0)), ("zoom -1", good_src, view(zoom=-1.0)),
             ("zoom nan", good_src, view(zoom=float("nan"))), ("zoom inf", good_src, view(zoom=float("inf"))),
             ("mip -1", good_src, view(mip_level=-1)), ("mip 31", good_src, view(mip_level=31)),
             ("source bits", good_src, view(channels=0x1)), ("unknown bits", good_src, view(channels=0x40))]
    return [(name, s, v, dst, a) for name, s, v in cases] + [("null dst", good_src, good_view, None, a)]


def test_rejections_before_any_cuda_call():
    p = T.product()
    for name, s, v, dst, keep in reject_cases(p):
        rc = p.preview_view_raw(s, v, dst.ctypes.data if dst is not None else 0)
        assert rc != 0 and p.last_error().startswith("itw_preview_view:"), name
        if dst is not None:
            assert (dst == 0xAB).all(), name
