"""The preview dialog for HDR documents (include/itw_bcn.h section 18), on the CPU.

The exposed view: the kernel's per-texel routines (view_channels / view_exposure / view_texel<true> of csrc/view.cuh, through
tests/emu/view_hdr_emu.cpp) against the reference's own FetchPreviewRGB with the exposure as an argument (oracle/build_ref_view_exposed.py),
byte for byte: every slider exposure, exposure 1, the extremes 2^-10 and 2^10 and exposures off the slider's grid, every channel mask,
depths 8 / 16 / 32 with 1-4 planes and both panes, the float specials and products that overflow or straddle a FloatToByte boundary
in float but not in double.  The HDR pane: the non-WIC claim from the reference's own _UseWICConversion, the conversion kernel's
element rule against the reference's _Convert over every half, and every refusal of both calls before any CUDA call."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import open_converted_lib as OC
import preview_hdr_lib as H
import test_preview_uncompressed as PU
import test_preview_view as PV

B = T.binding
ALPHA = B.FRONT_HAS_ALPHA
OFF_GRID = (1.0, 2.0 ** -10, 2.0 ** 10, 0.3, 1.2345678, 3.1415927, 1e-3, 1e3, 0.9999999, 1.0000001, 255.0, 1 / 255, 1e-30, 1e30)


@pytest.fixture(scope="module")
def ref():
    if H.ref_view_exposed() is None:
        pytest.skip("reference view not built (no reference tree and no prebuilt oracle/_ref)")
    return H.ref_view_exposed()


def float_source(values, planes):
    """A 1-row-per-16-texels depth-32 source holding `values` in its elements (padded with zeros)."""
    n = -(-len(values) // (16 * planes)) * 16 * planes
    a = np.zeros(n, np.float32)
    a[:len(values)] = values
    return a.reshape(-1, 16, planes)


def compare(src, fmt, depth, exposure, masks, pitch_extra=0, zoom=1.0, x=0, y=0, mip=0, matte=0x102030):
    """emu == ref over the whole source (view = source size) for each mask; returns the reference bytes per mask."""
    h, w, planes = src.shape
    pitch = w * planes * depth // 8 + pitch_extra
    buf = PV.with_pitch(src, pitch)
    out = []
    for mask in masks:
        want = H.ref_fetch(buf, pitch, w, h, planes, fmt, w, h, x, y, zoom, mip, mask, matte, exposure)
        got = H.emu_fetch(buf, pitch, w, h, planes, depth, w, h, x, y, zoom, mip, mask, matte, exposure)
        assert np.array_equal(got, want), (fmt, planes, float(exposure), mask)
        out.append(want)
    return out


def test_every_slider_exposure(ref):
    """All 2001 exposures of the slider on a 4-plane float document: RGB, a cycling mask and a mixture with alpha in the blue slot."""
    rng = np.random.default_rng(1)
    vals = np.concatenate([PV.SPECIALS32, rng.random(400, dtype=np.float32) * np.float32(1.2) - np.float32(0.1),
                           (rng.random(100, dtype=np.float32) * np.float32(0.01)), [f for f, _ in H.straddling_pairs(32, seed=2)]])
    src = float_source(vals.astype(np.float32), 4)
    assert H.SLIDER.size == 2001 and H.SLIDER[1000] == 1.0 and H.SLIDER[0] == np.float32(2.0 ** -10) and H.SLIDER[-1] == 1024.0
    for i, e in enumerate(H.SLIDER):
        compare(src, 32, 32, e, (0, PV.MASKS[i % 16], B.VIEW_RED | B.VIEW_ALPHA))


def test_off_grid_exposures_every_kind_and_mask(ref):
    """Exposure 1, the extremes and exposures off the grid, over every channel mask, depths 8 / 16 / 32 with 1-4 planes and both panes
    (R8G8B8A8_UNORM and R32G32B32A32_FLOAT), at zooms, offsets and mip levels of the view matrix of tests/test_preview_view.py."""
    for kind in PV.KINDS:
        fmt, planes, depth = kind
        src = PV.source(kind, seed=fmt * 10 + planes)
        pitch = PV.row_pitch(kind)
        buf = PV.with_pitch(src, pitch)
        for j, e in enumerate(OFF_GRID):
            for mask in PV.MASKS:
                x, y, zoom, mip, matte = PV.views()[(j * 16 + mask) % len(PV.views())]
                args = (buf, pitch, PV.SRC_W, PV.SRC_H, planes)
                want = H.ref_fetch(*args, fmt, PV.VIEW_W, PV.VIEW_H, x, y, zoom, mip, mask, matte, e)
                got = H.emu_fetch(*args, depth, PV.VIEW_W, PV.VIEW_H, x, y, zoom, mip, mask, matte, e)
                assert np.array_equal(got, want), (kind, e, mask)
                if depth != 32:                                  # depths 8 and 16 ignore the exposure
                    assert np.array_equal(got, PV.emu_fetch(kind, buf, pitch, PV.VIEW_W, PV.VIEW_H, x, y, zoom, mip, mask, matte))


def test_exposure_one_is_the_unexposed_view(ref):
    for kind in PV.KINDS:
        fmt, planes, depth = kind
        src = PV.source(kind, seed=7 + planes)
        pitch = PV.row_pitch(kind)
        buf = PV.with_pitch(src, pitch)
        for mask in PV.MASKS:
            for x, y, zoom, mip, matte in PV.views()[::5]:
                got = H.emu_fetch(buf, pitch, PV.SRC_W, PV.SRC_H, planes, depth, PV.VIEW_W, PV.VIEW_H, x, y, zoom, mip, mask, matte, 1.0)
                assert np.array_equal(got, PV.emu_fetch(kind, buf, pitch, PV.VIEW_W, PV.VIEW_H, x, y, zoom, mip, mask, matte))


def test_float_product_not_double(ref):
    """Values whose float product with a slider exposure lands on one side of a k/255 truncation boundary while the exact product
    lands on the other: the emulation matches the reference, and a double-product implementation does not."""
    pairs = H.straddling_pairs(96, seed=3)
    for f, e in pairs:
        src = float_source(np.array([f, f, f, f], np.float32), 4)
        (got,) = compare(src, 32, 32, e, (B.VIEW_RED,))
        double_byte = H.float_to_byte(float(f) * float(e))
        assert got[0, 0, 0] == H.float_to_byte(float(np.float32(f * e))) != double_byte, (f, e)


def test_specials_and_overflow(ref):
    """NaN, infinities, -0, subnormals, and products that overflow to infinity or underflow to zero, for every mask and planes 1-4."""
    f32 = np.float32
    vals = np.array([np.nan, -np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-45, -1e-45, 1e-40, 1.1754942e-38, 3.4e38, -3.4e38, 2e38, 1e38,
                     0.5, 0.998, 1.0, 1.5, -0.25, 1 / 255, 254.5 / 255], f32)
    for planes in (1, 2, 3, 4):
        src = float_source(vals, planes)
        for e in (f32(2.0 ** 10), f32(2.0 ** -10), f32(2.0), f32(0.5), f32(1.0000001), f32(3.4e38), f32(1e-45)):
            compare(src, 32, 32, e, PV.MASKS)
    src = float_source(np.array([3.4e38, 1e-45], f32), 1)       # overflow to +inf shows 255, underflow to 0 shows 0
    (out,) = compare(src, 32, 32, f32(4.0), (B.VIEW_RED,))
    assert out[0, 0, 0] == 255
    (out,) = compare(src, 32, 32, f32(0.25), (B.VIEW_RED,))
    assert out[0, 1, 0] == 0


def test_pure_alpha_resets_the_exposure_and_a_mixture_does_not(ref):
    src = float_source(np.linspace(0.0, 0.5, 64, dtype=np.float32), 4)
    one = compare(src, 32, 32, 1.0, (B.VIEW_ALPHA, B.VIEW_RED | B.VIEW_ALPHA))
    four = compare(src, 32, 32, 4.0, (B.VIEW_ALPHA, B.VIEW_RED | B.VIEW_ALPHA))
    assert np.array_equal(one[0], four[0])                        # the pure-alpha view: exposure 1 (:615-621)
    assert not np.array_equal(one[1][..., 2], four[1][..., 2])     # the alpha in the blue slot moves with the slider


def test_hdr_pane_conversion_is_not_wic():
    """g_WICFormats marks R16G16B16A16_FLOAT linear and R8G8B8A8_UNORM sRGB, so the reference's own _UseWICConversion says no."""
    if OC.ref() is None:
        pytest.skip("reference converted-open cut not built")
    assert OC.ref().ref_use_wic(10, 28) == 0


def test_hdr_element_rule_every_half():
    """display_hdr_unorm8 (the element of hdr_unorm8_kernel and of the display kernel's kDisplayHdrUnorm rule) against the
    reference's _Convert(R16G16B16A16_FLOAT -> R8G8B8A8_UNORM) over all 65536 halves in every channel slot."""
    if OC.ref() is None:
        pytest.skip("reference converted-open cut not built")
    halves = np.arange(65536, dtype=np.uint16)
    got = np.zeros(65536, np.uint8)
    H.emu().emu_hdr_unorm8(halves.ctypes.data, halves.size, got.ctypes.data)
    for shift in range(4):                                          # each half in each of R, G, B, A
        rolled = np.roll(halves, shift)
        assert np.array_equal(np.roll(got, shift), H.ref_hdr_unorm8(rolled))
    # DirectXMath 3.06 reads exponent 31 as a number, not as infinity or NaN: +-65536 and up, so 255 and 0
    assert got[0x3C00] == 255 and got[0x7E00] == 255 and got[0xFE00] == 0 and got[0xFC00] == 0 and got[0x3800] == 128


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
def view_refusals():
    cases = [(name, s, v, dst, keep, 1.0) for name, s, v, dst, keep in PV.reject_cases(None)]
    a = np.zeros((8, 8, 4), np.float32)
    good = B.PixelSource(a.ctypes.data, 8, 8, 4, 32, 0)
    view = B.View(6, 5, 0, 0, 1.0, 0, 0, 0)
    dst = np.full((5, 6, 3), 0xAB, np.uint8)
    for e in (0.0, -0.0, -1.0, float("nan"), float("inf"), float("-inf"), -1e-45):
        cases.append((f"exposure {e}", good, view, dst, a, e))
    return cases


def test_view_refusals_before_any_cuda_call():
    p = T.product()
    for name, s, v, dst, keep, e in view_refusals():
        before = p.launch_count()
        rc = p.preview_view_exposed_raw(s, v, e, dst.ctypes.data if dst is not None else 0)
        assert rc != 0 and p.last_error().startswith("itw_preview_view_exposed:"), (name, p.last_error())
        assert p.launch_count() == before, name
        if dst is not None:
            assert (dst == 0xAB).all(), name


def pane_refusals():
    """itw_preview_uncompressed's refusal list with 95 in place of the dialog's other encodings, and the refusals of its own."""
    cases, keep = PU.refusal_cases()
    out = []
    for name, o, doc, layers, flags, display in cases:
        if name.startswith(("BC4", "BC5", "BC6H", "format")):           # refusals of an encoding: their own list below
            continue
        if o is not None and o.dxgi_format in PU.U.ENCODINGS:
            o = B.PaneOptions(95, o.texture, o.mip_level)
        out.append((name, o, doc, layers, flags, display, None))
    doc = np.zeros((12, 16, 4), np.float32)
    disp = np.full((12, 16, 4), 0xAB, np.uint8)
    cross = np.full((3, 4, 4), 0xAB, np.uint8)
    keep += [doc, disp, cross]
    src = B.PixelSource(doc.ctypes.data, 16, 12, 4, 32, 0)
    surf = B.RgbaSurface(disp.ctypes.data, 16, 12, 64)
    csurf = B.RgbaSurface(cross.ctypes.data, 4, 3, 16)
    layer = B.ItwBcn.cube_faces([([doc[..., 0], doc[..., 1], doc[..., 2]], None)], np.float32, keep)
    O, D2, CR = B.PaneOptions, B.PANE_2D, B.PANE_CUBE_CROSS
    for fmt in (28, 71, 72, 77, 78, 80, 83, 98, 99, 96, 2, 10, 0):
        out.append((f"format {fmt}", O(fmt, D2, -1), src, layer, 0, surf, "itw_preview_uncompressed"))
    out += [("flip x", O(95, D2, -1), src, layer, B.FRONT_FLIP_X, surf, "normal-map"),
            ("flip y", O(95, D2, -1), src, layer, B.FRONT_FLIP_Y | ALPHA, surf, "normal-map"),
            ("flip on a cross", O(95, CR, 2), src, None, B.FRONT_FLIP_X, csurf, "normal-map"),
            ("gamma", O(95, CR, 2), src, None, B.FRONT_GAMMA, csurf, "gamma"),
            ("normalise", O(95, D2, -1), src, layer, B.FRONT_NORMALIZE, surf, "normalisation"),
            ("2-D without layer 0", O(95, D2, -1), src, None, 0, surf, "itw_preview_pixels"),
            ("2-D without layer 0, alpha", O(95, D2, -1), src, None, ALPHA, surf, "layer 0")]
    return out, keep


def test_pane_refusals_before_any_cuda_call():
    p = T.product()
    cases, keep = pane_refusals()
    for name, o, doc, layers, flags, display, text in cases:
        before = p.launch_count()
        rc = p.preview_uncompressed_hdr_raw(o, doc, layers, flags, display)
        err = p.last_error()
        assert rc != 0 and err != "", name
        assert p.launch_count() == before, name
        if text:                                                      # the refusals of this call name it and their reason
            assert err.startswith("itw_preview_uncompressed_hdr:") and text in err, (name, err)
    for a in keep:
        if isinstance(a, np.ndarray) and a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 4:
            assert (a == 0xAB).all()


def test_the_original_call_still_refuses_95():
    """itw_preview_uncompressed keeps its verdict and its text for 95."""
    p = T.product()
    doc = np.zeros((4, 4, 4), np.float32)
    disp = np.full((4, 4, 4), 0xAB, np.uint8)
    rc = p.preview_uncompressed_raw(B.PaneOptions(95, B.PANE_CUBE_CROSS, -1), B.PixelSource(doc.ctypes.data, 4, 4, 4, 32, 0), None, 0,
                                    B.RgbaSurface(disp.ctypes.data, 4, 4, 16), None)
    assert rc != 0 and p.last_error() == ("itw_preview_uncompressed: dxgi_format 95 (BC6H_UF16) is not supported: its pane is "
                                          "DirectX::Convert from R16G16B16A16_FLOAT, which DirectXTex hands to WIC")
    assert (disp == 0xAB).all()
