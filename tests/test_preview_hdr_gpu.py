"""The preview dialog for HDR documents on the GPU (include/itw_bcn.h section 18), byte for byte against the oracles of
tests/preview_hdr_lib.py.

itw_preview_view_exposed: the 32-bit document (host and device, 1-4 planes) and the R32G32B32A32_FLOAT panes itw_preview_pixels and
itw_preview_cube build for BC6H_UF16, at slider exposures, the extremes and exposures off the grid, with zoom, offset, mip level and
matte, against the reference's FetchPreviewRGB with the exposure; exposure 1 against itw_preview_view.
itw_preview_uncompressed_hdr: depths 8, 16 and 32 (the HDR corpus of tests/hdr_corpus.py at depth 32, with infinities, NaN and values
above the half range), crosses without and with a set level, the layers cube with missing faces and one-channel faces, layer 0 with
and without alpha; host and device documents and displays, displays built in place and staged; refusals and the kernel time."""
import ctypes
import itertools

import numpy as np
import pytest

import cube_lib as C
import hdr_corpus as HC
import itw_testlib as T
import preview_hdr_lib as H
import preview_uncompressed_lib as U

B = T.binding
ALPHA = B.FRONT_HAS_ALPHA
pytestmark = pytest.mark.gpu
EXPOSURES = (1.0, float(H.SLIDER[0]), float(H.SLIDER[-1]), float(H.SLIDER[1234]), float(H.SLIDER[777]), 0.3, 1.2345678, 1e-3)
MASKS = [m << 2 for m in range(16)]


@pytest.fixture(scope="module")
def ref_view():
    if H.ref_view_exposed() is None:
        pytest.skip("reference view not built (no reference tree and no prebuilt oracle/_ref)")


@pytest.fixture(scope="module")
def ref_pane():
    if not H.available():
        pytest.skip("reference cuts not built (no reference tree and no prebuilt oracle/_ref)")


def dev(a, keep):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    keep.append(t)
    return t.data_ptr()


def view_on_gpu(p, buf, pitch, w, h, planes, depth, view, exposure, device):
    """itw_preview_view_exposed of `buf` (h rows of `pitch` bytes) into a host or device dialog buffer."""
    import torch
    keep = []
    src = B.PixelSource(dev(buf, keep) if device else buf.ctypes.data, w, h, planes, depth, pitch)
    if device:
        out = torch.zeros((view.height, view.width, 3), dtype=torch.uint8, device="cuda")
        assert p.preview_view_exposed_raw(src, view, exposure, out.data_ptr()) == 0, p.last_error()
        torch.cuda.synchronize()
        return out.cpu().numpy()
    out = np.zeros((view.height, view.width, 3), np.uint8)
    assert p.preview_view_exposed_raw(src, view, exposure, out.ctypes.data) == 0, p.last_error()
    return out


def check_view(p, buf, pitch, w, h, planes, fmt, depth, i):
    """Every mask at one view per (exposure, mask), host and device operands in turn."""
    for j, (e, mask) in enumerate(itertools.product(EXPOSURES, MASKS)):
        k = i + j
        x, y = ((0, 0), (-5, 3), (7, -2), (w - 3, h - 2), (-40, -30))[k % 5]
        zoom = (1.0, float(np.float32(1) / np.float32(1.7)), float(np.float32(1) / np.float32(0.3)), 0.45)[k % 4]
        mip, matte = k % 3, (0x000000, 0xFF8040, 0x123456)[k % 3]
        view = B.View(41, 27, x, y, zoom, mip, mask, matte)
        got = view_on_gpu(p, buf, pitch, w, h, planes, depth, view, e, device=(k % 2 == 1))
        want = H.ref_fetch(buf, pitch, w, h, planes, fmt, 41, 27, x, y, zoom, mip, mask, matte, e)
        assert np.array_equal(got, want), (fmt, planes, e, mask, x, y, zoom, mip)
        if e == 1.0:
            src = B.PixelSource(buf.ctypes.data, w, h, planes, depth, pitch)
            plain = np.zeros_like(got)
            assert p.preview_view_raw(src, view, plain.ctypes.data) == 0
            assert np.array_equal(got, plain)


def test_view_of_the_document(ref_view):
    p = T.product()
    for planes in (1, 2, 3, 4):
        doc = HC.product_defined_planes(45, 60, seed=planes)[..., :planes].copy()
        doc.reshape(-1)[:8] = [np.nan, np.inf, -np.inf, -0.0, 1e-45, 3.4e38, 0.5, 1.0]
        pitch = 60 * planes * 4 + (16 if planes == 3 else 0)
        buf = np.zeros((45, pitch), np.uint8)
        buf[:, :60 * planes * 4] = doc.reshape(45, -1).view(np.uint8)
        check_view(p, buf, pitch, 60, 45, planes, 32, 32, planes)


def test_view_of_depth_8_and_16_ignores_the_exposure(ref_view):
    p = T.product()
    for depth, dtype, top in ((8, np.uint8, 256), (16, np.uint16, 32769)):
        doc = np.random.default_rng(depth).integers(0, top, (20, 30, 4)).astype(dtype)
        buf = np.ascontiguousarray(doc.reshape(20, -1).view(np.uint8))
        check_view(p, buf, 30 * 4 * depth // 8, 30, 20, 4, depth, depth, 0)


def test_view_of_the_bc6h_float_panes(ref_view):
    """The R32G32B32A32_FLOAT compressed panes of a 32-bit document saved as BC6H_UF16: itw_preview_pixels (2-D) and itw_preview_cube
    (a cross of level 1 and the layers cube), viewed through the exposed view."""
    p = T.product()
    doc = HC.family_planes("exposure_ramp", 48, 64)
    panes = [p.preview_pixels(95, [doc], 0, p.profile("bc6h_veryfast"))[0],
             p.preview_cube(B.CubeOptions(95, B.CUBE_CROSS, 0, 1), doc, None, 0, p.profile("bc6h_veryfast"))[0]]
    faces = U.cube_layers(16, 12, 32, seed=3, missing=(2,))
    panes.append(p.preview_cube(B.CubeOptions(95, B.CUBE_LAYERS, 0, -1), HC.family_planes("log_uniform", 12, 16), faces, ALPHA,
                                p.profile("bc6h_veryfast"))[0])
    for i, pane in enumerate(panes):
        assert pane.dtype == np.float32 and pane.shape[2] == 4
        h, w = pane.shape[:2]
        pitch = w * 16 + 32
        buf = np.zeros((h, pitch), np.uint8)
        buf[:, :w * 16] = np.ascontiguousarray(pane).reshape(h, -1).view(np.uint8)
        check_view(p, buf, pitch, w, h, 4, 2, 32, i)


# ---- itw_preview_uncompressed_hdr --------------------------------------------------------------------------------------------------
def run(p, texture, level, doc, layers, flags, device=False, pad=0, host_display=False):
    """The call with host operands, or with device document / layers and a device display `pad` bytes wider than a row (filled with
    a sentinel that must survive outside the pane; an odd pad makes the display unaligned, so it is staged)."""
    import torch
    if not device and host_display:
        return p.preview_uncompressed_hdr(B.PaneOptions(95, texture, level), doc, layers, flags)
    dh, dw = doc.shape[:2]
    w, h = U.pane_size(texture, level, dw, dh)
    keep = []
    docp = np.ascontiguousarray(doc)
    src = B.PixelSource(dev(docp, keep) if device else docp.ctypes.data, dw, dh, doc.shape[2], doc.itemsize * 8, 0)
    arr = None
    if layers is not None:
        arr = (B.LayerSource * 6)()
        for i, face in enumerate([layers] if texture == B.PANE_2D else layers):
            if face is None:
                continue
            channels, alpha = face
            arr[i].channel_count = len(channels)
            for c, pl in enumerate(channels):
                pl = np.ascontiguousarray(pl, doc.dtype)
                keep.append(pl)
                arr[i].channels[c] = dev(pl, keep) if device else pl.ctypes.data
            if alpha is not None:
                a = np.ascontiguousarray(alpha, doc.dtype)
                keep.append(a)
                arr[i].alpha = dev(a, keep) if device else a.ctypes.data
    stride = w * 4 + pad
    disp = torch.full((h * stride + 4,), 0xAB, dtype=torch.uint8, device="cuda")
    off = pad & 1                                                      # an odd pad: an unaligned pointer too
    rc = p.preview_uncompressed_hdr_raw(B.PaneOptions(95, texture, level), src, arr, flags,
                                        B.RgbaSurface(disp.data_ptr() + off, w, h, stride))
    assert rc == 0, p.last_error()
    torch.cuda.synchronize()
    out = disp.cpu().numpy()
    assert (out[:off] == 0xAB).all() and (out[off + h * stride:] == 0xAB).all()
    rows = out[off:off + h * stride].reshape(h, stride)
    assert (rows[:, w * 4:] == 0xAB).all()                             # nothing outside the pane's rows
    return rows[:, :w * 4].reshape(h, w, 4)


def check(p, texture, level, doc, layers, flags, device=False, pad=0, host_display=False):
    want = H.oracle_pane(texture, level, doc, layers, flags)
    got = run(p, texture, level, doc, layers, flags, device, pad, host_display)
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.argwhere((got != want).any(-1))
    assert bad.size == 0, (texture, level, doc.shape, doc.dtype, flags, device, pad, bad[:4].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])


def document(w, h, planes, depth, seed):
    """Depth 32 from the HDR corpus (infinities, NaN, values above the half range, negative values), else the uncompressed pane's
    documents."""
    if depth == 32:
        names = ("log_uniform", "order_cells", "exposure_ramp", "boundary", "normal_vectors")
        base = HC.product_defined_planes(h, w, seed) if seed % 3 == 0 else HC.family_planes(names[seed % len(names)], h, w, seed)
        return np.ascontiguousarray(base[..., :planes])
    return U.document(w, h, planes, depth, seed)


def layer(w, h, depth, channels, alpha, seed):
    d = document(w, h, channels + (1 if alpha else 0), depth, seed)
    return [d[..., c].copy() for c in range(channels)], (d[..., channels].copy() if alpha else None)


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_2d_pane_from_layer_0(ref_pane, depth):
    p = T.product()
    i = 0
    for (w, h), planes in itertools.product(((1, 1), (5, 3), (130, 67), (64, 64)), (1, 3, 4)):
        doc = document(w, h, planes, depth, seed=w * 7 + planes + depth)
        for channels, alpha in ((1, False), (3, True), (2, True), (3, False)):
            for flags in ((0, ALPHA) if planes == 4 or (planes == 3 and depth == 32) else (0,)):
                check(p, B.PANE_2D, -1, doc, layer(w, h, depth, channels, alpha, seed=i), flags, device=(i % 3 == 1), pad=(i % 4) * 3,
                      host_display=(i % 5 == 0))
                i += 1


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_cross_pane(ref_pane, depth):
    p = T.product()
    i = 0
    for (w, h), planes in itertools.product(((64, 48), (48, 64), (50, 31), (4, 3)), (1, 3, 4)):
        fw, fh = U.face_size(B.PANE_CUBE_CROSS, w, h)
        last = C.full_levels(fw, fh) - 1
        doc = document(w, h, planes, depth, seed=w + h * 3 + planes + depth)
        for level in sorted({-1, 0, last // 2, last}):
            for flags in ((0, ALPHA) if planes == 4 else (0,)):
                check(p, B.PANE_CUBE_CROSS, level, doc, None, flags, device=(i % 3 == 2), pad=(i % 4) * 2, host_display=(i % 5 == 1))
                i += 1


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_layers_pane(ref_pane, depth):
    p = T.product()
    i = 0
    for (w, h), missing in itertools.product(((13, 7), (16, 16), (1, 1), (40, 24)), ((), (5,), (0, 3), (0, 1, 2, 3, 4, 5))):
        last = C.full_levels(w, h) - 1
        doc = document(w, h, 4, depth, seed=w)
        faces = [None if f in missing else layer(w, h, depth, (1, 2, 3, 1, 2, 3)[f], f % 2 == 0, seed=w + h + f + depth)
                 for f in range(6)]
        for level in sorted({-1, 0, last // 2, last}):
            for flags in (0, ALPHA):
                check(p, B.PANE_CUBE_LAYERS, level, doc, faces, flags, device=(i % 3 == 0), pad=(i % 4) * 5, host_display=(i % 5 == 2))
                i += 1


def test_large_panes(ref_pane):
    p = T.product()
    cross = document(1024, 768, 4, 32, seed=13)
    check(p, B.PANE_CUBE_CROSS, 1, cross, None, ALPHA, device=True)
    check(p, B.PANE_CUBE_CROSS, -1, cross, None, 0, device=False, host_display=True)
    doc = document(1024, 1024, 4, 32, seed=11)
    check(p, B.PANE_2D, -1, doc, layer(1024, 1024, 32, 3, True, seed=12), ALPHA, device=True, pad=3)


def test_kernel_time_is_reported(ref_pane):
    p = T.product()
    doc = document(64, 48, 4, 32, seed=1)
    for texture, level, layers in ((B.PANE_2D, -1, layer(64, 48, 32, 3, False, 2)), (B.PANE_CUBE_CROSS, 2, None)):
        run(p, texture, level, doc, layers, 0, host_display=True)
        assert p.last_kernel_ms() >= 0.0


def test_refusals_leave_a_device_display_untouched(ref_pane):
    import torch
    import test_preview_hdr as CPU
    p = T.product()
    p.preview_uncompressed(B.PaneOptions(28, B.PANE_2D, -1), np.zeros((4, 4, 4), np.uint8))          # the context exists
    cases, keep = CPU.pane_refusals()
    for name, o, doc, layers, flags, display, _ in cases:
        if display is None or not display.ptr:
            continue
        disp = torch.full((max(display.height, 1), max(display.width, 1) * 4 + 16), 0xAB, dtype=torch.uint8, device="cuda")
        d = B.RgbaSurface(disp.data_ptr(), display.width, display.height, display.stride)
        before = p.launch_count()
        assert p.preview_uncompressed_hdr_raw(o, doc, layers, flags, d) != 0 and p.last_error() != "", name
        assert p.launch_count() == before, name
        torch.cuda.synchronize()
        assert bool((disp == 0xAB).all()), name


def test_original_pane_does_not_follow_the_slider(ref_pane, ref_view):
    """The finding of DESIGN section 7: the original pane is clamped RGBA8, so exposure 4 brightens the view of the compressed pane
    (float) but leaves texels of the original pane that were clamped at 255 or 0 where they were."""
    p = T.product()
    doc = HC.family_planes("exposure_ramp", 48, 64)
    original = p.preview_uncompressed_hdr(B.PaneOptions(95, B.PANE_CUBE_CROSS, 0), doc)
    compressed = p.preview_cube(B.CubeOptions(95, B.CUBE_CROSS, 0, 0), doc, None, 0, p.profile("bc6h_veryfast"))[0]
    view = B.View(64, 48, 0, 0, 1.0, 0, 0, 0)
    shown = [p.preview_view_exposed(original, view, e) for e in (1.0, 4.0)]
    assert np.array_equal(shown[0], shown[1])                          # depth 8: the exposure does nothing
    shown = [p.preview_view_exposed(compressed, view, e) for e in (1.0, 4.0)]
    assert (shown[1].astype(int) >= shown[0]).all() and (shown[1] > shown[0]).any()
