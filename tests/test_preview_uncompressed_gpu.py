"""itw_preview_uncompressed on the GPU (include/itw_bcn.h section 11): every pane equals the oracle of
tests/preview_uncompressed_lib.py byte for byte over the texture types (2-D with and without layer 0, horizontal and vertical crosses,
face layers with missing faces and 1-3-channel faces with and without alpha), depths 8 / 16 / 32, planes 1-4, every accepted encoding,
set levels -1 / 0 / middle / last, the flips, ragged sizes, faces of one texel and one 4096-class document; host and device operands,
a device display filled in place at its own stride, *compressed_bytes, refusals that leave a sentinel display untouched, and the
dialog's view (itw_preview_view) of a device pane against the reference's FetchPreviewRGB loops over the oracle pane."""
import ctypes
import itertools

import numpy as np
import pytest

import cube_lib as C
import itw_testlib as T
import preview_uncompressed_lib as U

B = T.binding
ALPHA = B.FRONT_HAS_ALPHA
FX, FY = B.FRONT_FLIP_X, B.FRONT_FLIP_Y
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    if not U.available():
        pytest.skip("reference cuts not built (no reference tree and no prebuilt oracle/_ref)")


def run(p, fmt, texture, level, doc, layers, flags, device=False, pad=0):
    """The call with host operands, or with device document / layers / display (the display `pad` bytes wider than a row, filled
    with a sentinel that must survive outside the pane).  Returns (pane, compressed bytes)."""
    import torch
    dh, dw = doc.shape[:2]
    w, h = U.pane_size(texture, level, dw, dh)
    if not device:
        return p.preview_uncompressed(B.PaneOptions(fmt, texture, level), doc, layers, flags)
    keep = []

    def dev(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr()
    docp = np.ascontiguousarray(doc)
    src = B.PixelSource(dev(docp), dw, dh, doc.shape[2], doc.itemsize * 8, 0)
    arr = None
    if layers is not None:
        arr = (B.LayerSource * 6)()
        for i, face in enumerate([layers] if texture == B.PANE_2D else layers):
            if face is None:
                continue
            channels, alpha = face
            arr[i].channel_count = len(channels)
            for c, pl in enumerate(channels):
                arr[i].channels[c] = dev(np.ascontiguousarray(pl, doc.dtype))
            arr[i].alpha = None if alpha is None else dev(np.ascontiguousarray(alpha, doc.dtype))
    stride = w * 4 + pad
    disp = torch.full((h, stride), 0xAB, dtype=torch.uint8, device="cuda")
    size = ctypes.c_size_t(0)
    rc = p.preview_uncompressed_raw(B.PaneOptions(fmt, texture, level), src, arr, flags, B.RgbaSurface(disp.data_ptr(), w, h, stride),
                                    ctypes.byref(size))
    assert rc == 0, p.last_error()
    torch.cuda.synchronize()
    out = disp.cpu().numpy()
    assert (out[:, w * 4:] == 0xAB).all()                              # nothing outside the pane's rows
    return out[:, :w * 4].reshape(h, w, 4), size.value


def check(p, fmt, texture, level, doc, layers, flags, device=False, pad=0):
    want, n = U.oracle_pane(fmt, texture, level, doc, layers, flags)
    got, size = run(p, fmt, texture, level, doc, layers, flags, device, pad)
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.argwhere((got != want).any(-1))
    assert bad.size == 0, (fmt, texture, level, doc.shape, doc.dtype, flags, device, bad[:4].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])
    assert size == n == (doc.shape[0] * doc.shape[1] * 4 if fmt == 28 else 0)


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_2d_pane(ref, depth):
    p = T.product()
    i = 0
    for (w, h), planes in itertools.product(((1, 1), (5, 3), (130, 67), (64, 64)), (1, 2, 3, 4)):
        doc = U.document(w, h, planes, depth, seed=w * 7 + planes + depth)
        layer_kinds = (None, U.layer(w, h, depth, 1, False, seed=i), U.layer(w, h, depth, 2, True, seed=i + 1),
                       U.layer(w, h, depth, 3, True, seed=i + 2))
        for fmt in U.ENCODINGS:
            for flags in (0, ALPHA, FX, FY | ALPHA, FX | FY):
                if (flags & ALPHA) and planes < 4:
                    continue
                layer0 = layer_kinds[i % len(layer_kinds)]
                check(p, fmt, B.PANE_2D, -1, doc, layer0, flags, device=(i % 3 == 1), pad=(i % 2) * 12)
                i += 1


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_cross_pane(ref, depth):
    p = T.product()
    i = 0
    for (w, h), planes in itertools.product(((64, 48), (48, 64), (50, 31), (31, 50), (4, 3), (3, 4)), (1, 3, 4)):
        fw, fh = U.face_size(B.PANE_CUBE_CROSS, w, h)
        last = C.full_levels(fw, fh) - 1
        doc = U.document(w, h, planes, depth, seed=w + h * 3 + planes + depth)
        for level in sorted({-1, 0, last // 2, last}):
            for flags in ((0, ALPHA) if planes == 4 else (0,)):
                fmt = U.CUBE_ENCODINGS[i % len(U.CUBE_ENCODINGS)]
                check(p, fmt, B.PANE_CUBE_CROSS, level, doc, None, flags, device=(i % 3 == 2), pad=(i % 2) * 8)
                i += 1


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_layers_pane(ref, depth):
    p = T.product()
    i = 0
    for (w, h), missing in itertools.product(((13, 7), (16, 16), (1, 1), (5, 3), (40, 24)), ((), (5,), (0, 3), (0, 1, 2, 3, 4, 5))):
        last = C.full_levels(w, h) - 1
        doc = U.document(w, h, 4, depth, seed=w)
        layers = U.cube_layers(w, h, depth, seed=w + h + depth + len(missing), missing=missing)
        for level in sorted({-1, 0, last // 2, last}):
            for flags in (0, ALPHA):
                fmt = U.CUBE_ENCODINGS[i % len(U.CUBE_ENCODINGS)]
                check(p, fmt, B.PANE_CUBE_LAYERS, level, doc, layers, flags, device=(i % 3 == 0), pad=(i % 2) * 4)
                i += 1


def test_every_encoding_on_each_texture_type(ref):
    """Every accepted encoding once per texture type, host and device."""
    p = T.product()
    doc = U.document(52, 39, 4, 16, seed=5)
    layers = U.cube_layers(52, 39, 16, seed=6, missing=(2,))
    for device in (False, True):
        for fmt in U.ENCODINGS:
            check(p, fmt, B.PANE_2D, -1, doc, U.layer(52, 39, 16, 2, True, seed=fmt), ALPHA | FY, device)
        for fmt in U.CUBE_ENCODINGS:
            check(p, fmt, B.PANE_CUBE_CROSS, 1, doc, None, ALPHA, device)
            check(p, fmt, B.PANE_CUBE_LAYERS, 2, doc, layers, ALPHA, device)


def test_large_documents(ref):
    p = T.product()
    doc = U.document(4096, 4096, 4, 8, seed=11)
    check(p, 28, B.PANE_2D, -1, doc, U.layer(4096, 4096, 8, 3, True, seed=12), ALPHA | FX, device=True)
    check(p, 98, B.PANE_2D, -1, doc, None, FY, device=False)
    cross = U.document(4096, 3072, 4, 32, seed=13)
    check(p, 28, B.PANE_CUBE_CROSS, 1, cross, None, ALPHA, device=True)
    check(p, 71, B.PANE_CUBE_CROSS, -1, cross, None, 0, device=False)


def test_kernel_time_is_reported(ref):
    p = T.product()
    doc = U.document(256, 192, 4, 8, seed=1)
    for texture, level in ((B.PANE_2D, -1), (B.PANE_CUBE_CROSS, 2)):
        run(p, 28, texture, level, doc, None, 0)
        assert p.last_kernel_ms() >= 0.0


def test_refusals_leave_a_device_display_untouched(ref):
    import torch
    import test_preview_uncompressed as CPU
    p = T.product()
    p.preview_uncompressed(B.PaneOptions(28, B.PANE_2D, -1), np.zeros((4, 4, 4), np.uint8))          # the context exists
    cases, keep = CPU.refusal_cases()
    for name, o, doc, layers, flags, display in cases:
        if display is None or not display.ptr:
            continue
        disp = torch.full((max(display.height, 1), max(display.width, 1) * 4 + 16), 0xAB, dtype=torch.uint8, device="cuda")
        d = B.RgbaSurface(disp.data_ptr(), display.width, display.height, display.stride)
        before = p.launch_count()
        size = ctypes.c_size_t(7)
        assert p.preview_uncompressed_raw(o, doc, layers, flags, d, ctypes.byref(size)) != 0 and p.last_error() != "", name
        assert p.launch_count() == before and size.value == 7, name
        torch.cuda.synchronize()
        assert bool((disp == 0xAB).all()), name


def test_view_of_a_device_pane(ref):
    """The dialog's flow: the pane stays on the device, every repaint is one itw_preview_view of it; the bytes equal the reference's
    FetchPreviewRGB loops over the oracle pane (R8G8B8A8_UNORM, format 28 of the loops)."""
    import torch
    import test_preview_view as V
    if V.ref_view() is None:
        pytest.skip("reference view not built")
    p = T.product()
    doc = U.document(96, 72, 4, 32, seed=21)
    layers = U.cube_layers(24, 18, 32, seed=22, missing=(4,))
    small = U.document(24, 18, 4, 32, seed=23)
    for fmt, texture, level, d, lay, flags in ((28, B.PANE_2D, -1, doc, U.layer(96, 72, 32, 3, True, seed=24), ALPHA | FX),
                                               (98, B.PANE_CUBE_CROSS, 1, doc, None, ALPHA),
                                               (28, B.PANE_CUBE_LAYERS, -1, small, layers, 0),
                                               (71, B.PANE_CUBE_LAYERS, 2, small, layers, ALPHA)):
        want, _ = U.oracle_pane(fmt, texture, level, d, lay, flags)
        h, w = want.shape[:2]
        stride = w * 4 + 32
        disp = torch.zeros((h, stride), dtype=torch.uint8, device="cuda")
        src = B.PixelSource(d.ctypes.data, d.shape[1], d.shape[0], 4, 32, 0)
        arr = None
        keep = []
        if lay is not None:
            arr = p.cube_faces([lay] if texture == B.PANE_2D else lay, d.dtype, keep)
        assert p.preview_uncompressed_raw(B.PaneOptions(fmt, texture, level), src, arr, flags, B.RgbaSurface(disp.data_ptr(), w, h, stride),
                                          None) == 0, p.last_error()
        pane = np.zeros((h, stride), np.uint8)
        pane[:, :w * 4] = want.reshape(h, -1)
        for mask, zoom, x, y, mip in ((0, 1.0, 0, 0, 0), (B.VIEW_RED, float(np.float32(1) / np.float32(1.7)), -5, 3, 0),
                                      (B.VIEW_GREEN | B.VIEW_ALPHA, float(np.float32(1) / np.float32(0.3)), 7, -2, 1),
                                      (B.VIEW_ALPHA, 0.45, 10, 4, 2), (0, float(np.float32(1) / np.float32(3.0)), -20, -9, 0)):
            view = B.View(80, 50, x, y, zoom, mip, mask, 0x203040)
            out = torch.zeros((50, 80, 3), dtype=torch.uint8, device="cuda")
            ps = B.PixelSource(disp.data_ptr(), w, h, 4, 8, stride)
            assert p.preview_view_raw(ps, view, out.data_ptr()) == 0, p.last_error()
            ref_out = np.zeros((50, 80, 3), np.uint8)
            V.ref_view().ref_fetch_preview_rgb(ref_out.ctypes.data, 80, 50, x, y, zoom, mask, 0x203040, pane.ctypes.data, w, h, 4, 28, stride, mip)
            assert np.array_equal(out.cpu().numpy(), ref_out), (fmt, texture, level, mask, zoom, mip)
