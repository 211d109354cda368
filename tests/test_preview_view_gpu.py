"""itw_preview_view on the GPU (include/itw_bcn.h section 11): the matrix of tests/test_preview_view.py against the reference's own
FetchPreviewRGB loops (oracle/build_ref_view.py), with host and device sources and destinations; a pane straight from
itw_preview_pixels' device display; rejections that launch nothing and leave dst untouched."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import test_preview_view as V

B = T.binding


def device_copy(buf):
    import torch
    return torch.from_numpy(buf).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", V.KINDS, ids=lambda k: f"fmt{k[0]}-p{k[1]}")
def test_gpu_view_matches_reference(kind):
    if V.ref_view() is None:
        pytest.skip("reference view not built")
    import torch
    p = T.product()
    fmt, planes, depth = kind
    pitch = V.row_pitch(kind)
    buf = V.with_pitch(V.source(kind, seed=fmt * 10 + planes), pitch)
    dev = device_copy(buf)
    out = np.zeros((V.VIEW_H, V.VIEW_W, 3), np.uint8)
    d_out = torch.zeros((V.VIEW_H, V.VIEW_W, 3), dtype=torch.uint8, device="cuda")
    for mask in V.MASKS:
        for i, (x, y, zoom, mip, matte) in enumerate(V.views()):
            want = V.ref_fetch(kind, buf, pitch, V.VIEW_W, V.VIEW_H, x, y, zoom, mip, mask, matte)
            view = B.View(V.VIEW_W, V.VIEW_H, x, y, zoom, mip, mask, matte)
            host = (i + mask) % 2 == 0                          # alternate host and device operands over the matrix
            src = B.PixelSource(buf.ctypes.data if host else dev.data_ptr(), V.SRC_W, V.SRC_H, planes, depth, pitch)
            if (i // 2 + mask) % 2 == 0:
                assert p.preview_view_raw(src, view, out.ctypes.data) == 0, p.last_error()
                got = out
            else:
                assert p.preview_view_raw(src, view, d_out.data_ptr()) == 0, p.last_error()
                got = d_out.cpu().numpy()
            assert np.array_equal(got, want), (mask, x, y, zoom, mip, matte, host)


@pytest.mark.gpu
def test_gpu_view_of_a_device_pane_from_preview_pixels():
    """The dialog's flow: the pane stays in device memory (itw_preview_pixels into a device display), every repaint is one
    itw_preview_view of it; the bytes equal the reference loop over the same pane copied to the host, for both pane formats."""
    if V.ref_view() is None:
        pytest.skip("reference view not built")
    import torch
    import preview_lib as PL
    p = T.product()
    for fmt, depth, prof, target in ((98, 8, "basic", 28), (95, 32, "bc6h_basic", 2)):
        doc = PL.document(200, 120, 4, depth, seed=depth)
        texel = 16 if target == 2 else 4
        disp = torch.zeros((120, 200 * texel), dtype=torch.uint8, device="cuda")
        src = (B.PixelSource * 1)(B.PixelSource(doc.ctypes.data, 200, 120, 4, depth, 0))
        settings = p.profile(prof)
        p.preview_pixels_raw(fmt, src, 1, B.FRONT_HAS_ALPHA, settings, disp.data_ptr(), 200, 120, 200 * texel)
        pane = disp.cpu().numpy()
        for mask in (0, B.VIEW_RED, B.VIEW_GREEN, B.VIEW_BLUE, B.VIEW_ALPHA):
            view = B.View(150, 90, -10, 20, float(np.float32(1) / np.float32(0.7)), 0, mask, 0x404040)
            out = torch.zeros((90, 150, 3), dtype=torch.uint8, device="cuda")
            ps = B.PixelSource(disp.data_ptr(), 200, 120, 4, 32 if target == 2 else 8, 200 * texel)
            assert p.preview_view_raw(ps, view, out.data_ptr()) == 0, p.last_error()
            want = np.zeros((90, 150, 3), np.uint8)
            V.ref_view().ref_fetch_preview_rgb(want.ctypes.data, 150, 90, -10, 20, view.zoom, mask, 0x404040, pane.ctypes.data, 200, 120, 4,
                                               target, 200 * texel, 0)
            assert np.array_equal(out.cpu().numpy(), want), (fmt, mask)


@pytest.mark.gpu
def test_gpu_rejections_launch_nothing():
    import torch
    p = T.product()
    a = np.zeros((8, 8, 4), np.uint8)
    p.preview_view(a, B.View(6, 5, 0, 0, 1.0, 0, 0, 0))          # warm: the context exists
    d_dst = torch.full((5, 6, 3), 0xAB, dtype=torch.uint8, device="cuda")
    for name, s, v, dst, keep in V.reject_cases(p):
        for target in ("host", "device"):
            before = p.launch_count()
            ptr = (dst.ctypes.data if target == "host" else d_dst.data_ptr()) if dst is not None else 0
            assert p.preview_view_raw(s, v, ptr) != 0 and p.last_error() != "", name
            assert p.launch_count() == before, name
            if dst is not None:
                assert (dst == 0xAB).all() and bool((d_dst == 0xAB).all()), name
