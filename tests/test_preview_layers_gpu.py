"""itw_preview_layers on the GPU (include/itw_bcn.h section 11): the compressed pane of "mip maps from layers" against the oracle
composed from the reference's own bodies (tests/preview_layers_lib.py: oracle_preview_layers), for every format the dialog offers, the
_SRGB forms, depths 8 / 16 / 32, 1-3 layer channels, with and without alpha, and the normal-map flip / normalise flags;
compressed_bytes; agreement with itw_preview_pixels when layer 0 holds the composite; device operands; rejections."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import preview_layers_lib as PLL
import preview_lib as PL

B = T.binding
PROFILE = {71: None, 72: None, 77: None, 78: None, 80: None, 83: None, 95: "bc6h_veryfast", 98: "veryfast", 99: "veryfast"}


def layer_planes(depth, w, h, channels, alpha, seed, specials=True):
    rng = np.random.default_rng(seed)
    planes = [PL.document(w, h, 1, depth, seed + c)[..., 0] for c in range(channels)]
    if depth == 32 and specials:                                # a few specials where the RGBA8 converters branch
        planes[0].reshape(-1)[:6] = [np.nan, np.inf, -1.0, 2.0, 1e-40, 0.5]
    a = PL.document(w, h, 1, depth, seed + 9)[..., 0] if alpha else None
    if a is not None:
        rng.shuffle(a.reshape(-1))
    return [np.ascontiguousarray(c) for c in planes], a


def skip_without_reference():
    if PL.ref() is None or PLL.ref_layers() is None or T.ref_frontend() is None:
        pytest.skip("reference cuts not built")


CASES = [  # fmt, depth, channels, alpha plane, flags, w, h
    (71, 8, 3, False, 0, 50, 27), (72, 8, 2, True, 1, 64, 32), (77, 16, 3, False, 1, 50, 27), (78, 16, 1, True, 1, 33, 20),
    (80, 8, 1, False, 0, 50, 27), (83, 16, 2, False, 4 | 8 | 16, 64, 32), (83, 8, 3, False, 4 | 16, 50, 27),
    (95, 8, 3, True, 1, 32, 16), (95, 16, 2, False, 0, 50, 27), (95, 32, 3, True, 1 | 8 | 16, 50, 27),
    (98, 32, 1, True, 1 | 2, 50, 27), (98, 8, 3, True, 1 | 4 | 8, 64, 32), (99, 8, 3, False, 4 | 8, 64, 32),
    (99, 32, 2, False, 2 | 16, 33, 20), (72, 32, 3, True, 1 | 2 | 4, 50, 27), (77, 32, 3, False, 0, 64, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,depth,channels,alpha,flags,w,h", CASES)
def test_gpu_layers_pane_matches_oracle(fmt, depth, channels, alpha, flags, w, h):
    skip_without_reference()
    p = T.product()
    planes = 4 if (flags & B.FRONT_HAS_ALPHA) else 3
    composite = PL.document(w, h, planes, depth, seed=w + depth + fmt)
    layer0 = layer_planes(depth, w, h, channels, alpha, seed=fmt + channels, specials=fmt != 95)
    if depth == 32 and fmt == 95:                               # HDR values the BC6H encoders take: non-negative
        composite = np.clip(composite, 0, 4).astype(np.float32)
        layer0 = ([np.clip(c, 0, 4).astype(np.float32) for c in layer0[0]], None if layer0[1] is None else np.clip(layer0[1], 0, 4).astype(np.float32))
    prof = PROFILE[fmt]
    got, n = p.preview_layers(fmt, composite, layer0, flags, p.profile(prof) if prof else None)
    want, n_want = PLL.oracle_preview_layers(fmt, composite, layer0, flags, prof)
    assert np.array_equal(got, want, equal_nan=True)
    assert n == n_want == PL.nblocks(w, h) * PL.bpb(fmt)         # the slice pitch of level 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,depth,flags", [(98, 8, 1), (77, 16, 1 | 4 | 16), (71, 32, 1 | 2), (95, 16, 1 | 8), (83, 8, 1 | 4 | 8 | 16)])
def test_gpu_layer_holding_the_composite_gives_preview_pixels(fmt, depth, flags):
    """Layer 0 = the composite's planes and alpha: the pane is itw_preview_pixels' pane of the composite (flip and normalise
    after the copy equal the front end's; 32-bit layers into RGBA8 always take the gamma step, so the composite's flags include it)."""
    p = T.product()
    w, h = 50, 27
    composite = PL.document(w, h, 4, depth, seed=fmt + depth)
    layer0 = ([np.ascontiguousarray(composite[..., c]) for c in range(3)], np.ascontiguousarray(composite[..., 3]))
    prof = PROFILE[fmt]
    s = p.profile(prof) if prof else None
    got, n = p.preview_layers(fmt, composite, layer0, flags, s)
    want, m = p.preview_pixels(fmt, [composite], flags, s)
    assert np.array_equal(got, want) and n == m


@pytest.mark.gpu
def test_gpu_device_operands_and_wide_rows():
    import torch
    p = T.product()
    w, h, depth, fmt = 50, 27, 16, 77
    composite = PL.document(w, h, 4, depth, seed=3)
    channels, alpha = layer_planes(depth, w, h, 3, True, seed=4)
    want, n = p.preview_layers(fmt, composite, (channels, alpha), B.FRONT_HAS_ALPHA | B.FRONT_FLIP_X)
    pitch = 64                                                   # elements per row: wider than the document
    keep = []

    def wide(a):
        buf = np.zeros((h, pitch), a.dtype)
        buf[:, :w] = a
        t = torch.from_numpy(buf.view(np.int16)).cuda()
        keep.append(t)
        return t.data_ptr()
    arr = (B.LayerSource * 1)()
    arr[0].channel_count = 3
    for c in range(3):
        arr[0].channels[c] = wide(channels[c])
    arr[0].alpha = wide(alpha)
    arr[0].row_bytes = pitch * 2
    d_comp = torch.from_numpy(composite.view(np.int16)).cuda()
    src = B.PixelSource(d_comp.data_ptr(), w, h, 4, depth, 0)
    disp = torch.zeros((h, w * 4 + 16), dtype=torch.uint8, device="cuda")
    size = ctypes.c_size_t(0)
    rc = p.preview_layers_raw(fmt, src, arr, B.FRONT_HAS_ALPHA | B.FRONT_FLIP_X, None, B.RgbaSurface(disp.data_ptr(), w, h, w * 4 + 16),
                              ctypes.byref(size))
    assert rc == 0, p.last_error()
    assert np.array_equal(disp.cpu().numpy()[:, :w * 4].reshape(h, w, 4), want) and size.value == n


@pytest.mark.gpu
def test_gpu_rejections_enqueue_nothing():
    p = T.product()
    w, h = 32, 16
    composite = PL.document(w, h, 4, 8, seed=1)
    channels, alpha = layer_planes(8, w, h, 3, True, seed=2)
    p.preview_layers(71, composite, (channels, alpha), 1)       # warm: the context exists
    keep = [composite]

    def layer(count=3, row_bytes=0, null=None):
        arr = (B.LayerSource * 1)()
        arr[0].channel_count = count
        for c in range(3):
            arr[0].channels[c] = None if c == null else channels[c].ctypes.data
        arr[0].alpha = alpha.ctypes.data
        arr[0].row_bytes = row_bytes
        return arr

    def call(fmt=71, source=B.PixelSource(composite.ctypes.data, w, h, 4, 8, 0), arr=None, flags=1, dw=w, dh=h, stride=w * 4, settings=None):
        arr = layer() if arr is None else arr
        out = np.full((dh, max(dw, 1), 4), 0xAB, np.uint8)
        before = p.launch_count()
        rc = p.preview_layers_raw(fmt, source, arr, flags, settings, B.RgbaSurface(out.ctypes.data, dw, dh, stride), None)
        assert rc != 0 and p.last_error() != ""
        assert (out == 0xAB).all() and p.launch_count() == before
    call(arr=layer(count=0))
    call(arr=layer(count=4))
    call(arr=layer(null=1))
    call(arr=layer(row_bytes=w - 1))                                        # row_bytes smaller than a document row
    call(flags=1 | 64)                                                      # unknown flag bits
    call(source=B.PixelSource(composite.ctypes.data, w, h, 4, 24, 0))      # depth 24
    call(source=B.PixelSource(None, w, h, 4, 8, 0))                         # null composite data
    call(source=B.PixelSource(composite.ctypes.data, w, h, 3, 8, 0))       # HAS_ALPHA without an alpha plane
    call(fmt=70)                                                            # not a format the library encodes
    call(fmt=98)                                                            # BC7 without settings
    call(dw=w + 4)                                                          # display of the wrong size
    call(stride=w * 4 - 4)                                                  # display stride below a row
    out = np.zeros((h, w, 4), np.uint8)
    before = p.launch_count()
    assert p.preview_layers_raw(71, B.PixelSource(composite.ctypes.data, w, h, 4, 8, 0), None, 1, None,
                                B.RgbaSurface(out.ctypes.data, w, h, w * 4), None) != 0           # null layer 0
    assert p.launch_count() == before
