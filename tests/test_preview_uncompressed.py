"""The uncompressed pane (include/itw_bcn.h section 11, itw_preview_uncompressed) on the CPU: every refusal happens before any CUDA
call, launches nothing and leaves the display untouched; and the oracle of tests/preview_uncompressed_lib.py keeps the plug-in's own
invariants -- the pane depends on the encoding only through its front end, a cross without a set level is the 2-D pane, and the
cube crosses equal the restatement that tests/test_cube_vs_reference.py pins to the reference (tests/cube_lib.py).
tests/test_preview_uncompressed_gpu.py holds the library to the oracle on the GPU."""
import itertools

import numpy as np
import pytest

import cube_lib as C
import itw_testlib as T
import preview_uncompressed_lib as U

B = T.binding
ALPHA = B.FRONT_HAS_ALPHA


def refusal_cases():
    """(description, options, document, layers, flags, display) that itw_preview_uncompressed must refuse.  The display is a
    sentinel-filled host buffer of the pane's size unless the case is about the display."""
    keep = []
    doc = np.full((12, 16, 4), 0xAB, np.uint8)
    keep.append(doc)
    disp = np.full((12, 16, 4), 0xAB, np.uint8)
    cross_disp = np.full((3, 4, 4), 0xAB, np.uint8)                   # the 16 x 12 cross of 4 x 4 faces at L = 2

    def src(**kw):
        s = B.PixelSource(doc.ctypes.data, 16, 12, 4, 8, 0)
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def surf(a=disp, **kw):
        keep.append(a)
        s = B.RgbaSurface(a.ctypes.data, a.shape[1], a.shape[0], a.strides[0])
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def layer(channels=3, null=None, row_bytes=0, dtype=np.uint8, w=16, h=12):
        arr = (B.LayerSource * 6)()
        planes = [np.zeros((h, w), dtype) for _ in range(3)]
        keep.extend(planes)
        arr[0].channel_count = channels
        for c in range(min(channels, 3)):
            arr[0].channels[c] = None if c == null else planes[c].ctypes.data
        arr[0].row_bytes = row_bytes
        return arr

    def faces(bad=None, **kw):
        arr = (B.LayerSource * 6)()
        p = np.zeros((12, 16), np.uint8)
        keep.append(p)
        for i in range(6):
            if i == 5:
                continue                                               # a face without a layer of that name
            arr[i].channel_count = 1
            arr[i].channels[0] = p.ctypes.data
            if i == bad:
                for k, v in kw.items():
                    setattr(arr[i], k, v)
        return arr

    O = B.PaneOptions
    D2, CR, LY = B.PANE_2D, B.PANE_CUBE_CROSS, B.PANE_CUBE_LAYERS
    cases = [
        ("null options", None, src(), None, 0, surf()),
        ("null document", O(28, D2, -1), None, None, 0, surf()),
        ("null display", O(28, D2, -1), src(), None, 0, None),
        ("null display ptr", O(28, D2, -1), src(), None, 0, surf(ptr=None)),
        ("BC6H_UF16 needs WIC", O(95, D2, -1), src(), None, 0, surf()),
        ("BC6H_SF16", O(96, D2, -1), src(), None, 0, surf()),
        ("format 0", O(0, D2, -1), src(), None, 0, surf()),
        ("format 29", O(29, D2, -1), src(), None, 0, surf()),
        ("format 2", O(2, D2, -1), src(), None, 0, surf()),
        ("format 74", O(74, D2, -1), src(), None, 0, surf()),
        ("format 1000", O(1000, D2, -1), src(), None, 0, surf()),
        ("BC4 cross", O(80, CR, -1), src(), None, 0, surf()),
        ("BC5 layers", O(83, LY, -1), src(), faces(), 0, surf()),
        ("texture 3", O(28, 3, -1), src(), None, 0, surf()),
        ("texture -1", O(28, -1, -1), src(), None, 0, surf()),
        ("gamma", O(28, D2, -1), src(), None, B.FRONT_GAMMA, surf()),
        ("normalise", O(71, D2, -1), src(), None, B.FRONT_NORMALIZE, surf()),
        ("unknown flag", O(71, D2, -1), src(), None, 32, surf()),
        ("high flag", O(71, D2, -1), src(), None, 1 << 31, surf()),
        ("flip on a cross", O(71, CR, 2), src(), None, B.FRONT_FLIP_X, surf(cross_disp)),
        ("flip on layers", O(71, LY, -1), src(), faces(), B.FRONT_FLIP_Y, surf()),
        ("level on 2-D", O(28, D2, 0), src(), None, 0, surf()),
        ("level -2 on 2-D", O(28, D2, -2), src(), None, 0, surf()),
        ("level -2 on a cross", O(71, CR, -2), src(), None, 0, surf()),
        ("level past the chain", O(71, CR, 3), src(), None, 0, surf(cross_disp)),      # 4 x 4 faces: levels 0..2
        ("depth 24", O(28, D2, -1), src(depth=24), None, 0, surf()),
        ("planes 0", O(28, D2, -1), src(planes=0), None, 0, surf()),
        ("planes 5", O(28, D2, -1), src(planes=5), None, 0, surf()),
        ("short row_bytes", O(28, D2, -1), src(row_bytes=63), None, 0, surf()),
        ("width 0", O(28, D2, -1), src(width=0), None, 0, surf()),
        ("height -1", O(28, D2, -1), src(height=-1), None, 0, surf()),
        ("null data", O(28, D2, -1), src(data=None), None, 0, surf()),
        ("alpha without a fourth plane", O(28, D2, -1), src(planes=3, row_bytes=48), None, ALPHA, surf()),
        ("cross of null data", O(71, CR, 1), src(data=None), None, 0, surf()),
        ("cross smaller than a texel per face", O(71, CR, -1), src(width=3, height=3), None, 0, surf()),
        ("layer 0 channel_count 0", O(28, D2, -1), src(), layer(channels=0), 0, surf()),
        ("layer 0 channel_count 4", O(28, D2, -1), src(), layer(channels=4), 0, surf()),
        ("layer 0 null channel", O(28, D2, -1), src(), layer(null=1), 0, surf()),
        ("layer 0 short rows", O(28, D2, -1), src(), layer(row_bytes=15), 0, surf()),
        ("layer 0 of depth 24", O(28, D2, -1), src(depth=24), layer(), 0, surf()),
        ("null face list", O(71, LY, -1), src(), None, 0, surf(np.full((36, 64, 4), 0xAB, np.uint8))),
        ("face channel_count 4", O(71, LY, -1), src(), faces(bad=2, channel_count=4), 0, surf(np.full((36, 64, 4), 0xAB, np.uint8))),
        ("face short rows", O(71, LY, -1), src(), faces(bad=0, row_bytes=8), 0, surf(np.full((36, 64, 4), 0xAB, np.uint8))),
        ("faces of depth 24", O(71, LY, -1), src(depth=24), faces(), 0, surf(np.full((36, 64, 4), 0xAB, np.uint8))),
        ("2-D display too wide", O(28, D2, -1), src(), None, 0, surf(width=17)),
        ("2-D display too short", O(28, D2, -1), src(), None, 0, surf(height=11)),
        ("2-D display stride", O(28, D2, -1), src(), None, 0, surf(stride=63)),
        ("2-D display stride -4", O(28, D2, -1), src(), None, 0, surf(stride=-4)),
        ("cross without L: document-sized display", O(71, CR, -1), src(), None, 0, surf(cross_disp)),
        ("cross with L: cross-sized display", O(71, CR, 2), src(), None, 0, surf()),
        ("cross display stride", O(71, CR, 2), src(), None, 0, surf(cross_disp, stride=15)),
        ("layers: document-sized display", O(71, LY, -1), src(), faces(), 0, surf()),
        ("oversized cross", O(28, LY, -1), src(data=None, width=(1 << 28) + 1, height=1), (B.LayerSource * 6)(), 0, surf()),
    ]
    return cases, keep


def test_refusals_before_any_cuda_call():
    p = T.product()
    cases, keep = refusal_cases()
    for name, o, doc, layers, flags, display in cases:
        before = p.launch_count()
        size = B.ctypes.c_size_t(12345)
        rc = p.preview_uncompressed_raw(o, doc, layers, flags, display, B.ctypes.byref(size))
        err = p.last_error()
        assert rc != 0 and err != "", name
        assert p.launch_count() == before, name
        assert size.value == 12345, name
        if name.startswith("BC6H_UF16"):
            assert "WIC" in err, err
    for a in keep:                                                    # every display of the list still holds the sentinel
        if a.dtype == np.uint8 and a.ndim == 3:
            assert (a == 0xAB).all()


def test_error_text_names_the_call():
    p = T.product()
    doc = np.zeros((4, 4, 4), np.uint8)
    disp = np.zeros((4, 4, 4), np.uint8)
    src = B.PixelSource(doc.ctypes.data, 4, 4, 4, 8, 0)
    rc = p.preview_uncompressed_raw(B.PaneOptions(95, B.PANE_2D, -1), src, None, 0, B.RgbaSurface(disp.ctypes.data, 4, 4, 16), None)
    assert rc != 0 and p.last_error().startswith("itw_preview_uncompressed:") and "WIC" in p.last_error()
    rc = p.preview_uncompressed_raw(B.PaneOptions(80, B.PANE_CUBE_CROSS, -1), src, None, 0, B.RgbaSurface(disp.ctypes.data, 4, 4, 16), None)
    assert rc != 0 and "BC4 and BC5" in p.last_error()


# ---- the oracle's invariants ----
@pytest.fixture(scope="module")
def ref():
    if not U.available():
        pytest.skip("reference cuts not built (no reference tree and no prebuilt oracle/_ref)")


COLOUR = (71, 72, 77, 78, 98, 99)


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_pane_depends_on_the_encoding_only_through_its_front_end(ref, depth):
    for (w, h), planes in itertools.product(((1, 1), (5, 3), (19, 13)), (1, 2, 3, 4)):
        doc = U.document(w, h, planes, depth, seed=w + planes + depth)
        for flags, layer0 in itertools.product((0, ALPHA, B.FRONT_FLIP_X, B.FRONT_FLIP_Y | ALPHA, B.FRONT_FLIP_X | B.FRONT_FLIP_Y),
                                               (None, U.layer(w, h, depth, 2, True, seed=depth), U.layer(w, h, depth, 1, False, seed=3))):
            if (flags & ALPHA) and planes < 4:
                continue
            want, size = U.oracle_pane(28, B.PANE_2D, -1, doc, layer0, flags)
            assert size == w * h * 4 and want.shape == (h, w, 4)
            for fmt in COLOUR:
                got, n = U.oracle_pane(fmt, B.PANE_2D, -1, doc, layer0, flags)
                assert n == 0 and np.array_equal(got, want), (fmt, w, h, planes, flags, layer0 is not None)
            bc4 = U.oracle_pane(80, B.PANE_2D, -1, doc, layer0, flags)[0]
            assert np.array_equal(bc4, U.oracle_pane(83, B.PANE_2D, -1, doc, layer0, flags)[0])
            if layer0 is None and not (flags & (B.FRONT_FLIP_X | B.FRONT_FLIP_Y)):
                # ConvertToBC4or5From* copies plane 0 where ConvertToBCFrom* writes 0 (IntelPlugin.cpp:412-427, :795-806)
                for c in range(4):
                    if c < planes or c == 3:
                        assert np.array_equal(bc4[..., c], want[..., c]), (c, planes)
                    else:
                        assert np.array_equal(bc4[..., c], bc4[..., 0]) and not want[..., c].any(), (c, planes)


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_cross_without_a_level_is_the_2d_pane(ref, depth):
    for (w, h), planes in itertools.product(((64, 48), (48, 64), (50, 31), (4, 3)), (3, 4)):
        doc = U.document(w, h, planes, depth, seed=w * h + depth)
        for flags in ((0, ALPHA) if planes == 4 else (0,)):
            for fmt in U.CUBE_ENCODINGS:
                got, n = U.oracle_pane(fmt, B.PANE_CUBE_CROSS, -1, doc, None, flags)
                assert np.array_equal(got, U.oracle_pane(fmt, B.PANE_2D, -1, doc, None, flags)[0]), (fmt, w, h, flags)
                assert n == (w * h * 4 if fmt == 28 else 0)


@pytest.mark.parametrize("depth", (8, 16, 32))
def test_cube_crosses_equal_the_cube_restatement(ref, depth):
    """The crosses of the reference cuts equal cube_lib's oracle_level_cross of cube_lib's preview faces, at every level, for both
    orientations, ragged faces, faces of one texel, missing faces and 1-3-channel face layers with and without alpha."""
    for (w, h), planes, flags in itertools.product(((64, 48), (48, 64), (50, 31), (31, 50), (4, 3)), (3, 4), (0, ALPHA)):
        if (flags & ALPHA) and planes < 4:
            continue
        doc = U.document(w, h, planes, depth, seed=w + h + planes + depth)
        fw, fh = U.face_size(B.PANE_CUBE_CROSS, w, h)
        faces = C.oracle_faces(B.CubeOptions(71, B.CUBE_CROSS, 0, 0), doc, None, flags, preview=True)
        for L in range(-1, C.full_levels(fw, fh)):
            if L < 0:
                continue
            got = U.oracle_pane(28, B.PANE_CUBE_CROSS, L, doc, None, flags)[0]
            assert np.array_equal(got, C.oracle_level_cross(71, faces, L)), (w, h, planes, flags, L)
    for (w, h), missing, flags in itertools.product(((13, 7), (16, 16), (1, 1), (5, 3)), ((), (5,), (0, 3)), (0, ALPHA)):
        doc = U.document(w, h, 4, depth, seed=1)
        layers = U.cube_layers(w, h, depth, seed=w + depth, missing=missing)
        faces = C.oracle_faces(B.CubeOptions(71, B.CUBE_LAYERS, 0, 0), doc, layers, flags, preview=True)
        for L in range(-1, C.full_levels(w, h)):
            got = U.oracle_pane(71, B.PANE_CUBE_LAYERS, L, doc, layers, flags)[0]
            assert np.array_equal(got, C.oracle_level_cross(71, faces, max(L, 0))), (w, h, missing, flags, L)
