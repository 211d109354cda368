"""The cube types' placement pinned to the reference's own bodies: ConvertToCubeMapFromCross, ConvertToCubeMapFromLayers,
ConvertToHorizontalCrossFromCubeMap, IsCubeMapWithSetMipLevelOverride and DirectX::CopyRectangle, cut from the reference and compiled
behind a shim by oracle/build_ref_cube.py (oracle/_ref/libitw_ref_cube.so), against the restatement in tests/cube_lib.py that the GPU
tests of tests/test_cube_maps.py compare the library with.  CPU only."""
import ctypes
import itertools
import os
import sys

import numpy as np
import pytest

import cube_lib as C
import itw_testlib as T
import preview_lib as PL

B = T.binding
COLOR, COLOR_ALPHA, CUBEMAP_LAYERS, CUBEMAP_CROSSED, NORMALMAP = range(5)          # IntelPlugin.h:98-106


@pytest.fixture(scope="module")
def ref():
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_cube
        try:
            path = build_ref_cube.build(verbose=False)
        except FileNotFoundError:
            pytest.skip("reference cube functions not built (no reference tree and no prebuilt oracle/_ref)")
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    for n in ("ref_cube_set_level_override", "ref_cube_from_cross", "ref_cube_from_layers", "ref_cross_from_cube"):
        getattr(lib, n).restype = ctypes.c_int
    return lib


def ref_cross(lib, fmt, scratch, doc_format):
    h, w = scratch.shape[:2]
    fw, fh = ctypes.c_int(0), ctypes.c_int(0)
    scratch = np.ascontiguousarray(scratch)
    assert lib.ref_cube_from_cross(fmt, doc_format, w, h, scratch.ctypes.data_as(ctypes.c_void_p), None, ctypes.byref(fw), ctypes.byref(fh)) == 0
    out = np.zeros((6, fh.value, fw.value, 4), scratch.dtype)
    lib.ref_cube_from_cross(fmt, doc_format, w, h, scratch.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p),
                            ctypes.byref(fw), ctypes.byref(fh))
    return list(out)


def test_set_level_override_truth_table(ref):
    for set_level, ttype in itertools.product((0, 1), range(5)):
        assert ref.ref_cube_set_level_override(set_level, ttype) == int(bool(set_level) and ttype in (CUBEMAP_LAYERS, CUBEMAP_CROSSED))


@pytest.mark.parametrize("fmt,depth", list(itertools.product((71, 99, 95), (8, 16, 32))))
def test_cross_cut_equals_restatement(ref, fmt, depth):
    """Both orientations, faces that are not multiples of 4 or powers of two, with and without alpha, and the linearising copy of an
    _SRGB save with mip maps: the reference's ConvertToCubeMapFromCross + CopyRectangle on the front end's scratch."""
    o = T.oracle()
    for (dw, dh), planes, flags in itertools.product(((64, 48), (48, 64), (50, 31), (31, 50), (4, 3), (3, 4)), (3, 4), (0, 1, 2)):
        if (flags & 1) and planes < 4:
            continue
        doc = PL.document(dw, dh, planes, depth, seed=dw * 3 + depth + planes + flags)
        scratch = o.convert_pixels(PL.NAME[fmt], np.ascontiguousarray(doc), flags, pad=False)
        for linear in ((False, True) if fmt != 95 else (False,)):
            doc_format = 10 if fmt == 95 else (29 if linear else 28)          # CopyDataForEncoding's scratch (IntelPlugin.cpp:152-154)
            got = ref_cross(ref, fmt, scratch, doc_format)
            want = C.oracle_cross_faces(fmt, doc, flags, linear)
            for f in range(6):
                assert np.array_equal(got[f], want[f]), (dw, dh, planes, flags, linear, f)


def test_linearising_copy_rectangle_of_all_256_bytes(ref):
    """CopyRectangle from R8G8B8A8_UNORM_SRGB into R8G8B8A8_UNORM: every byte in r, g and b, alpha untouched."""
    v = np.arange(256, dtype=np.uint8)
    scratch = np.zeros((3, 4 * 256, 4), np.uint8)
    scratch[1, :, 0] = np.tile(v, 4)
    scratch[1, :, 1] = np.tile(v[::-1], 4)
    scratch[1, :, 2] = np.tile(np.roll(v, 77), 4)
    scratch[1, :, 3] = np.tile(np.roll(v, 5), 4)
    got = ref_cross(ref, 99, scratch, 29)
    lin = C.srgb_in_bytes()
    for f in (0, 1, 4, 5):
        px = got[f][0]
        assert np.array_equal(px[:, 0], lin[v]) and np.array_equal(px[:, 1], lin[v[::-1]]) and np.array_equal(px[:, 2], lin[np.roll(v, 77)])
        assert np.array_equal(px[:, 3], np.roll(v, 5))
    same = ref_cross(ref, 98, scratch, 28)                                      # UNORM -> UNORM: a plain copy
    assert np.array_equal(same[0][0], scratch[1, 512:768])


def ref_layers(lib, fmt, depth, w, h, named, has_alpha):
    """`named` = [(name, channels, alpha)] in layer order."""
    n = len(named)
    names = (ctypes.c_char_p * n)(*[nm.encode() for nm, _, _ in named])
    planes = (ctypes.c_void_p * (4 * n))()
    keep = []
    for i, (_, channels, alpha) in enumerate(named):
        for c, p in enumerate(channels):
            p = np.ascontiguousarray(p)
            keep.append(p)
            planes[4 * i + c] = p.ctypes.data
        if alpha is not None:
            a = np.ascontiguousarray(alpha)
            keep.append(a)
            planes[4 * i + 3] = a.ctypes.data
    counts = (ctypes.c_int * n)(*[len(c) for _, c, _ in named])
    out = np.zeros((6, h, w, 4), np.uint16 if fmt == 95 else np.uint8)
    ok = lib.ref_cube_from_layers(fmt, depth, w, h, names, planes, counts, n, int(has_alpha), out.ctypes.data_as(ctypes.c_void_p))
    return ok, list(out)


FACE_NAMES = ("+X", "-X", "+Y", "-Y", "+Z", "-Z")


@pytest.mark.parametrize("fmt,depth", list(itertools.product((77, 99, 95), (8, 16, 32))))
def test_layers_cut_equals_restatement(ref, fmt, depth):
    """Missing faces, one-channel layers, alpha planes and none (the 16-bit white of 15360), layers of other names, and the last layer
    of a name winning, as the plug-in walks the list."""
    import test_cube_maps as CM
    w, h = 13, 7
    for k, has_alpha in itertools.product(range(3), (0, 1)):
        faces = CM.face_layers(fmt, w, h, depth, seed=fmt + depth + 10 * k + has_alpha, missing=((4,), (1, 5), ())[k])
        decoy = CM.face_layers(fmt, w, h, depth, seed=99 + k, missing=())
        named = [("Background", [np.zeros((h, w), decoy[2][0][0].dtype)], None)]        # a layer of no face name is ignored
        for i in (3, 0):                                                 # overwritten by the later layers of the same name
            named.append((FACE_NAMES[i], decoy[i][0], decoy[i][1]))
        for i, face in enumerate(faces):
            if face is not None:
                named.append((FACE_NAMES[i], face[0], face[1]))
        named.append(("+x", decoy[2][0], None))                          # names are matched exactly
        for i in (3, 0):                                                 # without a later layer of its name, the earlier one stays
            if faces[i] is None:
                faces[i] = decoy[i]
        ok, got = ref_layers(ref, fmt, depth, w, h, named, has_alpha)
        assert ok == 1
        want = C.oracle_layer_faces(fmt, w, h, depth, faces, has_alpha)
        for f in range(6):
            assert np.array_equal(got[f], want[f]), (k, has_alpha, f)


def test_fewer_than_six_layers_is_refused(ref):
    ok, _ = ref_layers(ref, 98, 8, 4, 4, [(n, [np.zeros((4, 4), np.uint8)], None) for n in FACE_NAMES[:5]], 0)
    assert ok == 0


@pytest.mark.parametrize("fmt", (98, 95))
def test_level_cross_cut_equals_restatement(ref, fmt):
    """ConvertToHorizontalCrossFromCubeMap with and without a set level, for both cube types: faces that are powers of two (box) and
    faces that are not (linear filter), every level of the chain."""
    rng = np.random.default_rng(fmt)
    for (w, h) in ((16, 16), (13, 7), (12, 10), (1, 5)):
        if fmt == 95:
            faces = rng.integers(0, 0x5C00, (6, h, w, 4), dtype=np.uint16)
        else:
            faces = rng.integers(0, 256, (6, h, w, 4), dtype=np.uint8)
        faces = np.ascontiguousarray(faces)
        for ttype, set_level, L in [(CUBEMAP_LAYERS, 0, 0), (COLOR, 1, 0)] + [(t, 1, l) for t in (CUBEMAP_LAYERS, CUBEMAP_CROSSED)
                                                                              for l in range(C.full_levels(w, h))]:
            cw, ch = ctypes.c_int(0), ctypes.c_int(0)
            errors = ref.ref_cross_from_cube(fmt, ttype, set_level, L, w, h, faces.ctypes.data_as(ctypes.c_void_p), None, ctypes.byref(cw), ctypes.byref(ch))
            assert errors == 0
            got = np.zeros((ch.value, cw.value, 4), faces.dtype)
            ref.ref_cross_from_cube(fmt, ttype, set_level, L, w, h, faces.ctypes.data_as(ctypes.c_void_p), got.ctypes.data_as(ctypes.c_void_p),
                                    ctypes.byref(cw), ctypes.byref(ch))
            shown = L if ref.ref_cube_set_level_override(set_level, ttype) else 0
            want = C.oracle_level_cross(fmt, list(faces), shown)
            assert got.shape == want.shape and np.array_equal(got, want), (w, h, ttype, set_level, L)
