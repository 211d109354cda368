"""The oracle of the uncompressed pane (itw_preview_uncompressed, include/itw_bcn.h section 11): the plug-in's
GetUncompressedImageForPreview (IntelPlugin.cpp:1085-1167) for every encoding whose scratch is R8G8B8A8_UNORM, restated as glue over
the reference's own bodies:

  CopyDataForEncoding(DoMipMaps = false, gammaCorrect = false)   the converters of oracle/build_ref_frontend.py (ref_convert)
  ConvertToCubeMapFromCross / FromLayers (:1105-1121)            the cuts of oracle/build_ref_cube.py (ref_cube_from_cross / _layers)
  ConvertToHorizontalCrossFromCubeMap (:1421-1501)               the same file's ref_cross_from_cube (the chain to L included)
  CopyLayersIntoMipMaps(..., 0, 1) (:1128-1134)                  the cut of oracle/build_ref_layers.py
  FlipXYChannelNormalMap (:1137-1140)                            oracle/build_ref_frontend.py

No Convert: the scratch is R16G16B16A16_FLOAT only for BC6H_UF16, which the call refuses."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
from preview_layers_lib import ref_convert, ref_layers

B = T.binding
ENCODINGS = (71, 72, 77, 78, 80, 83, 98, 99, 28)       # the dialog's encodings whose pane needs no WIC
CUBE_ENCODINGS = (71, 72, 77, 78, 98, 99, 28)          # BC4 and BC5 have no cube column (IntelPlugin.cpp:44-62)
FACE_NAMES = ("+X", "-X", "+Y", "-Y", "+Z", "-Z")
CUBEMAP_LAYERS, CUBEMAP_CROSSED = 2, 3                 # IntelPlugin.h:98-106
FLIPS = B.FRONT_FLIP_X | B.FRONT_FLIP_Y


@functools.lru_cache(None)
def ref_cube():
    """oracle/_ref/libitw_ref_cube.so (oracle/build_ref_cube.py); None if unavailable."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_cube
        try:
            path = build_ref_cube.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    for n in ("ref_cube_set_level_override", "ref_cube_from_cross", "ref_cube_from_layers", "ref_cross_from_cube"):
        getattr(lib, n).restype = ctypes.c_int
    return lib


def available():
    return T.ref_frontend() is not None and ref_layers() is not None and ref_cube() is not None


def face_size(texture, dw, dh):
    if texture == B.PANE_CUBE_LAYERS:
        return dw, dh
    return (dw // 3, dh // 4) if dw < dh else (dw // 4, dh // 3)


def pane_size(texture, level, dw, dh):
    if texture == B.PANE_2D or (texture == B.PANE_CUBE_CROSS and level < 0):
        return dw, dh
    fw, fh = face_size(texture, dw, dh)
    L = max(level, 0)
    return 4 * max(1, fw >> L), 3 * max(1, fh >> L)


def convert(fmt, doc, flags):
    """CopyDataForEncoding with gammaCorrect = false, then the flip: ConvertToBC4or5From* for 80 / 83, ConvertToBCFrom* for every other
    id (28 included: ref_convert_pixels dispatches as CopyDataForEncoding does, :93-147)."""
    h, w = doc.shape[:2]
    return np.ascontiguousarray(ref_convert(fmt, doc, flags & (B.FRONT_HAS_ALPHA | FLIPS))[:h, :w])


def copy_layer0(top, depth, layer0, has_alpha):
    """CopyLayersIntoMipMaps(scratch, hasAlpha, 0, 1) over the R8G8B8A8_UNORM scratch `top`, in place."""
    h, w = top.shape[:2]
    channels, alpha = layer0
    channels = [np.ascontiguousarray(c) for c in channels]
    alpha = None if alpha is None else np.ascontiguousarray(alpha)
    planes = (ctypes.c_void_p * 4)(*([c.ctypes.data for c in channels] + [None] * (3 - len(channels))
                                      + [alpha.ctypes.data if alpha is not None else None]))
    assert ref_layers().ref_copy_layers_into_mips(98, depth, w, h, (ctypes.c_void_p * 1)(top.ctypes.data), 1, planes,
                                                  (ctypes.c_longlong * 1)(w * depth // 8), (ctypes.c_int * 1)(len(channels)),
                                                  (ctypes.c_int * 1)(0), 1, int(bool(has_alpha)), 0, ctypes.c_int(1)) == 0


def cube_from_cross(scratch):
    lib = ref_cube()
    h, w = scratch.shape[:2]
    fw, fh = ctypes.c_int(0), ctypes.c_int(0)
    scratch = np.ascontiguousarray(scratch)
    assert lib.ref_cube_from_cross(71, 28, w, h, scratch.ctypes.data_as(ctypes.c_void_p), None, ctypes.byref(fw), ctypes.byref(fh)) == 0
    out = np.zeros((6, fh.value, fw.value, 4), np.uint8)
    lib.ref_cube_from_cross(71, 28, w, h, scratch.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p),
                            ctypes.byref(fw), ctypes.byref(fh))
    return out


def cube_from_layers(depth, w, h, faces, has_alpha):
    """`faces` = six entries, None or (channels, alpha).  The plug-in wants at least six layers; layers of no face name fill the list."""
    named = [(FACE_NAMES[i], f[0], f[1]) for i, f in enumerate(faces) if f is not None]
    dtype = {8: np.uint8, 16: np.uint16, 32: np.float32}[depth]
    while len(named) < 6:
        named.insert(0, ("Background", [np.zeros((h, w), dtype)], None))
    n = len(named)
    names = (ctypes.c_char_p * n)(*[nm.encode() for nm, _, _ in named])
    planes = (ctypes.c_void_p * (4 * n))()
    keep = []
    for i, (_, channels, alpha) in enumerate(named):
        for c, p in enumerate(channels):
            p = np.ascontiguousarray(p, dtype)
            keep.append(p)
            planes[4 * i + c] = p.ctypes.data
        if alpha is not None:
            a = np.ascontiguousarray(alpha, dtype)
            keep.append(a)
            planes[4 * i + 3] = a.ctypes.data
    counts = (ctypes.c_int * n)(*[len(c) for _, c, _ in named])
    out = np.zeros((6, h, w, 4), np.uint8)
    assert ref_cube().ref_cube_from_layers(71, depth, w, h, names, planes, counts, n, int(bool(has_alpha)), out.ctypes.data_as(ctypes.c_void_p)) == 1
    return out


def cross_of(texture, level, faces):
    """ConvertToHorizontalCrossFromCubeMap with the dialog's SetMipLevel / MipLevel: the chain to L when set, the zeroed cross."""
    lib = ref_cube()
    faces = np.ascontiguousarray(faces)
    h, w = faces.shape[1:3]
    ttype = CUBEMAP_CROSSED if texture == B.PANE_CUBE_CROSS else CUBEMAP_LAYERS
    cw, ch = ctypes.c_int(0), ctypes.c_int(0)
    args = (71, ttype, int(level >= 0), max(level, 0), w, h, faces.ctypes.data_as(ctypes.c_void_p))
    assert lib.ref_cross_from_cube(*args, None, ctypes.byref(cw), ctypes.byref(ch)) == 0
    out = np.zeros((ch.value, cw.value, 4), np.uint8)
    lib.ref_cross_from_cube(*args, out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(cw), ctypes.byref(ch))
    return out


def oracle_faces(texture, doc, layers, flags):
    """The six level-0 faces of a cube pane (R8G8B8A8_UNORM)."""
    h, w = doc.shape[:2]
    if texture == B.PANE_CUBE_CROSS:
        return cube_from_cross(convert(71, doc, flags & B.FRONT_HAS_ALPHA))
    return cube_from_layers(doc.itemsize * 8, w, h, layers, flags & B.FRONT_HAS_ALPHA)


def oracle_pane(fmt, texture, level, doc, layers, flags):
    """GetUncompressedImageForPreview: (the H x W x 4 uint8 pane, the dialog's compressed size).  `layers`: None or layer 0 for
    PANE_2D, six faces for PANE_CUBE_LAYERS, ignored for PANE_CUBE_CROSS."""
    h, w = doc.shape[:2]
    size = w * h * 4 if fmt == 28 else 0                 # GetCompressedImageForPreview of the "none" encoding (:936-941)
    has_alpha = flags & B.FRONT_HAS_ALPHA
    if texture == B.PANE_2D:
        if layers is None:
            return convert(fmt, doc, flags), size
        top = convert(fmt, doc, has_alpha)
        copy_layer0(top, doc.itemsize * 8, layers, has_alpha)
        # FlipXYChannelNormalMap of the result: the converter of an RGBA8 scratch with alpha is the identity at depth 8
        return convert(fmt, top, (flags & FLIPS) | B.FRONT_HAS_ALPHA), size
    if texture == B.PANE_CUBE_CROSS and level < 0:       # :1105 does not fire
        return convert(fmt, doc, has_alpha), size
    return cross_of(texture, level, oracle_faces(texture, doc, layers, flags)), size


def document(w, h, planes, depth, seed):
    """A document of `depth` bits with values that reach every conversion rule (32-bit: some values outside 0..1)."""
    rng = np.random.default_rng(seed)
    if depth == 8:
        return rng.integers(0, 256, (h, w, planes), dtype=np.uint8)
    if depth == 16:
        return rng.integers(0, 32769, (h, w, planes), dtype=np.uint16)
    return rng.uniform(-0.1, 1.2, (h, w, planes)).astype(np.float32)


def layer(w, h, depth, channels, alpha, seed):
    """One layer (channels, alpha) of `channels` planes, with an alpha plane when `alpha`."""
    d = document(w, h, channels + (1 if alpha else 0), depth, seed)
    return [d[..., c].copy() for c in range(channels)], (d[..., channels].copy() if alpha else None)


def cube_layers(w, h, depth, seed, missing=(), channels=(1, 2, 3, 3, 2, 1), alpha=(True, False, True, False, True, False)):
    return [None if i in missing else layer(w, h, depth, channels[i], alpha[i], seed + i) for i in range(6)]
