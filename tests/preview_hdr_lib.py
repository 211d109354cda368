"""The oracles of the preview dialog for HDR documents (include/itw_bcn.h section 18).

  itw_preview_view_exposed      FetchPreviewRGB with the exposure as an argument (oracle/build_ref_view_exposed.py)
  itw_preview_uncompressed_hdr  GetUncompressedImageForPreview for BC6H_UF16: the glue of tests/preview_uncompressed_lib.py over the
                                reference's own bodies with the R16G16B16A16_FLOAT scratch (the BC6H converters of
                                build_ref_frontend.py, the cube and cross cuts of build_ref_cube.py for encoding 95, the
                                CopyLayersIntoMipMaps cut for encoding 95), then the reference's non-WIC _Convert of
                                build_ref_open_converted.py: ref_convert_texels(10, 28)
and the CPU emulation of the kernels' element routines (tests/emu/view_hdr_emu.cpp)."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
import open_converted_lib as OC
import preview_uncompressed_lib as U
from preview_layers_lib import ref_convert, ref_layers

B = T.binding
HDR = 95
# the dialog's slider: exposure = float(pow(2, pos * 0.01)) for pos in -1000..1000 (PreviewDialog.cpp:868-887)
SLIDER = np.array([2.0 ** (pos * 0.01) for pos in range(-1000, 1001)], np.float32)


@functools.lru_cache(None)
def ref_view_exposed():
    """oracle/_ref/libitw_ref_view_exposed.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_view_exposed
        try:
            path = build_ref_view_exposed.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_fetch_preview_rgb_exposed.restype = None
    lib.ref_fetch_preview_rgb_exposed.argtypes = ([ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double]
                                                  + [ctypes.c_int] * 2 + [ctypes.c_void_p] + [ctypes.c_int] * 6 + [ctypes.c_float])
    return lib


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_view_hdr_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_view_exposed.restype = None
    lib.emu_view_exposed.argtypes = ([ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_longlong] + [ctypes.c_int] * 4
                                     + [ctypes.c_double, ctypes.c_int, ctypes.c_uint, ctypes.c_uint, ctypes.c_float, ctypes.c_void_p])
    lib.emu_hdr_unorm8.restype = None
    lib.emu_hdr_unorm8.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    return lib


def ref_fetch(buf, pitch, src_w, src_h, planes, fmt, w, h, x, y, zoom, mip, mask, matte, exposure):
    """FetchPreviewRGB of the reference cut, exposure included, into an h x w x 3 buffer.  `fmt`: the depth or DXGI format it switches on."""
    out = np.zeros((h, w, 3), np.uint8)
    ref_view_exposed().ref_fetch_preview_rgb_exposed(out.ctypes.data, w, h, x, y, zoom, mask, matte, buf.ctypes.data, src_w, src_h, planes,
                                                     fmt, pitch, mip, float(np.float32(exposure)))
    return out


def emu_fetch(buf, pitch, src_w, src_h, planes, depth, w, h, x, y, zoom, mip, mask, matte, exposure):
    out = np.zeros((h, w, 3), np.uint8)
    emu().emu_view_exposed(buf.ctypes.data, src_w, src_h, planes, depth, pitch, w, h, x, y, zoom, mip, mask, matte,
                           float(np.float32(exposure)), out.ctypes.data)
    return out


def float_to_byte(v):
    """FloatToByte (IntelPlugin.h:41-48) of float64 values: the clamps, then the truncation of v * 255 (NaN -> 0)."""
    v = np.asarray(v, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        b = np.where(v > 1, 255, np.where(v < 0, 0, np.nan_to_num(v * 255.0, nan=0.0))).astype(np.int64)
    return b.astype(np.uint8)


def straddling_pairs(count=64, seed=0):
    """(f, exposure) float pairs whose float product f * exposure and exact product lie on opposite sides of a k / 255 boundary of
    FloatToByte: an implementation that multiplies in double shows a byte one off from the plug-in's.  Exposures from the slider."""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    out = []
    while len(out) < count:
        e = SLIDER[rng.integers(0, SLIDER.size)]
        k = int(rng.integers(1, 255))
        base = f32(k / 255.0 / float(e))
        for d in range(-8, 9):
            f = np.nextafter(base, f32(np.inf) if d > 0 else f32(-np.inf), dtype=np.float32) if d else base
            for _ in range(abs(d) - 1):
                f = np.nextafter(f, f32(np.inf) if d > 0 else f32(-np.inf), dtype=np.float32)
            prod_f = float(f32(f * e))                        # the float product, then widened
            prod_d = float(f) * float(e)                      # exact in double (24 + 24 bits)
            if float_to_byte(prod_f) != float_to_byte(prod_d):
                out.append((f32(f), f32(e)))
                break
    return out


def ref_hdr_unorm8(halves):
    """_Convert(R16G16B16A16_FLOAT -> R8G8B8A8_UNORM, filter 0) of the reference: one byte per half (n a multiple of 4)."""
    halves = np.ascontiguousarray(halves, np.uint16)
    out = np.zeros(halves.size, np.uint8)
    assert OC.ref().ref_convert_texels(10, 28, halves.ctypes.data, halves.size // 4, out.ctypes.data) == 0
    return out


# ---- GetUncompressedImageForPreview for 95 ------------------------------------------------------------------------------------
def available():
    return U.available() and OC.ref() is not None


def convert_hdr(doc, flags):
    """CopyDataForEncoding with gammaCorrect = false through ConvertToBC6From*: the H x W x 4 RGBA16F scratch (uint16 halves)."""
    h, w = doc.shape[:2]
    return np.ascontiguousarray(ref_convert(HDR, doc, flags & B.FRONT_HAS_ALPHA)[:h, :w])


def copy_layer0_hdr(top, depth, layer0, has_alpha):
    """CopyLayersIntoMipMaps(scratch, hasAlpha, 0, 1) over the RGBA16F scratch `top`, in place."""
    h, w = top.shape[:2]
    channels, alpha = layer0
    channels = [np.ascontiguousarray(c) for c in channels]
    alpha = None if alpha is None else np.ascontiguousarray(alpha)
    planes = (ctypes.c_void_p * 4)(*([c.ctypes.data for c in channels] + [None] * (3 - len(channels))
                                      + [alpha.ctypes.data if alpha is not None else None]))
    assert ref_layers().ref_copy_layers_into_mips(HDR, depth, w, h, (ctypes.c_void_p * 1)(top.ctypes.data), 1, planes,
                                                  (ctypes.c_longlong * 1)(w * depth // 8), (ctypes.c_int * 1)(len(channels)),
                                                  (ctypes.c_int * 1)(0), 1, int(bool(has_alpha)), 0, ctypes.c_int(1)) == 0


def cube_from_cross_hdr(scratch):
    lib = U.ref_cube()
    h, w = scratch.shape[:2]
    fw, fh = ctypes.c_int(0), ctypes.c_int(0)
    scratch = np.ascontiguousarray(scratch)
    assert lib.ref_cube_from_cross(HDR, 10, w, h, scratch.ctypes.data_as(ctypes.c_void_p), None, ctypes.byref(fw), ctypes.byref(fh)) == 0
    out = np.zeros((6, fh.value, fw.value, 4), np.uint16)
    lib.ref_cube_from_cross(HDR, 10, w, h, scratch.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p),
                            ctypes.byref(fw), ctypes.byref(fh))
    return out


def cube_from_layers_hdr(depth, w, h, faces, has_alpha):
    """`faces` = six entries, None or (channels, alpha); unnamed layers fill the list up to the six the plug-in wants."""
    named = [(U.FACE_NAMES[i], f[0], f[1]) for i, f in enumerate(faces) if f is not None]
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
    out = np.zeros((6, h, w, 4), np.uint16)
    assert U.ref_cube().ref_cube_from_layers(HDR, depth, w, h, names, planes, counts, n, int(bool(has_alpha)),
                                             out.ctypes.data_as(ctypes.c_void_p)) == 1
    return out


def cross_of_hdr(texture, level, faces):
    """ConvertToHorizontalCrossFromCubeMap of the RGBA16F cube: the chain to L when set, the zeroed cross of level L."""
    lib = U.ref_cube()
    faces = np.ascontiguousarray(faces)
    h, w = faces.shape[1:3]
    ttype = U.CUBEMAP_CROSSED if texture == B.PANE_CUBE_CROSS else U.CUBEMAP_LAYERS
    cw, ch = ctypes.c_int(0), ctypes.c_int(0)
    args = (HDR, ttype, int(level >= 0), max(level, 0), w, h, faces.ctypes.data_as(ctypes.c_void_p))
    assert lib.ref_cross_from_cube(*args, None, ctypes.byref(cw), ctypes.byref(ch)) == 0
    out = np.zeros((ch.value, cw.value, 4), np.uint16)
    lib.ref_cross_from_cube(*args, out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(cw), ctypes.byref(ch))
    return out


def oracle_scratch(texture, level, doc, layers, flags):
    """The R16G16B16A16_FLOAT scratch GetUncompressedImageForPreview builds for 95, before its Convert."""
    h, w = doc.shape[:2]
    has_alpha = flags & B.FRONT_HAS_ALPHA
    if texture == B.PANE_2D:
        top = convert_hdr(doc, has_alpha)
        copy_layer0_hdr(top, doc.itemsize * 8, layers, has_alpha)
        return top
    if texture == B.PANE_CUBE_CROSS and level < 0:       # :1105 does not fire: the converted document
        return convert_hdr(doc, has_alpha)
    if texture == B.PANE_CUBE_CROSS:
        faces = cube_from_cross_hdr(convert_hdr(doc, has_alpha))
    else:
        faces = cube_from_layers_hdr(doc.itemsize * 8, w, h, layers, has_alpha)
    return cross_of_hdr(texture, level, faces)


def oracle_pane(texture, level, doc, layers, flags):
    """The H x W x 4 uint8 pane of itw_preview_uncompressed_hdr."""
    scratch = oracle_scratch(texture, level, doc, layers, flags)
    return ref_hdr_unorm8(scratch.reshape(-1)).reshape(scratch.shape)
