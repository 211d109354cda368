"""The oracle of the mip-maps-from-layers preview pane (itw_preview_layers, include/itw_bcn.h section 11): the plug-in's
GetCompressedImageForPreview with IsMipMapsDefinedByLayer (IntelPlugin.cpp:957-1059), composed from the reference's own bodies --
the front-end converters, flip and normalisation of oracle/build_ref_frontend.py, the CopyLayersIntoMipMaps cut of
oracle/build_ref_layers.py, the handwritten oracle's encoder and the DirectX::Decompress cut of oracle/build_ref_preview.py (through
tests/preview_lib.py, whose display rules it shares)."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
from preview_lib import NAME, ref_decompress, shown_format

B = T.binding


@functools.lru_cache(None)
def ref_layers():
    """oracle/_ref/libitw_ref_layers.so: the reference's CopyLayersIntoMipMaps (oracle/build_ref_layers.py); None if unavailable."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_layers
        try:
            path = build_ref_layers.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_copy_layers_into_mips.restype = ctypes.c_int
    return lib


def ref_convert(fmt, px, flags):
    """The reference's CopyDataForEncoding converters, flip, normalise and pad (ref_convert_pixels of oracle/_ref/libitw_ref_frontend)."""
    h, w, planes = px.shape
    px = np.ascontiguousarray(px)
    out = np.zeros(((h + 3) & ~3, (w + 3) & ~3, 4), np.uint16 if fmt == 95 else np.uint8)
    assert T.ref_frontend().ref_convert_pixels(fmt, px.ctypes.data, w, h, planes, px.itemsize * 8, flags, out.ctypes.data) == 0
    return out


def oracle_preview_layers(fmt, composite, layer0, flags, profile):
    """GetCompressedImageForPreview with IsMipMapsDefinedByLayer (IntelPlugin.cpp:957-1059) from the reference's own bodies, in its order:
    CopyDataForEncoding (the converters of ref_convert_pixels, no flip or normalisation) -> CopyLayersIntoMipMaps(..., 0, 1) of layer
    0 -> FlipXYChannelNormalMap -> NormalizeNormalMapChain -> pad (ref_convert_pixels once more, of the RGBA result: an identity
    conversion of RGBA8, and of RGBA16F widened by the reference's own half conversion) -> the handwritten oracle's encoder ->
    DirectX::Decompress of the reference.  Returns (display image, compressed bytes)."""
    name = NAME[fmt]
    enc = B.FORMATS[name][0]
    hdr = name == "BC6H"
    h, w = composite.shape[:2]
    depth = composite.itemsize * 8
    top = np.ascontiguousarray(ref_convert(enc, composite, flags & (B.FRONT_HAS_ALPHA | B.FRONT_GAMMA))[:h, :w])
    channels, alpha = layer0
    planes = (ctypes.c_void_p * 4)(*([c.ctypes.data for c in channels] + [None] * (3 - len(channels))
                                      + [alpha.ctypes.data if alpha is not None else None]))
    assert ref_layers().ref_copy_layers_into_mips(95 if hdr else 98, depth, w, h, (ctypes.c_void_p * 1)(top.ctypes.data), 1, planes,
                                                  (ctypes.c_longlong * 1)(w * depth // 8), (ctypes.c_int * 1)(len(channels)),
                                                  (ctypes.c_int * 1)(0), 1, int(bool(flags & B.FRONT_HAS_ALPHA)), 0, ctypes.c_int(1)) == 0
    post = flags & (B.FRONT_FLIP_X | B.FRONT_FLIP_Y | B.FRONT_NORMALIZE)
    if hdr:                                                       # BC6H ignores alpha; the display's is 1.0
        widen = np.vectorize(lambda v: T.ref_frontend().ref_half_to_float(int(v)), otypes=[np.float32])
        padded = ref_convert(95, widen(top), post)
    else:
        padded = ref_convert(enc, top, post | B.FRONT_HAS_ALPHA)
    o = T.oracle()
    blocks = o.encode(name, np.ascontiguousarray(padded), o.profile(profile) if profile else None)
    src, target = shown_format(fmt, depth)
    return ref_decompress(src, blocks, w, h, target), blocks.size
