"""The oracle of the "none" save (itw_dds_save_none, include/itw_bcn.h section 12): the plug-in's DoWriteDDS with encoding 28
(IntelPlugin.cpp:2051-2194), restated as glue over the reference's own bodies:

  CopyDataForEncoding(DoMipMaps, gammaCorrect = true) + FlipXYChannelNormalMap   ref_convert_pixels (oracle/build_ref_frontend.py)
  ConvertToCubeMapFromCross / FromLayers                                           the cuts of oracle/build_ref_cube.py (through
                                                                                   tests/preview_uncompressed_lib.py)
  CopyLayersIntoMipMaps(..., 0, 1) and (..., 1)                                    the cut of oracle/build_ref_layers.py
  GenerateMipMaps (the non-WIC generators) and NormalizeNormalMapChain            oracle/build_ref_frontend.py
  SaveToDDSMemory / SaveCubeMipLevelToDDSFile: _EncodeDDSHeader                     oracle/build_ref_dds_none.py, then every level
                                                                                   unpadded, item-major and mip-minor
No encode: CompressToScratchImage swaps the scratch in for 28 (:262-268)."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
import preview_uncompressed_lib as U
from preview_layers_lib import ref_convert, ref_layers

B = T.binding
ALPHA, GAMMA, NORMALIZE = B.FRONT_HAS_ALPHA, B.FRONT_GAMMA, B.FRONT_NORMALIZE
FLIPS = B.FRONT_FLIP_X | B.FRONT_FLIP_Y


def lvl(v, l):
    return max(1, v >> l)


def full_levels(w, h):
    return max(w, h).bit_length()


@functools.lru_cache(None)
def ref_dds_none():
    """oracle/_ref/libitw_ref_dds_none.so (oracle/build_ref_dds_none.py); None if unavailable."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_dds_none
        try:
            path = build_ref_dds_none.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_dds_header.restype = ctypes.c_size_t
    lib.ref_dds_header.argtypes = [ctypes.c_uint32] * 6 + [ctypes.c_void_p, ctypes.c_size_t]
    return lib


def available():
    return U.available() and ref_dds_none() is not None


def dds_header(desc):
    """_EncodeDDSHeader of `desc` (any format the cut knows, R8G8B8A8_UNORM included)."""
    buf = np.zeros(256, np.uint8)
    n = ref_dds_none().ref_dds_header(desc.width, desc.height, desc.mip_levels, desc.array_size, desc.dxgi_format, desc.is_cubemap,
                                      buf.ctypes.data, buf.size)
    assert n in (128, 148)
    return buf[:n]


def ref_chain(top, levels):
    """GenerateMipMaps of an R8G8B8A8_UNORM image through the reference's non-WIC generators: `levels` tight levels."""
    f = T.ref_frontend().ref_mip_chain_rgba8
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    h, w = top.shape[:2]
    dims = [(lvl(h, l), lvl(w, l)) for l in range(levels)]
    out = np.zeros(sum(a * b * 4 for a, b in dims), np.uint8)
    src = np.ascontiguousarray(top)
    assert f(src.ctypes.data, w, h, levels, 0, out.ctypes.data) == 0
    res, off = [], 0
    for a, b in dims:
        res.append(out[off:off + a * b * 4].reshape(a, b, 4).copy())
        off += a * b * 4
    return res


def copy_layers(images, depth, doc_w, doc_h, layers, has_alpha, start):
    """CopyLayersIntoMipMaps(scratch, hasAlpha, start[, 1]) over the R8G8B8A8_UNORM levels `images`, in place."""
    n = len(layers)
    planes = (ctypes.c_void_p * (4 * n))()
    keep = []
    for i, (channels, alpha) in enumerate(layers):
        for c, p in enumerate(channels):
            p = np.ascontiguousarray(p)
            keep.append(p)
            planes[4 * i + c] = p.ctypes.data
        if alpha is not None:
            a = np.ascontiguousarray(alpha)
            keep.append(a)
            planes[4 * i + 3] = a.ctypes.data
    rows = (ctypes.c_longlong * n)(*[doc_w * depth // 8] * n)
    counts = (ctypes.c_int * n)(*[len(c) for c, _ in layers])
    slots = (ctypes.c_int * n)(*[0] * n)
    ptrs = (ctypes.c_void_p * len(images))(*[im.ctypes.data for im in images])
    end = 1 if start == 0 else 2 ** 31 - 1
    assert ref_layers().ref_copy_layers_into_mips(98, depth, doc_w, doc_h, ptrs, len(images), planes, rows, counts, slots, n,
                                                  int(bool(has_alpha)), start, ctypes.c_int(end)) == 0


def normalize(level):
    """NormalizeNormalMapChain on one level: ref_convert_pixels of the RGBA8 level with alpha is the identity, then the normalisation."""
    h, w = level.shape[:2]
    return np.ascontiguousarray(ref_convert(71, level, ALPHA | NORMALIZE)[:h, :w])


def oracle_2d(doc, layers, flags, mip_maps):
    """The levels of a 2-D "none" save (COLOR, COLOR+A, NORMAL MAP; `layers` = [] or the document's layers for FROM_LAYERS)."""
    h, w = doc.shape[:2]
    depth = doc.itemsize * 8
    levels = full_levels(w, h) if mip_maps else 1
    has_alpha = flags & ALPHA
    if layers:
        top = np.ascontiguousarray(ref_convert(71, doc, flags & (ALPHA | GAMMA))[:h, :w])
        copy_layers([top], depth, w, h, layers, has_alpha, 0)
        if flags & FLIPS:                                # FlipXYChannelNormalMap of the result (IntelPlugin.cpp:2100-2105)
            top = np.ascontiguousarray(ref_convert(71, top, (flags & FLIPS) | ALPHA)[:h, :w])
    else:
        top = np.ascontiguousarray(ref_convert(71, doc, flags & (ALPHA | GAMMA | FLIPS))[:h, :w])
    chain = ref_chain(top, levels)
    if len(layers) > 1 and levels > 1:
        copy_layers(chain, depth, w, h, layers, has_alpha, 1)
    if flags & NORMALIZE:
        chain = [normalize(c) for c in chain]
    return B.DdsDesc(w, h, levels, 1, 28, 0), chain


def oracle_faces(texture, doc, layers, flags):
    """The six level-0 faces of a "none" cube: the saved conversion (gamma step included) for a cross, the face layers otherwise."""
    h, w = doc.shape[:2]
    if texture == B.PANE_CUBE_CROSS:
        return U.cube_from_cross(np.ascontiguousarray(ref_convert(71, doc, flags & (ALPHA | GAMMA))[:h, :w]))
    return U.cube_from_layers(doc.itemsize * 8, w, h, layers, flags & ALPHA)


def oracle_cube(texture, doc, layers, flags, mip_maps, L):
    """The levels of a "none" cube save: every level of every face, or level L of every face (SaveCubeMipLevelToDDSFile)."""
    faces = oracle_faces(texture, doc, layers, flags)
    fh, fw = faces.shape[1:3]
    levels = L + 1 if L >= 0 else (full_levels(fw, fh) if mip_maps else 1)
    images = []
    for f in faces:
        chain = ref_chain(f, levels)
        images += [chain[L]] if L >= 0 else chain
    n = 1 if L >= 0 else levels
    return B.DdsDesc(lvl(fw, max(L, 0)), lvl(fh, max(L, 0)), n, 6, 28, 1), images


def oracle_save(opts, doc, layers=None, flags=0):
    """DoWriteDDS with encoding 28: the whole file."""
    if opts.texture == B.PANE_2D:
        desc, images = oracle_2d(doc, layers or [], flags, opts.mip_maps)
    else:
        desc, images = oracle_cube(opts.texture, doc, layers, flags, opts.mip_maps, opts.mip_level)
    return np.concatenate([dds_header(desc)] + [np.ascontiguousarray(im).reshape(-1) for im in images])


def file_bytes(desc):
    """128 + the sum over items and levels of 4 * w_l * h_l."""
    return 128 + desc.array_size * sum(4 * lvl(desc.width, l) * lvl(desc.height, l) for l in range(desc.mip_levels))
