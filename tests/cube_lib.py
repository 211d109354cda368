"""The plug-in's cube-map save and preview (IntelPlugin.cpp) restated line by line for the tests, composed from the handwritten oracle's
front end, chains and encoders, the layer-copy oracle (oracle/itw_oracle_layers.cpp), the reference's own DDS header body
(oracle/build_ref_dds.py) and its own DirectX::Decompress (oracle/build_ref_preview.py).

  DoWriteDDS, cube branches (:2062-2171)   faces -> [chain] -> encode -> DDS
  ConvertToCubeMapFromCross (:1200-1265)   six cells; a vertical cross (doc width < doc height) takes -Z from cell (1, 3)
  CopyRectangle of an sRGB document scratch into the UNORM cube (DirectXTexMisc.cpp:174-274): r, g, b through XMColorSRGBToRGB + the
                                           UNORM8 store, alpha as is
  ConvertToCubeMapFromLayers (:1270-1416)  zeroed faces, then each named layer by CopyFromLayerChannelIntoImage / FillLayerDataToWhite
  SaveCubeMipLevelToDDSFile (:1856-1871)   the one-level cube of level L
  GetCompressedImageForPreview (:933-1080) and ConvertToHorizontalCrossFromCubeMap (:1421-1501): the cross of level L, zero cells
"""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
import preview_lib as PL

B = T.binding
F32 = np.float32
CELLS = (((2, 1), (0, 1), (1, 0), (1, 2), (1, 1), (3, 1)),          # horizontal 4x3, IntelPlugin.cpp:1211
         ((2, 1), (0, 1), (1, 0), (1, 2), (1, 1), (1, 3)))          # vertical 3x4, :1225-1226
SRGB = (72, 78, 99)


def lvl(v, l):
    return max(1, v >> l)


def full_levels(w, h):
    return max(w, h).bit_length()


def face_size(source, dw, dh):
    if source == B.CUBE_LAYERS:
        return dw, dh
    return (dw // 3, dh // 4) if dw < dh else (dw // 4, dh // 3)


@functools.lru_cache(None)
def srgb_in_bytes():
    """byte b -> store8(XMColorSRGBToRGB(b * (1/255))) with the oracle's own conversion (C library powf)."""
    lib = T.oracle().lib
    f = lib.oracle_srgb_to_linear
    f.restype = ctypes.c_float
    f.argtypes = [ctypes.c_float]
    step = np.array([1.0 / 255.0], F32)[0]
    out = []
    for b in range(256):
        x = F32(f(float(F32(b) * step)))
        x = min(max(x, F32(0.0)), F32(1.0))
        out.append(int(F32(x * F32(255.0) + F32(0.5))))
    return np.array(out, np.uint8)


def oracle_cross_faces(fmt, doc, flags, linear):
    """ConvertToCubeMapFromCross on the front end's output: six w x h faces (RGBA8 / RGBA16F bit patterns)."""
    o = T.oracle()
    dh, dw = doc.shape[:2]
    w, h = face_size(B.CUBE_CROSS, dw, dh)
    cells = CELLS[1 if dw < dh else 0]
    conv = o.convert_pixels(PL.NAME[fmt], np.ascontiguousarray(doc), flags, pad=False)
    faces = []
    for cx, cy in cells:
        f = np.ascontiguousarray(conv[cy * h:(cy + 1) * h, cx * w:(cx + 1) * w])
        if linear:
            f = f.copy()
            f[..., :3] = srgb_in_bytes()[f[..., :3]]
        faces.append(f)
    return faces


def oracle_layer_faces(fmt, w, h, depth, faces, has_alpha):
    """ConvertToCubeMapFromLayers: zeroed faces, each named layer copied whole by the layer-copy oracle."""
    import test_mips_from_layers as ML
    hdr = fmt == 95
    out = []
    for face in faces:
        img = np.zeros((h, w, 4), np.uint16 if hdr else np.uint8)
        if face is not None:
            ML.oracle_copy(img, depth, w, face, has_alpha)
        out.append(img)
    return out


def oracle_faces(opts, doc, faces, flags, preview=False):
    fmt = opts.dxgi_format
    if opts.source == B.CUBE_CROSS:
        # the document scratch is R8G8B8A8_UNORM_SRGB only for an _SRGB save with mip maps (IntelPlugin.cpp:152-154, :957)
        return oracle_cross_faces(fmt, doc, flags, linear=(not preview) and bool(opts.mip_maps) and fmt in SRGB)
    h, w = doc.shape[:2]
    return oracle_layer_faces(fmt, w, h, doc.itemsize * 8, faces, flags & B.FRONT_HAS_ALPHA)


def oracle_chain(fmt, face, levels):
    """The cube scratch's chain: R8G8B8A8_UNORM (never the sRGB chain) or RGBA16F, DirectXTex's non-WIC generators."""
    import test_mips_f16 as HM
    if fmt == 95:
        return HM.oracle_chain(face, levels)
    return T.oracle_mip_chain_rgba8(face, 0, levels, pad=False)


def settings_of(fmt, prof):
    return T.oracle().profile(prof) if prof else None


def encode_level(fmt, level, prof):
    return T.oracle().encode(PL.NAME[fmt], np.ascontiguousarray(pad4(level)), settings_of(fmt, prof))


def pad4(level):
    h, w = level.shape[:2]
    return np.pad(level, ((0, (-h) % 4), (0, (-w) % 4), (0, 0)), mode="edge")


@functools.lru_cache(None)
def ref_dds():
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_dds
        path = build_ref_dds.build(verbose=False)
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_dds_header.restype = ctypes.c_size_t
    lib.ref_dds_header.argtypes = [ctypes.c_uint32] * 6 + [ctypes.c_void_p, ctypes.c_size_t]
    return lib


def dds_header(desc):
    buf = np.zeros(256, np.uint8)
    n = ref_dds().ref_dds_header(desc.width, desc.height, desc.mip_levels, desc.array_size, desc.dxgi_format, desc.is_cubemap,
                                 buf.ctypes.data, buf.size)
    assert n in (128, 148)
    return buf[:n]


def oracle_save(opts, doc, faces, flags, prof, threads=1):
    """DoWriteDDS for the cube types, and SaveCubeMipLevelToDDSFile when a level is set: the whole file.  `threads` > 1 runs the six
    faces' chains and encodes side by side (the oracle's C calls release the GIL)."""
    fmt = opts.dxgi_format
    dh, dw = doc.shape[:2]
    w, h = face_size(opts.source, dw, dh)
    full = full_levels(w, h)
    L = opts.mip_level
    levels = full if (opts.mip_maps or L >= 0) else 1             # the set level forces the chain (IntelPlugin.cpp:2112)
    keep = [L] if L >= 0 else list(range(levels))
    if L >= 0:
        levels = L + 1                                            # the levels after L do not change level L
    def one(face):
        chain = oracle_chain(fmt, face, levels)
        return [encode_level(fmt, chain[l], prof) for l in keep]
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max(1, threads)) as pool:
        parts = [part for face_parts in pool.map(one, oracle_faces(opts, doc, faces, flags)) for part in face_parts]
    desc = B.DdsDesc(lvl(w, max(L, 0)), lvl(h, max(L, 0)), len(keep), 6, fmt, 1)
    return np.concatenate([dds_header(desc)] + parts)


def oracle_preview(opts, doc, faces, flags, prof):
    """GetCompressedImageForPreview for the cube types: (display image, compressed bytes)."""
    fmt = opts.dxgi_format
    depth = doc.itemsize * 8
    if opts.source == B.CUBE_CROSS and opts.mip_level < 0:
        return PL.oracle_preview(fmt, [doc], flags, prof)
    L = max(opts.mip_level, 0)
    cross = oracle_level_cross(fmt, oracle_faces(opts, doc, faces, flags, preview=True), L)
    blocks = encode_level(fmt, cross, prof)
    src, target = PL.shown_format(fmt, depth)
    return PL.ref_decompress(src, blocks, cross.shape[1], cross.shape[0], target), blocks.size


def oracle_level_cross(fmt, faces, L):
    """ConvertToHorizontalCrossFromCubeMap: the chain to level L when a level is set, then a zeroed 4 wL x 3 hL image (Initialize2D)
    with level L of each face in its cell."""
    h, w = faces[0].shape[:2]
    wl, hl = lvl(w, L), lvl(h, L)
    cross = np.zeros((3 * hl, 4 * wl, 4), faces[0].dtype)
    for face, (cx, cy) in zip(faces, CELLS[0]):
        level = oracle_chain(fmt, face, L + 1)[L] if L > 0 else face
        cross[cy * hl:(cy + 1) * hl, cx * wl:(cx + 1) * wl] = level
    return cross
