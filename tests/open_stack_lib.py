"""Helpers of the tests of the stack open path (include/itw_bcn.h section 17: volumes, 1-D textures and arrays): the reference cut
(oracle/build_ref_open_stack.py: _DecodeDDSHeader, ScratchImage::Initialize, the image table, _CopyImage's size check and GetImage),
DDS files of every shape in one form of each family, and the open oracle: DoReadStart / DoReadContinue (IntelPlugin.cpp:2419-2742)
over the reference's loader and image choice, with each family's own reference decode / convert / expand and alpha check taken from
the libraries of sections 9 and 13-16."""
import ctypes
import functools
import os
import struct
import sys

import numpy as np

import itw_testlib as T
import open_converted_lib as C
import open_expanded_lib as E
import open_lib
import open_other_bc_lib as O
import open_uncompressed_lib as U
import preview_lib as P

B = T.binding
OPTIONS = open_lib.OPTIONS
VOLUME, HEIGHT = 0x00800000, 0x2

# label -> (section, legacy DDS_PIXELFORMAT or None, DX10 format or None, loaded format, unit bytes, blocks, expanded form name)
FORMS = {
    "BC1": (B.STACK_BC, None, 71, 71, 8, True, None),
    "BC7": (B.STACK_BC, None, 98, 98, 16, True, None),
    "BC6H": (B.STACK_BC, None, 95, 95, 16, True, None),
    "DXT5": (B.STACK_BC, (U.FOURCC, U.fourcc("DXT5"), 0, 0, 0, 0, 0), None, 77, 16, True, None),
    "A8B8G8R8": (B.STACK_RAW, U.PF["A8B8G8R8"], None, 28, 4, False, None),
    "R8G8B8": (B.STACK_RAW, U.PF["R8G8B8"], None, 28, 3, False, None),
    "DX10-11": (B.STACK_RAW, None, 11, 11, 8, False, None),
    "DX10-2": (B.STACK_RAW, None, 2, 2, 16, False, None),
    "A4R4G4B4": (B.STACK_CONVERTED, C.LEGACY["A4R4G4B4"][0], None, 115, 2, False, None),
    "X4R4G4B4": (B.STACK_CONVERTED, C.LEGACY["X4R4G4B4"][0], None, 115, 2, False, None),
    "DX10-10": (B.STACK_CONVERTED, None, 10, 10, 8, False, None),
    "DX10-65": (B.STACK_CONVERTED, None, 65, 65, 1, False, None),
    "DX10-16": (B.STACK_CONVERTED, None, 16, 16, 8, False, None),
    "DXT3": (B.STACK_OTHER_BC, (U.FOURCC, U.fourcc("DXT3"), 0, 0, 0, 0, 0), None, 74, 16, True, None),
    "BC4S": (B.STACK_OTHER_BC, (U.FOURCC, U.fourcc("BC4S"), 0, 0, 0, 0, 0), None, 81, 8, True, None),
    "DX10-94": (B.STACK_OTHER_BC, None, 94, 94, 16, True, None),
    "P8": (B.STACK_EXPANDED, E.FORMS["P8"][0], None, 28, 1, False, "P8"),
    "A8P8": (B.STACK_EXPANDED, E.FORMS["A8P8"][0], None, 28, 2, False, "A8P8"),
    "A8R3G3B2": (B.STACK_EXPANDED, E.FORMS["A8R3G3B2"][0], None, 28, 2, False, "A8R3G3B2"),
    "A4L4": (B.STACK_EXPANDED, E.FORMS["A4L4"][0], None, 115, 1, False, "A4L4"),
}
# shape label -> (dimension, header kind, items, cube)
SHAPES = {
    "legacy-volume": (3, "legacy", 1, False),
    "dx10-volume": (3, "dx10", 1, False),
    "1d": (1, "dx10", 1, False),
    "1d-array-3": (1, "dx10", 3, False),
    "1d-array-6": (1, "dx10", 6, False),
    "2d-array-2": (2, "dx10", 2, False),
    "2d-array-6": (2, "dx10", 6, False),
    "cube-array-2": (2, "dx10", 2, True),
}


def level(v, l):
    return max(1, v >> l)


def count_mips(w, h, d=1):
    n = 1
    while w > 1 or h > 1 or d > 1:
        w, h, d = max(1, w >> 1), max(1, h >> 1), max(1, d >> 1)
        n += 1
    return n


def palette_of(name):
    return E.has_palette(name) if name else False


def shape_ok(label, shape):
    """Whether the form can express the shape: legacy headers only the legacy volume, 'DX10' forms every 'DX10' shape; section 9 has no
    2-D arrays here (itw_dds_open serves them)."""
    section, pf, dx10 = FORMS[label][:3]
    dim, kind = SHAPES[shape][:2]
    if (kind == "legacy") != (pf is not None):
        return False
    return not (dim == 2 and section == B.STACK_BC)


def image_bytes(label, w, h, mip):
    unit, blocks = FORMS[label][4:6]
    lw, lh = level(w, mip), level(h, mip)
    return ((lw + 3) // 4) * ((lh + 3) // 4) * unit if blocks else lw * lh * unit


def payload_bytes(label, w, h, depth, mips, items):
    """ScratchImage's layout restated: items of mip chains; a volume's levels with every slice, the slice count halving."""
    return items * sum(level(depth, m) * image_bytes(label, w, h, m) for m in range(mips))


def header(label, shape, w, h, depth, mips, hflags=None, count=None, dim=None, height=None):
    """magic + DDS_HEADER (+ DDS_HEADER_DXT10) of a form in a shape; `count`, `dim` and `height` override the 'DX10' count, dimension
    and the header's height field."""
    section, pf, dx10 = FORMS[label][:3]
    sdim, kind, items, cube = SHAPES[shape]
    flags = 0x1007 | (0x20000 if mips > 1 else 0) | (VOLUME if sdim == 3 else 0) if hflags is None else hflags
    hh = (1 if sdim == 1 else h) if height is None else height
    if kind == "legacy":
        head = U.header(w, hh, mips, pf, hflags=flags)
    else:
        ddim = {1: 2, 2: 3, 3: 4}[sdim] if dim is None else dim
        head = U.header(w, hh, mips, hflags=flags, dx10=(dx10, ddim, 0x4 if cube else 0, items if count is None else count))
    return head[:24] + struct.pack("<I", depth if sdim == 3 else 0) + head[28:]


def make_file(label, shape, w, h, depth, mips, seed=0, payload=None, palette=None):
    """A file of form `label` in `shape` with a random payload (or `payload`) and, for P8 / A8P8, a random palette (or `palette`)."""
    sdim, _, items, cube = SHAPES[shape]
    hh = 1 if sdim == 1 else h
    d = depth if sdim == 3 else 1
    n = payload_bytes(label, w, hh, d, mips, items * (6 if cube else 1))
    rng = np.random.default_rng(seed)
    if payload is None:
        payload = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    assert len(payload) == n
    pal = b""
    if palette_of(FORMS[label][6]):
        pal = (E.random_palette(seed + 1) if palette is None else np.asarray(palette, np.uint32)).astype("<u4").tobytes()
    return np.frombuffer(header(label, shape, w, h, depth, mips) + pal + bytes(payload), np.uint8).copy()


# ---- the reference cut ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_open_stack.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_open_stack
        try:
            path = build_ref_open_stack.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_stack_load.restype = ctypes.c_long
    lib.ref_stack_load.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.ref_stack_images.restype = ctypes.c_longlong
    lib.ref_stack_images.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_longlong]
    lib.ref_stack_get_image.restype = ctypes.c_longlong
    lib.ref_stack_get_image.argtypes = [ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_uint64] * 3
    return lib


def refs_ready():
    return all(r() is not None for r in (ref, U.ref, C.ref, E.ref, O.ref, open_lib.ref, P.ref))


def _buf(file):
    return np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))


def ref_load(file):
    """LoadFromDDSMemory's metadata and size check: dict, or None when it fails."""
    f = _buf(file)
    out = (ctypes.c_uint64 * 12)()
    if ref().ref_stack_load(f.ctypes.data, f.size, out) != 0:
        return None
    keys = ("width", "height", "depth", "mip_levels", "array_size", "format", "cube", "dimension", "conv", "offset", "images", "payload")
    return dict(zip(keys, [int(v) for v in out]))


def ref_images(file):
    """Every image of the loaded file in ScratchImage's order: (file offset, width, height, rowPitch, slicePitch)."""
    f = _buf(file)
    m = ref_load(f)
    out = (ctypes.c_uint64 * (5 * m["images"]))()
    n = ref().ref_stack_images(f.ctypes.data, f.size, out, m["images"])
    assert n == m["images"]
    return [tuple(int(v) for v in out[5 * i:5 * i + 5]) for i in range(n)]


def ref_get_image(file, mip, item, slice_):
    f = _buf(file)
    return ref().ref_stack_get_image(f.ctypes.data, f.size, mip, item, slice_)


# ---- DoReadStart / DoReadContinue over each family's reference -----------------------------------------------------------------
def _target(label):
    section, loaded = FORMS[label][0], FORMS[label][3]
    if section == B.STACK_BC:
        return (2, 32) if loaded in (95, 96) else ((29, 8) if loaded in (72, 78, 99) else (28, 8))
    if section == B.STACK_RAW:
        return U.TARGETS[loaded]
    if section == B.STACK_CONVERTED:
        return C.LOADED[loaded][2], C.LOADED[loaded][3]
    if section == B.STACK_OTHER_BC:
        return O.ref_target(loaded)
    return 28, 8


def _loaded_texels(label, file, m, im):
    """One image's loaded texels as the family's loader leaves them (uncompressed families), as bytes."""
    section, loaded, name = FORMS[label][0], FORMS[label][3], FORMS[label][6]
    off, w, h, _, slice_pitch = im
    src = _buf(bytes(file[off:off + slice_pitch]))
    if section == B.STACK_RAW:
        out = np.zeros(w * h * U.TEXEL[loaded], np.uint8)
        assert U.ref().ref_copy_image(src.ctypes.data, w, h, 1, 1, loaded, m["conv"], out.ctypes.data) == out.size
        return out
    if section == B.STACK_CONVERTED:
        return _buf(C.set_alpha_4444(src) if m["conv"] & 0x2 else src)
    pal = np.frombuffer(bytes(file[128:1152]), "<u4") if palette_of(name) else None
    return E.ref_expand(name, src, pal)


def ref_all_opaque(label, file):
    """ScratchImage::IsAlphaAllOpaque over every image of the loaded file, through the family's cut branch."""
    section, loaded = FORMS[label][0], FORMS[label][3]
    m = ref_load(file)
    for im in ref_images(file):
        off, w, h, _, sp = im
        if section in (B.STACK_BC, B.STACK_OTHER_BC):
            blocks = _buf(bytes(file[off:off + sp]))
            lib = open_lib.ref() if section == B.STACK_BC else O.ref()
            fn = lib.ref_is_alpha_all_opaque if section == B.STACK_BC else lib.ref_obc_is_alpha_all_opaque
            ok = fn(loaded, blocks.ctypes.data, w, h, 1, 1)
        else:
            texels = _loaded_texels(label, file, m, im)
            fmt = 115 if section == B.STACK_EXPANDED and loaded == 115 else loaded
            lib = U.ref() if fmt in U.TARGETS else C.ref()
            ok = lib.ref_is_alpha_all_opaque(fmt, texels.ctypes.data, w, h, 1, 1)
        if not ok:
            return False
    return True


def ref_has_alpha(label, file):
    """loadInfo.hasAlpha (:2468-2472): HasAlpha(loaded) && !IsAlphaAllOpaque(), not BC1."""
    section, loaded = FORMS[label][0], FORMS[label][3]
    if section == B.STACK_BC:
        has = loaded in (77, 78, 98, 99)
    elif section == B.STACK_OTHER_BC:
        has = bool(O.ref().ref_has_alpha(loaded))
    elif section == B.STACK_CONVERTED:
        has = C.LOADED[loaded][4]
    else:
        has = True
    return has and not ref_all_opaque(label, file)


def image_texels(label, file, m, im, target):
    """One image through the family's reference decode / convert / expand into the target: (h, w, 4)."""
    section, loaded, name = FORMS[label][0], FORMS[label][3], FORMS[label][6]
    off, w, h, _, sp = im
    if section == B.STACK_BC:
        return P.ref_decompress(loaded, bytes(file[off:off + sp]), w, h, target)
    if section == B.STACK_OTHER_BC:
        return O.ref_decompress(loaded, bytes(file[off:off + sp]), w, h, target)
    texels = _loaded_texels(label, file, m, im)
    if section == B.STACK_RAW:
        return texels.view(U.DTYPES[loaded]).reshape(h, w, 4)
    if section == B.STACK_CONVERTED:
        return C.ref_convert(loaded, texels).view(C.DTYPES[C.LOADED[loaded][3]]).reshape(h, w, 4)
    return (C.ref_convert(115, texels) if loaded == 115 else texels).reshape(h, w, 4)


def call_image(start, call):
    """DoReadContinue's GetImage arguments (:2656-2672): (mip, item, slice)."""
    if start["is_cube"]:
        return 0, call, 0
    return (call, 0, 0) if start["load_mip_layers"] else (0, 0, 0)


def oracle_open(label, file, options):
    """(metadata, DoReadStart's decisions, every layer) of the reference pipeline."""
    m = ref_load(file)
    has_alpha = ref_has_alpha(label, file)
    proxy = B.DdsDesc(m["width"], m["height"], m["mip_levels"], m["array_size"], 77, m["cube"])       # HasAlpha, not BC1
    start = open_lib.read_start(proxy, not has_alpha, options)
    start["target_dxgi"], start["depth"] = _target(label)
    images = ref_images(file)
    dtype = {8: np.uint8, 16: np.uint16, 32: np.float32}[start["depth"]]
    forced = {8: 255, 16: U.ref().ref_convert_to_16bit_255(), 32: 1.0}[start["depth"]]
    layers = []
    for call in range(start["calls"]):
        index = ref_get_image(file, *call_image(start, call))
        im = images[index]
        img = image_texels(label, file, m, im, start["target_dxgi"])
        ih, iw = img.shape[:2]
        planes = start["planes"]
        out = np.zeros((m["height"], m["width"], planes), dtype)                                       # :2646
        out[:ih, :iw] = img[..., :planes]
        if start["is_cube"] and start["has_alpha"]:                                                     # :2696, :2711, :2724
            out[:ih, :iw, planes - 1] = forced
        layers.append(out)
    return m, start, layers


info_fields = U.info_fields
