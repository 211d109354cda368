"""Helpers of the tests of the converted open path (include/itw_bcn.h section 14): the reference cut (oracle/build_ref_open_converted.py:
_LoadScanline's cases, _ConvertScanline, _StoreScanline, IsAlphaAllOpaque's non-compressed branch), the CPU execution of the product's
per-texel routines (tests/emu/open_conv_emu.cpp), DDS files of every header form, and the open oracle: DoReadStart / DoReadContinue
(IntelPlugin.cpp:2419-2742) with DirectX::Convert's non-WIC _Convert over the reference's own bodies.  The header decoder, the file
writers and DoReadStart's layer decisions are open_uncompressed_lib's."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
import open_uncompressed_lib as U

B = T.binding
OPTIONS = U.OPTIONS
RGBA, RGB, FOURCC, LUM, LUMA, ALPHA = U.RGBA, U.RGB, U.FOURCC, U.LUM, U.LUMA, U.ALPHA

# loaded DXGI format -> (csrc/open_raw.cuh texel form, bytes per texel, target, depth, HasAlpha)
LOADED = {
    10: (5, 8, 11, 16, True), 54: (6, 2, 11, 16, False), 34: (7, 4, 11, 16, False), 13: (8, 8, 11, 16, True),
    35: (9, 4, 11, 16, False), 37: (10, 4, 11, 16, False), 58: (11, 2, 11, 16, False), 26: (12, 4, 11, 16, False),
    67: (13, 4, 11, 16, False), 49: (14, 2, 28, 8, False), 51: (15, 2, 28, 8, False), 31: (16, 4, 28, 8, True),
    63: (17, 1, 28, 8, False), 65: (18, 1, 28, 8, True), 115: (19, 2, 28, 8, True), 16: (21, 8, 2, 32, False),
}
KIND_BGRX4 = 20
DTYPES = {8: np.uint8, 16: np.uint16, 32: np.float32}
# legacy header forms: name -> (DDS_PIXELFORMAT, ITW_CONV_*, loaded format)
LEGACY = {
    "G16R16": ((RGB, 0, 32, 0xffff, 0xffff0000, 0, 0), B.CONV_G16R16, 35),
    "A8L8": ((LUMA, 0, 16, 0xff, 0, 0, 0xff00), B.CONV_A8L8, 49),
    "A8": ((ALPHA, 0, 8, 0, 0, 0, 0xff), B.CONV_A8, 65),
    "A4R4G4B4": ((RGBA, 0, 16, 0x0f00, 0x00f0, 0x000f, 0xf000), B.CONV_A4R4G4B4, 115),
    "X4R4G4B4": ((RGB, 0, 16, 0x0f00, 0x00f0, 0x000f, 0), B.CONV_X4R4G4B4, 115),
    "FourCC110": ((FOURCC, 110, 0, 0, 0, 0, 0), B.CONV_Q16W16V16U16, 13),
    "FourCC111": ((FOURCC, 111, 0, 0, 0, 0, 0), B.CONV_R16F, 54),
    "FourCC112": ((FOURCC, 112, 0, 0, 0, 0, 0), B.CONV_G16R16F, 34),
    "FourCC113": ((FOURCC, 113, 0, 0, 0, 0, 0), B.CONV_A16B16G16R16F, 10),
    "FourCC115": ((FOURCC, 115, 0, 0, 0, 0, 0), B.CONV_G32R32F, 16),
}


def kind_of(loaded, form):
    return KIND_BGRX4 if form == B.CONV_X4R4G4B4 else LOADED[loaded][0]


def legacy_file(name, w, h, mips=1, cube=False, payload=None, seed=0):
    pf, _, loaded = LEGACY[name]
    n = U.payload_bytes(w, h, mips, 6 if cube else 1, LOADED[loaded][1])
    if payload is None:
        payload = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()
    assert len(payload) == n
    return np.frombuffer(U.header(w, h, mips, pf, cube) + bytes(payload), np.uint8).copy()


def dx10_file(fmt, w, h, mips=1, cube=False, payload=None, seed=0):
    n = U.payload_bytes(w, h, mips, 6 if cube else 1, LOADED[fmt][1])
    if payload is None:
        payload = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()
    assert len(payload) == n
    return np.frombuffer(U.header(w, h, mips, dx10=(fmt, 3, 0x4 if cube else 0, 1)) + bytes(payload), np.uint8).copy()


# every header form: (label, writer(w, h, mips, cube, payload=None, seed=0))
FORMS = [(name, functools.partial(legacy_file, name)) for name in LEGACY] + \
        [(f"DX10-{fmt}", functools.partial(dx10_file, fmt)) for fmt in LOADED]


# ---- the reference cut and the product's per-texel routines ---------------------------------------------------------------------
@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_open_converted.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_open_converted
        try:
            path = build_ref_open_converted.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_convert_texels.restype = ctypes.c_int
    lib.ref_convert_texels.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    lib.ref_is_alpha_all_opaque.restype = ctypes.c_int
    lib.ref_is_alpha_all_opaque.argtypes = [ctypes.c_uint32, ctypes.c_void_p] + [ctypes.c_uint32] * 4
    lib.ref_texels_opaque.restype = None
    lib.ref_texels_opaque.argtypes = [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    for name in ("ref_use_wic", "ref_is_srgb", "ref_has_alpha"):
        getattr(lib, name).restype = ctypes.c_int
    lib.ref_use_wic.argtypes = [ctypes.c_uint32, ctypes.c_uint32]
    lib.ref_is_srgb.argtypes = lib.ref_has_alpha.argtypes = [ctypes.c_uint32]
    lib.ref_bits_per_color.restype = ctypes.c_uint
    lib.ref_bits_per_color.argtypes = [ctypes.c_uint32]
    return lib


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_open_conv_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_conv_texels.restype = ctypes.c_int
    lib.emu_conv_texels.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]
    lib.emu_conv_alpha_below.restype = ctypes.c_int
    lib.emu_conv_alpha_below.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]
    lib.emu_conv_scope.restype = None
    lib.emu_conv_scope.argtypes = [ctypes.c_uint, ctypes.c_void_p]
    return lib


def set_alpha_4444(src):
    """_CopyScanline's TEXP_SCANLINE_SETALPHA for B4G4R4A4 (the X4R4G4B4 header, CONV_FLAGS_NOALPHA): the alpha nibble becomes 0xF."""
    return (np.frombuffer(bytes(src), np.uint16) | 0xF000).astype(np.uint16).tobytes()


def ref_convert(loaded, src):
    """_Convert of loaded texels `src` into DoReadStart's target: the target's texels as bytes."""
    src = np.ascontiguousarray(np.frombuffer(bytes(src), np.uint8))
    n = src.size // LOADED[loaded][1]
    target = LOADED[loaded][2]
    out = np.zeros(n * {2: 16, 11: 8, 28: 4}[target], np.uint8)
    assert ref().ref_convert_texels(loaded, target, src.ctypes.data, n, out.ctypes.data) == 0
    return out


def emu_texels(kind, planes, src, force=False):
    src = np.ascontiguousarray(np.frombuffer(bytes(src), np.uint8))
    nbytes = {20: 2}.get(kind) or next(v[1] for v in LOADED.values() if v[0] == kind)
    plane = {5: 2, 6: 2, 7: 2, 8: 2, 9: 2, 10: 2, 11: 2, 12: 2, 13: 2, 21: 4}.get(kind, 1)
    n = src.size // nbytes
    out = np.zeros(n * planes * plane, np.uint8)
    assert emu().emu_conv_texels(kind, planes, src.ctypes.data, n, int(force), out.ctypes.data) == 0
    return out


def ref_opaque(loaded, src):
    src = np.ascontiguousarray(np.frombuffer(bytes(src), np.uint8))
    n = src.size // LOADED[loaded][1]
    out = np.zeros(n, np.uint8)
    ref().ref_texels_opaque(loaded, src.ctypes.data, n, out.ctypes.data)
    return out


def emu_below(kind, src, nbytes, slot=0):
    """The scan's predicate on each texel, placed at alpha slot `slot` of its word (byte 0..3 for A8, ushort 0..1 for 4444)."""
    src = np.ascontiguousarray(np.frombuffer(bytes(src), np.uint8))
    n = src.size // nbytes
    out = np.zeros(n, np.uint8)
    assert emu().emu_conv_alpha_below(kind, src.ctypes.data, n, slot, out.ctypes.data) == 0
    return out


def emu_scope(dxgi):
    """The product's decisions for a loaded format: (texel form or -1, target, depth, HasAlpha)."""
    out = (ctypes.c_int * 4)()
    emu().emu_conv_scope(dxgi, out)
    return tuple(out)


def ref_target(loaded):
    """DoReadStart's target and depth (IntelPlugin.cpp:2534-2544, :2591) from the compiled BitsPerColor and IsSRGB."""
    bpc = ref().ref_bits_per_color(loaded)
    if loaded in (95, 96) or bpc > 16:
        return 2, 32
    if bpc > 8:
        return 11, 16
    return (29 if ref().ref_is_srgb(loaded) else 28), 8


# ---- DoReadStart / DoReadContinue ----------------------------------------------------------------------------------------------
def oracle_open(file, options):
    """(metadata, DoReadStart's decisions, every layer) of the reference pipeline: LoadFromDDSMemory (the header cut of
    open_uncompressed_lib; tight rows; X4R4G4B4 with its alpha set), HasAlpha && !IsAlphaAllOpaque, Convert per texel, the layers."""
    m = U.ref_header(file)
    fmt, mips, items = m["format"], m["mip_levels"], m["array_size"]
    _, tb, target, depth, has_alpha = LOADED[fmt]
    n = U.payload_bytes(m["width"], m["height"], mips, items, tb)
    loaded = bytes(np.asarray(file)[m["offset"]:m["offset"] + n])
    if m["conv"] & 0x2:                                            # CONV_FLAGS_NOALPHA: X4R4G4B4
        loaded = set_alpha_4444(loaded)
    buf = np.frombuffer(loaded, np.uint8).copy()
    opaque = not has_alpha or bool(ref().ref_is_alpha_all_opaque(fmt, buf.ctypes.data, m["width"], m["height"], mips, items))
    proxy = B.DdsDesc(m["width"], m["height"], mips, items, 77, 1 if m["cube"] else 0)
    start = U.open_lib.read_start(proxy, opaque, options)
    start["target_dxgi"], start["depth"] = target, depth
    dtype = DTYPES[depth]
    forced = {8: 255, 16: U.ref().ref_convert_to_16bit_255(), 32: 1.0}[depth]
    per_item = U.payload_bytes(m["width"], m["height"], mips, 1, tb)
    layers = []
    for call in range(start["calls"]):
        item, mip = (call, 0) if start["is_cube"] else ((0, call) if start["load_mip_layers"] else (0, 0))     # :2656-2672
        iw, ih = U.level(m["width"], mip), U.level(m["height"], mip)
        at = item * per_item + U.payload_bytes(m["width"], m["height"], mip, 1, tb)
        img = ref_convert(fmt, loaded[at:at + iw * ih * tb]).view(dtype).reshape(ih, iw, 4)
        planes = start["planes"]
        out = np.zeros((m["height"], m["width"], planes), dtype)                                       # :2646
        out[:ih, :iw] = img[..., :planes]
        if start["is_cube"] and start["has_alpha"]:                                                     # :2696, :2711, :2724
            out[:ih, :iw, planes - 1] = forced
        layers.append(out)
    return m, start, layers


info_fields = U.info_fields
