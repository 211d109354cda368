"""Helpers of the tests of the uncompressed open path (include/itw_bcn.h section 13): the reference cut (oracle/build_ref_open_uncompressed.py:
_DecodeDDSHeader, _CopyImage's row paths, IsAlphaAllOpaque's non-compressed branch, ConvertTo16Bit), the CPU execution of the product's
per-texel routines (tests/emu/open_raw_emu.cpp), DDS files of every header form, and the open oracle: DoReadStart / DoReadContinue
(IntelPlugin.cpp:2419-2742) over the reference's own loader and alpha check.  DoReadStart's layer and plane decisions are open_lib.read_start's,
with its target table extended by the four formats that are their own target."""
import ctypes
import functools
import os
import struct
import sys

import numpy as np

import itw_testlib as T
import open_lib

B = T.binding
OPTIONS = open_lib.OPTIONS
# DoReadStart's target and Photoshop depth of each loaded format that needs no conversion (:2534-2544, :2591)
TARGETS = {28: (28, 8), 29: (29, 8), 11: (11, 16), 2: (2, 32)}
DTYPES = {28: np.uint8, 29: np.uint8, 11: np.uint16, 2: np.float32}
TEXEL = {28: 4, 29: 4, 11: 8, 2: 16}

# legacy DDS_PIXELFORMAT (flags, fourcc, bits, r, g, b, a) of DDS.h's DDSPF_* and g_LegacyDDSMap's inline entries
RGBA, RGB, FOURCC, LUM, LUMA, ALPHA, PAL8 = 0x41, 0x40, 0x4, 0x20000, 0x20001, 0x2, 0x20
PF = {
    "A8B8G8R8": (RGBA, 0, 32, 0xff, 0xff00, 0xff0000, 0xff000000),
    "X8B8G8R8": (RGB, 0, 32, 0xff, 0xff00, 0xff0000, 0),
    "R8G8B8": (RGB, 0, 24, 0xff0000, 0xff00, 0xff, 0),
    "A16B16G16R16": (FOURCC, 36, 0, 0, 0, 0, 0),
    "A32B32G32R32F": (FOURCC, 116, 0, 0, 0, 0, 0),
}
SOURCES = {"A8B8G8R8": B.RAW_A8B8G8R8, "X8B8G8R8": B.RAW_X8B8G8R8, "R8G8B8": B.RAW_R8G8B8, "A16B16G16R16": B.RAW_A16B16G16R16,
           "A32B32G32R32F": B.RAW_A32B32G32R32F}
SRC_BYTES = {"A8B8G8R8": 4, "X8B8G8R8": 4, "R8G8B8": 3, "A16B16G16R16": 8, "A32B32G32R32F": 16}
# csrc/open_raw.cuh's texel forms
KIND = {"A8B8G8R8": 0, "X8B8G8R8": 1, "R8G8B8": 2, "A16B16G16R16": 3, "A32B32G32R32F": 4}


def fourcc(s):
    return struct.unpack("<I", s.encode())[0]


def level(v, l):
    return max(1, v >> l)


def full_chain(w, h):
    return max(w, h).bit_length()


def header(w, h, mips=1, pf=PF["A8B8G8R8"], cube=False, caps2=None, hflags=None, dx10=None):
    """magic + DDS_HEADER (+ DDS_HEADER_DXT10 when `dx10` = (dxgi, dimension, misc, array_size)) as DDS.h lays them out."""
    flags = 0x1007 | (0x20000 if mips > 1 else 0) | 0x8 if hflags is None else hflags
    caps = 0x1000 | (0x400008 if mips > 1 else 0) | (0x8 if cube else 0)
    if caps2 is None:
        caps2 = 0xFE00 if cube else 0
    if dx10 is not None:
        pf = (FOURCC, fourcc("DX10"), 0, 0, 0, 0, 0)
    head = struct.pack("<4s7I", b"DDS ", 124, flags, h, w, 0, 0, mips) + b"\0" * 44
    head += struct.pack("<8I", 32, *pf) + struct.pack("<5I", caps, caps2, 0, 0, 0)
    assert len(head) == 128
    if dx10 is not None:
        head += struct.pack("<5I", *dx10, 0)
    return head


def payload_bytes(w, h, mips, items, texel):
    return items * sum(level(w, m) * level(h, m) * texel for m in range(mips))


def legacy_file(name, w, h, mips=1, cube=False, payload=None, seed=0):
    """A file of legacy form `name` (PF) with a random payload (or `payload`)."""
    n = payload_bytes(w, h, mips, 6 if cube else 1, SRC_BYTES[name])
    if payload is None:
        payload = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()
    assert len(payload) == n
    return np.frombuffer(header(w, h, mips, PF[name], cube) + bytes(payload), np.uint8).copy()


def dx10_file(fmt, w, h, mips=1, cube=False, payload=None, seed=0):
    n = payload_bytes(w, h, mips, 6 if cube else 1, TEXEL[fmt])
    if payload is None:
        payload = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()
    assert len(payload) == n
    return np.frombuffer(header(w, h, mips, dx10=(fmt, 3, 0x4 if cube else 0, 1)) + bytes(payload), np.uint8).copy()


# ---- the reference cut and the product's per-texel routines ---------------------------------------------------------------------
@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_open_uncompressed.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_open_uncompressed
        try:
            path = build_ref_open_uncompressed.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_decode_header.restype = ctypes.c_long
    lib.ref_decode_header.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.ref_copy_image.restype = ctypes.c_longlong
    lib.ref_copy_image.argtypes = [ctypes.c_void_p] + [ctypes.c_uint32] * 6 + [ctypes.c_void_p]
    lib.ref_is_alpha_all_opaque.restype = ctypes.c_int
    lib.ref_is_alpha_all_opaque.argtypes = [ctypes.c_uint32, ctypes.c_void_p] + [ctypes.c_uint32] * 4
    lib.ref_texels_opaque.restype = None
    lib.ref_texels_opaque.argtypes = [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    lib.ref_convert_to_16bit_255.restype = ctypes.c_uint
    return lib


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_open_raw_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_raw_texels.restype = ctypes.c_int
    lib.emu_raw_texels.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]
    lib.emu_raw_alpha_below.restype = ctypes.c_int
    lib.emu_raw_alpha_below.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    return lib


def ref_header(file):
    """_DecodeDDSHeader(DDS_FLAGS_NONE): dict of the metadata, or None when it fails."""
    file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
    out = (ctypes.c_uint64 * 9)()
    if ref().ref_decode_header(file.ctypes.data, file.size, out) != 0:
        return None
    keys = ("width", "height", "mip_levels", "array_size", "format", "cube", "conv", "dimension", "offset")
    return dict(zip(keys, [int(v) for v in out]))


def ref_load(file):
    """(metadata, the loaded payload as LoadFromDDSMemory leaves it: item-major, mip-minor, tight rows of the loaded format)."""
    m = ref_header(file)
    file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
    n = payload_bytes(m["width"], m["height"], m["mip_levels"], m["array_size"], TEXEL[m["format"]])
    out = np.zeros(n, np.uint8)
    got = ref().ref_copy_image(file.ctypes.data + m["offset"], m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"],
                               m["conv"], out.ctypes.data)
    assert got == n, (got, n)
    return m, out


# ---- DoReadStart / DoReadContinue ----------------------------------------------------------------------------------------------
def read_start(m, all_opaque, options):
    """open_lib.read_start's decisions for a loaded format whose HasAlpha holds (a BC3 stand-in: HasAlpha, not BC1), with the
    target table extended."""
    proxy = B.DdsDesc(m["width"], m["height"], m["mip_levels"], m["array_size"], 77, 1 if m["cube"] else 0)
    start = open_lib.read_start(proxy, all_opaque, options)
    start["target_dxgi"], start["depth"] = TARGETS[m["format"]]
    return start


def oracle_open(file, options):
    """(metadata, DoReadStart's decisions, every layer) of the reference pipeline."""
    m, loaded = ref_load(file)
    opaque = bool(ref().ref_is_alpha_all_opaque(m["format"], loaded.ctypes.data, m["width"], m["height"], m["mip_levels"],
                                                m["array_size"]))
    start = read_start(m, opaque, options)
    fmt, mips = m["format"], m["mip_levels"]
    texel = TEXEL[fmt]
    per_item = payload_bytes(m["width"], m["height"], mips, 1, texel)
    forced = {8: 255, 16: ref().ref_convert_to_16bit_255(), 32: 1.0}[start["depth"]]
    layers = []
    for call in range(start["calls"]):
        item, mip = (call, 0) if start["is_cube"] else ((0, call) if start["load_mip_layers"] else (0, 0))     # :2656-2672
        iw, ih = level(m["width"], mip), level(m["height"], mip)
        at = item * per_item + payload_bytes(m["width"], m["height"], mip, 1, texel)
        img = loaded[at:at + iw * ih * texel].view(DTYPES[fmt]).reshape(ih, iw, 4)
        planes = start["planes"]
        out = np.zeros((m["height"], m["width"], planes), DTYPES[fmt])                                 # :2646
        out[:ih, :iw] = img[..., :planes]
        if start["is_cube"] and start["has_alpha"]:                                                     # :2696, :2711, :2724
            out[:ih, :iw, planes - 1] = forced
        layers.append(out)
    return m, start, layers


def info_fields(info):
    return {k: getattr(info, k) for k in ("has_alpha", "has_mips", "ask_user", "layers", "calls", "planes", "depth", "width", "height",
                                          "target_dxgi")}


def emu_texels(kind, planes, src, force):
    """The product's per-texel rule on host texels (emulation): layer texels as bytes."""
    src = np.ascontiguousarray(np.frombuffer(bytes(src), np.uint8))
    n = src.size // [4, 4, 3, 8, 16][kind]
    out = np.zeros(n * planes * [1, 1, 1, 2, 4][kind], np.uint8)
    assert emu().emu_raw_texels(kind, planes, src.ctypes.data, n, int(force), out.ctypes.data) == 0
    return out
