"""Helpers of the tests of the expanded open path (include/itw_bcn.h section 16): the reference cut (oracle/build_ref_open_expanded.py:
_DecodeDDSHeader, LoadFromDDSMemory's palette step, _CopyImage's EXPAND rows, _LegacyExpandScanline with a palette), the CPU execution
of the product's per-texel routines (tests/emu/open_exp_emu.cpp), DDS files of the four forms, and the open oracle: DoReadStart /
DoReadContinue (IntelPlugin.cpp:2419-2742) over the reference's own loader, alpha check and, for A4L4, the non-WIC _Convert of
open_converted_lib.  The header writer and DoReadStart's layer decisions are open_uncompressed_lib's."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
import open_converted_lib as C
import open_uncompressed_lib as U

B = T.binding
OPTIONS = U.OPTIONS
PAL8 = U.PAL8
# header form -> (DDS_PIXELFORMAT, ITW_EXP_*, loaded format, bytes per source texel, csrc/open_raw.cuh texel form)
FORMS = {
    "P8": ((PAL8, 0, 8, 0, 0, 0, 0), B.EXP_P8, 28, 1, 24),
    "A8P8": ((PAL8, 0, 16, 0, 0, 0, 0), B.EXP_A8P8, 28, 2, 25),
    "A8R3G3B2": ((U.RGB, 0, 16, 0xe0, 0x1c, 0x03, 0xff00), B.EXP_A8R3G3B2, 28, 2, 23),
    "A4L4": ((U.LUM, 0, 8, 0x0f, 0, 0, 0xf0), B.EXP_A4L4, 115, 1, 22),
}
R3G3B2 = (U.RGB, 0, 8, 0xe0, 0x1c, 0x03, 0)


def has_palette(name):
    return FORMS[name][1] in (B.EXP_P8, B.EXP_A8P8)


def random_palette(seed, alpha=None):
    """256 palette words (R, G, B, alpha bytes); `alpha` forces every alpha byte."""
    pal = np.random.default_rng(seed).integers(0, 1 << 32, 256, dtype=np.uint64).astype(np.uint32)
    if alpha is not None:
        pal = (pal & np.uint32(0x00FFFFFF)) | np.uint32(alpha << 24)
    return pal


def file_of(name, w, h, mips=1, cube=False, payload=None, palette=None, seed=0):
    """A file of form `name` with a random payload (or `payload`) and, for P8 / A8P8, a random palette (or `palette`)."""
    pf, _, _, tb, _ = FORMS[name]
    n = U.payload_bytes(w, h, mips, 6 if cube else 1, tb)
    rng = np.random.default_rng(seed)
    if payload is None:
        payload = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    assert len(payload) == n
    pal = b""
    if has_palette(name):
        pal = (random_palette(seed + 1) if palette is None else np.asarray(palette, np.uint32)).astype("<u4").tobytes()
    return np.frombuffer(U.header(w, h, mips, pf, cube) + pal + bytes(payload), np.uint8).copy()


WRITERS = [(name, functools.partial(file_of, name)) for name in FORMS]


# ---- the reference cut and the product's per-texel routines ---------------------------------------------------------------------
@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_open_expanded.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_open_expanded
        try:
            path = build_ref_open_expanded.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_load_expanded.restype = ctypes.c_longlong
    lib.ref_load_expanded.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
    lib.ref_expand_texels.restype = ctypes.c_int
    lib.ref_expand_texels.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def refs_ready():
    return ref() is not None and C.ref() is not None and U.ref() is not None


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_open_exp_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_exp_texels.restype = ctypes.c_int
    lib.emu_exp_texels.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int,
                                   ctypes.c_void_p]
    lib.emu_exp_alpha_below.restype = ctypes.c_int
    lib.emu_exp_alpha_below.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32,
                                        ctypes.c_void_p]
    lib.emu_exp_scope.restype = None
    lib.emu_exp_scope.argtypes = [ctypes.c_int, ctypes.c_void_p]
    return lib


def _buf(a, dtype=np.uint8):
    return np.ascontiguousarray(np.frombuffer(bytes(a), dtype))


def conv_flags(name):
    """The g_LegacyDDSMap convFlags of a form, from the compiled _DecodeDDSHeader."""
    return U.ref_header(file_of(name, 1, 1))["conv"]


def ref_expand(name, src, pal=None):
    """_LegacyExpandScanline on the source texels `src` of form `name`: the loaded texels (28: 4 bytes, 115: 2 bytes each)."""
    _, _, loaded, tb, _ = FORMS[name]
    src = _buf(src)
    n = src.size // tb
    out = np.zeros(n * (2 if loaded == 115 else 4), np.uint8)
    p = None if pal is None else _buf(np.asarray(pal, np.uint32).astype("<u4").tobytes(), np.uint32)
    assert ref().ref_expand_texels(conv_flags(name), loaded, src.ctypes.data, n, None if p is None else p.ctypes.data, out.ctypes.data) == 0
    return out


def ref_texels(name, src, pal=None):
    """The reference's layer texels (R8G8B8A8_UNORM) of source texels: the expansion, and for A4L4 _Convert 115 -> 28."""
    loaded = ref_expand(name, src, pal)
    return C.ref_convert(115, loaded) if FORMS[name][2] == 115 else loaded


def emu_texels(name, planes, src, pal=None, force=False):
    src = _buf(src)
    n = src.size // FORMS[name][3]
    out = np.zeros(n * planes, np.uint8)
    p = None if pal is None else _buf(np.asarray(pal, np.uint32).astype("<u4").tobytes(), np.uint32)
    assert emu().emu_exp_texels(FORMS[name][4], planes, src.ctypes.data, n, None if p is None else p.ctypes.data, int(force),
                                out.ctypes.data) == 0
    return out


def emu_below(name, src, slot, pal=None, fill=0xFFFF):
    """The scan's predicate on each source texel at slot `slot` of its word, `fill` in the other slots."""
    src = _buf(src)
    n = src.size // FORMS[name][3]
    out = np.zeros(n, np.uint8)
    p = None if pal is None else _buf(np.asarray(pal, np.uint32).astype("<u4").tobytes(), np.uint32)
    assert emu().emu_exp_alpha_below(FORMS[name][4], src.ctypes.data, n, slot, None if p is None else p.ctypes.data, fill,
                                     out.ctypes.data) == 0
    return out


def emu_scope(form):
    """The product's decisions for a header form: (texel form, loaded format, palette, source bytes per texel)."""
    out = (ctypes.c_int * 4)()
    emu().emu_exp_scope(form, out)
    return tuple(out)


def ref_opaque(loaded, texels):
    """The cut IsAlphaAllOpaque branch of the loaded format (28 or 115) on each loaded texel: 1 when opaque."""
    src = _buf(texels)
    n = src.size // (4 if loaded == 28 else 2)
    out = np.zeros(n, np.uint8)
    (U.ref() if loaded == 28 else C.ref()).ref_texels_opaque(loaded, src.ctypes.data, n, out.ctypes.data)
    return out


# ---- DoReadStart / DoReadContinue ----------------------------------------------------------------------------------------------
def ref_load(file):
    """(metadata, the loaded payload as LoadFromDDSMemory leaves it), or (None, HRESULT) when it fails."""
    file = _buf(file)
    m = U.ref_header(file)
    n = 0 if m is None else U.payload_bytes(m["width"], m["height"], m["mip_levels"], m["array_size"], 2 if m["format"] == 115 else 4)
    out = np.zeros(max(n, 1), np.uint8)
    meta = (ctypes.c_uint64 * 8)()
    got = ref().ref_load_expanded(file.ctypes.data, file.size, out.ctypes.data, meta)
    if got < 0:
        return None, got
    keys = ("width", "height", "mip_levels", "array_size", "format", "cube", "conv", "offset")
    m = dict(zip(keys, [int(v) for v in meta]))
    assert got == n, (got, n)
    return m, out[:n]


def oracle_open(file, options):
    """(metadata, DoReadStart's decisions, every layer) of the reference pipeline: LoadFromDDSMemory with the palette, HasAlpha &&
    !IsAlphaAllOpaque on the loaded format, Convert 115 -> 28 for A4L4, the layers."""
    m, loaded = ref_load(file)
    fmt, mips, items = m["format"], m["mip_levels"], m["array_size"]
    lb = 2 if fmt == 115 else 4
    opaque = bool((U.ref() if fmt == 28 else C.ref()).ref_is_alpha_all_opaque(fmt, loaded.ctypes.data, m["width"], m["height"], mips,
                                                                                 items))
    proxy = B.DdsDesc(m["width"], m["height"], mips, items, 77, 1 if m["cube"] else 0)
    start = U.open_lib.read_start(proxy, opaque, options)
    start["target_dxgi"], start["depth"] = 28, 8
    per_item = U.payload_bytes(m["width"], m["height"], mips, 1, lb)
    layers = []
    for call in range(start["calls"]):
        item, mip = (call, 0) if start["is_cube"] else ((0, call) if start["load_mip_layers"] else (0, 0))     # :2656-2672
        iw, ih = U.level(m["width"], mip), U.level(m["height"], mip)
        at = item * per_item + U.payload_bytes(m["width"], m["height"], mip, 1, lb)
        img = loaded[at:at + iw * ih * lb]
        if fmt == 115:
            img = C.ref_convert(115, img)
        img = img.reshape(ih, iw, 4)
        planes = start["planes"]
        out = np.zeros((m["height"], m["width"], planes), np.uint8)                                     # :2646
        out[:ih, :iw] = img[..., :planes]
        if start["is_cube"] and start["has_alpha"]:                                                     # :2696, :2724
            out[:ih, :iw, planes - 1] = 255
        layers.append(out)
    return m, start, layers


info_fields = U.info_fields
