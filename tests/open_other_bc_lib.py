"""Helpers of the tests of the open path for the block-compressed files itw_dds_open does not serve (include/itw_bcn.h section 15): the
reference cut (oracle/build_ref_open_other_bc.py: D3DXDecodeBC2 / BC4S / BC5S, _DecompressBC, _IsAlphaAllOpaqueBC and the compressed
branch of IsAlphaAllOpaque; BitsPerColor, IsSRGB and HasAlpha), the CPU execution of the product's per-block routines
(tests/emu/open_other_bc_emu.cpp), DDS files of every header form, and the open oracle: DoReadStart / DoReadContinue
(IntelPlugin.cpp:2419-2742) with DirectX::Decompress over the reference's own bodies.  The header decoder and the header writer are
open_uncompressed_lib's, DoReadStart's layer decisions open_lib's."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T
import open_lib
import open_uncompressed_lib as U

B = T.binding
OPTIONS = open_lib.OPTIONS

# loaded DXGI format -> (decoder instantiation, bytes per block, target, depth, HasAlpha).  77 is served in its DXT4 form only.
LOADED = {
    70: (71, 8, 28, 8, True), 73: (74, 16, 28, 8, True), 74: (74, 16, 28, 8, True), 75: (74, 16, 29, 8, True),
    76: (77, 16, 28, 8, True), 77: (77, 16, 28, 8, True), 79: (80, 8, 28, 8, False), 81: (81, 8, 28, 8, False),
    82: (83, 16, 28, 8, False), 84: (84, 16, 28, 8, False), 94: (94, 16, 11, 16, False), 97: (98, 16, 28, 8, True),
}
DX10 = sorted(f for f in LOADED if f != 77)
# legacy FourCC forms: name -> (ITW_OBC_*, loaded format)
LEGACY = {"DXT3": (B.OBC_DXT3, 74), "DXT2": (B.OBC_DXT2, 74), "DXT4": (B.OBC_DXT4, 77), "BC4S": (B.OBC_BC4S, 81),
          "BC5S": (B.OBC_BC5S, 84)}
DTYPES = {8: np.uint8, 16: np.uint16}
TEXEL = {28: 4, 29: 4, 11: 8}


def level(v, l):
    return max(1, v >> l)


def image_bytes(w, h, mip, bpb):
    return ((level(w, mip) + 3) // 4) * ((level(h, mip) + 3) // 4) * bpb


def payload_bytes(w, h, mips, items, bpb):
    return items * sum(image_bytes(w, h, m, bpb) for m in range(mips))


def opaque_blocks(fmt, n):
    """`n` blocks of loaded format `fmt` whose texels are all opaque (random colours)."""
    bpb = LOADED[fmt][1]
    b = np.random.default_rng(n).integers(0, 256, (n, bpb), dtype=np.uint8)
    dec = LOADED[fmt][0]
    if dec == 74:
        b[:, :8] = 0xFF                                    # every alpha nibble 15
    elif dec == 77:
        b[:, :8] = 0
        b[:, :2] = 0xFF                                    # a0 = a1 = 255, every index 0
    elif dec == 98:
        b[:, 0] = 0x02                                     # BC7 mode 1: no alpha bits, every texel 255
    elif dec == 71:
        c = b[:, :4].copy().view(np.uint16)
        lo, hi = np.minimum(c[:, 0], c[:, 1]), np.maximum(c[:, 0], c[:, 1])
        hi = np.where(hi == lo, hi + 1, hi).astype(np.uint16)
        lo = np.where(hi == 0, 0, lo).astype(np.uint16)
        b[:, :4] = np.stack([hi, lo], 1).view(np.uint8)  # c0 > c1: four-colour mode, no punch-through
    return b.reshape(-1)


def payload(fmt, w, h, mips, items, seed=0, opaque=False):
    bpb = LOADED[fmt][1]
    n = payload_bytes(w, h, mips, items, bpb)
    if opaque:
        return opaque_blocks(fmt, n // bpb).tobytes()
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def dx10_file(fmt, w, h, mips=1, cube=False, payload_=None, seed=0, opaque=False):
    if payload_ is None:
        payload_ = payload(fmt, w, h, mips, 6 if cube else 1, seed, opaque)
    assert len(payload_) == payload_bytes(w, h, mips, 6 if cube else 1, LOADED[fmt][1])
    return np.frombuffer(U.header(w, h, mips, dx10=(fmt, 3, 0x4 if cube else 0, 1)) + bytes(payload_), np.uint8).copy()


def legacy_file(name, w, h, mips=1, cube=False, payload_=None, seed=0, opaque=False):
    fmt = LEGACY[name][1]
    if payload_ is None:
        payload_ = payload(fmt, w, h, mips, 6 if cube else 1, seed, opaque)
    assert len(payload_) == payload_bytes(w, h, mips, 6 if cube else 1, LOADED[fmt][1])
    pf = (U.FOURCC, U.fourcc(name), 0, 0, 0, 0, 0)
    return np.frombuffer(U.header(w, h, mips, pf, cube, hflags=0x1007 | 0x80000 | (0x20000 if mips > 1 else 0)) + bytes(payload_),
                         np.uint8).copy()


# every header form: (label, loaded format, writer(w, h, mips, cube, payload_=None, seed=0, opaque=False))
FORMS = [(name, LEGACY[name][1], functools.partial(legacy_file, name)) for name in LEGACY] + \
        [(f"DX10-{f}", f, functools.partial(dx10_file, f)) for f in DX10]


# ---- the reference cut and the product's per-block routines -----------------------------------------------------------------------
@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_open_other_bc.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_open_other_bc
        try:
            path = build_ref_open_other_bc.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_obc_decompress.restype = ctypes.c_int
    lib.ref_obc_decompress.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.ref_obc_blocks_opaque.restype = None
    lib.ref_obc_blocks_opaque.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.ref_obc_is_alpha_all_opaque.restype = ctypes.c_int
    lib.ref_obc_is_alpha_all_opaque.argtypes = [ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 4
    for name in ("ref_is_srgb", "ref_has_alpha"):
        getattr(lib, name).restype = ctypes.c_int
        getattr(lib, name).argtypes = [ctypes.c_uint32]
    lib.ref_bits_per_color.restype = ctypes.c_uint
    lib.ref_bits_per_color.argtypes = [ctypes.c_uint32]
    return lib


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_open_other_bc_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_obc_blocks.restype = ctypes.c_int
    lib.emu_obc_blocks.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    lib.emu_obc_blocks_opaque.restype = ctypes.c_int
    lib.emu_obc_blocks_opaque.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.emu_obc_scope.restype = None
    lib.emu_obc_scope.argtypes = [ctypes.c_uint, ctypes.c_void_p]
    return lib


def ref_target(loaded):
    """DoReadStart's target and depth (IntelPlugin.cpp:2534-2544, :2591) from the compiled BitsPerColor and IsSRGB."""
    bpc = ref().ref_bits_per_color(loaded)
    if loaded in (95, 96) or bpc > 16:
        return 2, 32
    if bpc > 8:
        return 11, 16
    return (29 if ref().ref_is_srgb(loaded) else 28), 8


def ref_decompress(source, blocks, w, h, target):
    """DirectX::Decompress of one w x h image of `source` blocks into `target`: h x w x 4 texels (uint8 or uint16)."""
    blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
    out = np.zeros(w * h * TEXEL[target], np.uint8)
    assert ref().ref_obc_decompress(source, blocks.ctypes.data, w, h, target, out.ctypes.data) == 0
    return out.view(np.uint16 if target == 11 else np.uint8).reshape(h, w, 4)


def ref_blocks(source, blocks, target):
    """ref_decompress of `blocks` laid out as one row of 4x4 images: (n, 16, 4) texels in block order."""
    bpb = 8 if source in (70, 71, 79, 80, 81) else 16
    n = len(bytes(blocks)) // bpb
    img = ref_decompress(source, blocks, 4 * n, 4, target)
    return img.reshape(4, n, 4, 4).transpose(1, 0, 2, 3).reshape(n, 16, 4)


def emu_blocks(decoder, blocks):
    """The product's per-block routine on `blocks`: (n, 16, 4) texels."""
    blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
    bpb = 8 if decoder in (71, 80, 81) else 16
    n = blocks.size // bpb
    out = np.zeros(n * 16 * 4 * (2 if decoder == 94 else 1), np.uint8)
    assert emu().emu_obc_blocks(decoder, blocks.ctypes.data, n, out.ctypes.data) == 0
    return out.view(np.uint16 if decoder == 94 else np.uint8).reshape(n, 16, 4)


def blocks_opaque(which, fmt, blocks, cols=4, rows=4):
    """Per block: 1 if its cols x rows texels are all opaque, by the reference's _IsAlphaAllOpaqueBC (which = "ref", fmt a DXGI format)
    or the product's predicate (which = "emu", fmt a scan decoder)."""
    blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
    bpb = 8 if fmt in (70, 71) else 16
    out = np.zeros(blocks.size // bpb, np.uint8)
    if which == "ref":
        ref().ref_obc_blocks_opaque(fmt, blocks.ctypes.data, out.size, cols, rows, out.ctypes.data)
    else:
        assert emu().emu_obc_blocks_opaque(fmt, blocks.ctypes.data, out.size, cols, rows, out.ctypes.data) == 0
    return out


def emu_scope(dxgi):
    """The product's decisions for a loaded format: (decoder or -1, target, depth, HasAlpha, block bytes)."""
    out = (ctypes.c_int * 5)()
    emu().emu_obc_scope(dxgi, out)
    return tuple(out)


# ---- DoReadStart / DoReadContinue ----------------------------------------------------------------------------------------------
def oracle_open(file, options):
    """(metadata, DoReadStart's decisions, every layer) of the reference pipeline: LoadFromDDSMemory's header (open_uncompressed_lib's
    cut), HasAlpha && !IsAlphaAllOpaque (the plug-in's BC1 exclusion names 71 / 72 only), Decompress of each image read, the layers."""
    m = U.ref_header(file)
    fmt, mips, items, w, h = m["format"], m["mip_levels"], m["array_size"], m["width"], m["height"]
    _, bpb, target, depth, _ = LOADED[fmt]
    n = payload_bytes(w, h, mips, items, bpb)
    pay = np.ascontiguousarray(np.asarray(file)[m["offset"]:m["offset"] + n])
    opaque = bool(ref().ref_obc_is_alpha_all_opaque(fmt, pay.ctypes.data, w, h, mips, items))
    has_alpha = bool(ref().ref_has_alpha(fmt)) and not opaque and fmt not in (71, 72)            # :2469-2472
    proxy = B.DdsDesc(w, h, mips, items, 77, 1 if m["cube"] else 0)                              # HasAlpha, not BC1
    start = open_lib.read_start(proxy, not has_alpha, options)
    start["target_dxgi"], start["depth"] = ref_target(fmt)
    per_item = payload_bytes(w, h, mips, 1, bpb)
    layers = []
    for call in range(start["calls"]):
        item, mip = (call, 0) if start["is_cube"] else ((0, call) if start["load_mip_layers"] else (0, 0))     # :2656-2672
        iw, ih = level(w, mip), level(h, mip)
        at = item * per_item + payload_bytes(w, h, mip, 1, bpb)
        img = ref_decompress(fmt, pay[at:at + image_bytes(w, h, mip, bpb)], iw, ih, start["target_dxgi"])
        planes = start["planes"]
        out = np.zeros((h, w, planes), img.dtype)                                                    # :2646
        out[:ih, :iw] = img[..., :planes]
        if start["is_cube"] and start["has_alpha"]:                                                   # :2696, :2724
            out[:ih, :iw, planes - 1] = 255
        layers.append(out)
    return m, start, layers


info_fields = U.info_fields
