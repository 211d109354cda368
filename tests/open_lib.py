"""Helpers of the open-path tests: the reference cut of the alpha check (oracle/build_ref_open.py), the CPU execution of the product's
per-block alpha predicate (tests/emu/open_emu.cpp), DDS files built from chosen blocks, and the open oracle: the plug-in's
DoReadStart decisions and DoReadContinue copy loop (IntelPlugin.cpp:2419-2742), restated here because they are Photoshop glue that
cannot be compiled, over the reference's own IsAlphaAllOpaque and DirectX::Decompress."""
import ctypes
import functools
import os
import struct
import sys

import numpy as np

import itw_testlib as T
import preview_lib as P

B = T.binding
FORMATS = (71, 72, 77, 78, 80, 83, 95, 96, 98, 99)
OPTIONS = (0, B.OPEN_SEPARATE_ALPHA, B.OPEN_MIPS, B.OPEN_SEPARATE_ALPHA | B.OPEN_MIPS)


def bpb(fmt):
    return 8 if fmt in (71, 72, 80) else 16


def level(v, l):
    return max(1, v >> l)


def image_bytes(desc, mip):
    return ((level(desc.width, mip) + 3) // 4) * ((level(desc.height, mip) + 3) // 4) * bpb(desc.dxgi_format)


def payload_bytes(desc):
    return desc.array_size * sum(image_bytes(desc, m) for m in range(desc.mip_levels))


def image_slice(file, desc, item, mip):
    """The blocks of image (item, mip): the payload ends the file, item-major, mip-minor (DirectXTexDDS.cpp:1676-1720)."""
    start = len(file) - payload_bytes(desc)
    per_item = sum(image_bytes(desc, m) for m in range(desc.mip_levels))
    at = start + item * per_item + sum(image_bytes(desc, m) for m in range(mip))
    return np.frombuffer(bytes(file[at:at + image_bytes(desc, mip)]), np.uint8)


def desc(w, h, fmt, mips=1, cube=False):
    return B.DdsDesc(w, h, mips, 6 if cube else 1, fmt, 1 if cube else 0)


def full_chain(w, h):
    return max(w, h).bit_length()


def make_file(d, payload):
    """Header (the product's itw_dds_write_header, pinned by tests/test_dds.py) + `payload`."""
    lib = T.product().lib
    head = np.zeros(148, np.uint8)
    n = lib.itw_dds_write_header(ctypes.byref(d), head.ctypes.data, head.size)
    assert n and len(payload) == payload_bytes(d)
    return np.concatenate([head[:n], np.frombuffer(bytes(payload), np.uint8)])


def legacy_file(fourcc, w, h, mips, payload, cube=False):
    """A DDS file with a legacy FourCC header as other tools write it (DDS.h:207-223): 'DXT1', 'DXT5', 'ATI1', 'ATI2', 'BC4U', 'BC5U'."""
    flags = 0x1007 | 0x80000 | (0x20000 if mips > 1 else 0)
    caps = 0x1000 | (0x400008 if mips > 1 else 0) | (0x8 if cube else 0)
    caps2 = 0xFE00 if cube else 0
    pf = struct.pack("<II4s5I", 32, 0x4, fourcc.encode(), 0, 0, 0, 0, 0)
    head = struct.pack("<4s7I", b"DDS ", 124, flags, h, w, 0, 0, mips) + b"\0" * 44 + pf + struct.pack("<5I", caps, caps2, 0, 0, 0)
    assert len(head) == 128
    return np.frombuffer(head + bytes(payload), np.uint8).copy()


def dx10_file(d, payload):
    """A DDS file with the 'DX10' extension header (DDS.h:225-232) for ANY format, as texconv -dx10 and DirectXTex's
    DDS_FLAGS_FORCE_DX10_EXT write it: the payload starts at byte 148 also where the library itself writes a 128-byte legacy header."""
    mips, cube = d.mip_levels, bool(d.is_cubemap)
    head = bytearray(legacy_file("DX10", d.width, d.height, mips, b"", cube).tobytes())
    head += struct.pack("<5I", d.dxgi_format, 3, 0x4 if cube else 0, d.array_size // 6 if cube else d.array_size, 0)
    assert len(head) == 148 and len(payload) == payload_bytes(d)
    return np.frombuffer(bytes(head) + bytes(payload), np.uint8).copy()


def padding_only_block(fmt, cols, rows, inside_bad=False):
    """A BC3 (77/78) or BC7 (98/99) block that is transparent only outside its first cols x rows texels (also at texel 0 when
    inside_bad)."""
    inside = [(k & 3) < cols and (k >> 2) < rows for k in range(16)]
    if fmt in (77, 78):
        idx = [0 if ins else 1 for ins in inside]                  # a0 = 255 opaque, a1 = 0 transparent
        if inside_bad:
            idx[0] = 1
        return bc3_block(255, 0, idx)
    idx = [0 if ins else 15 for ins in inside]
    if inside_bad:
        idx[0] = 7                                                 # texel 0 is an anchor: three bits
    return bc7_mode6(255, 0, idx)


def padding_only_payload(d):
    """Every image of `d` (item-major, mip-minor) made of padding_only_block: opaque inside every image, transparent in the padding
    of its ragged edge blocks."""
    images = []
    for _ in range(d.array_size):
        for m in range(d.mip_levels):
            lw, lh = level(d.width, m), level(d.height, m)
            bw, bh = (lw + 3) // 4, (lh + 3) // 4
            blk = np.zeros((bh, bw, 16), np.uint8)
            for by in range(bh):
                for bx in range(bw):
                    blk[by, bx] = padding_only_block(d.dxgi_format, min(4, lw - 4 * bx), min(4, lh - 4 * by))
            images.append(blk.reshape(-1))
    return np.concatenate(images)


# ---- the reference's alpha check and the product's per-block predicate ---------------------------------------------------------
@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_open.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_open
        try:
            path = build_ref_open.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_is_alpha_all_opaque.restype = ctypes.c_int
    lib.ref_is_alpha_all_opaque.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.ref_blocks_alpha_opaque.restype = None
    lib.ref_blocks_alpha_opaque.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return lib


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_open_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_blocks_alpha_opaque.restype = ctypes.c_int
    lib.emu_blocks_alpha_opaque.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return lib


def blocks_opaque(which, fmt, blocks, cols=4, rows=4):
    """Per 16-byte block: 1 if its cols x rows texels are all opaque, by the reference (`which` = ref()) or the emulation (emu())."""
    blocks = np.ascontiguousarray(blocks, np.uint8).reshape(-1, 16)
    out = np.zeros(len(blocks), np.uint8)
    fn = which.ref_blocks_alpha_opaque if hasattr(which, "ref_blocks_alpha_opaque") else which.emu_blocks_alpha_opaque
    fn(fmt, blocks.ctypes.data, len(blocks), cols, rows, out.ctypes.data)
    return out


def ref_all_opaque(file, d):
    payload = np.ascontiguousarray(np.frombuffer(bytes(file[len(file) - payload_bytes(d):]), np.uint8))
    return bool(ref().ref_is_alpha_all_opaque(d.dxgi_format, payload.ctypes.data, d.width, d.height, d.mip_levels, d.array_size))


# ---- DoReadStart (IntelPlugin.cpp:2461-2602) ---------------------------------------------------------------------------------
def read_start(d, all_opaque, options):
    """The plug-in's decisions for a texture of description `d` whose ScratchImage::IsAlphaAllOpaque() is `all_opaque`, with the
    load dialog's answers (or the batch values) `options`."""
    fmt = d.dxgi_format
    has_alpha = fmt in (71, 72, 77, 78, 98, 99) and not all_opaque and fmt not in (71, 72)      # :2469-2472
    loadinfo_has_alpha = has_alpha
    has_mips = d.mip_levels > 1                                                                   # :2475
    separate = bool(options & B.OPEN_SEPARATE_ALPHA)                                             # :2477-2478 (batch) or :2498
    load_mips = bool(options & B.OPEN_MIPS)
    cube = d.array_size == 6                                                                      # :2479
    if cube:                                                                                      # :2482-2486
        has_alpha = has_mips = separate = False
    ask_user = has_alpha or has_mips                                                              # :2490
    layers, is_cube, load_mip_layers = 0, False, False
    if cube:                                                                                      # :2511-2525
        is_cube, layers = True, 6
    elif has_mips and load_mips:
        load_mip_layers, layers = True, d.mip_levels
    if not separate and has_alpha and layers == 0:                                                # :2529-2532
        layers = 1
    target = 2 if fmt in (95, 96) else (29 if fmt in (72, 78, 99) else 28)                       # :2534-2544
    depth = 32 if target == 2 else 8                                                              # :2591
    planes = (4 if has_alpha else 3) if separate else (4 if layers > 0 else 3)                    # :2593-2602
    return dict(has_alpha=loadinfo_has_alpha, has_mips=d.mip_levels > 1, ask_user=ask_user, layers=layers, calls=max(1, layers),
                planes=planes, depth=depth, width=d.width, height=d.height, target_dxgi=target, is_cube=is_cube,
                load_mip_layers=load_mip_layers)


def info_fields(info):
    return {k: getattr(info, k) for k in ("has_alpha", "has_mips", "ask_user", "layers", "calls", "planes", "depth", "width", "height",
                                          "target_dxgi")}


# ---- DoReadContinue (IntelPlugin.cpp:2614-2742) ------------------------------------------------------------------------------
def read_continue(file, d, start, call):
    """Layer `call` as Photoshop receives it: a zeroed height x width x planes buffer, the decompressed image copied into its top-left
    corner, the last plane forced to 255 / 1.0f for a cube map with alpha."""
    if start["is_cube"]:                                                                          # :2656-2672
        item, mip = call, 0
    elif start["load_mip_layers"]:
        item, mip = 0, call
    else:
        item, mip = 0, 0
    iw, ih = level(d.width, mip), level(d.height, mip)
    img = P.ref_decompress(d.dxgi_format, image_slice(file, d, item, mip), iw, ih, start["target_dxgi"])
    planes = start["planes"]
    out = np.zeros((d.height, d.width, planes), img.dtype)                                        # :2646
    out[:ih, :iw] = img[..., :planes]
    if start["is_cube"] and start["has_alpha"]:                                                   # :2696, :2724
        out[:ih, :iw, planes - 1] = 1.0 if img.dtype == np.float32 else 255
    return out


def oracle_open(file, d, options):
    """(DoReadStart's decisions, every layer) of the reference pipeline: cut alpha check + ref_decompress + the restated copy."""
    start = read_start(d, ref_all_opaque(file, d), options)
    return start, [read_continue(file, d, start, c) for c in range(start["calls"])]


# ---- blocks with chosen alpha ---------------------------------------------------------------------------------------------------
def pack_bits(fields):
    """LSB-first bit packer: [(value, nbits), ...] -> 16 bytes."""
    v, pos = 0, 0
    for val, n in fields:
        assert 0 <= val < (1 << n), (val, n)
        v |= int(val) << pos
        pos += n
    assert pos == 128, pos
    return np.frombuffer(v.to_bytes(16, "little"), np.uint8)


def bc7_mode6(alpha0, alpha1, indices, rgb=(40, 80, 120)):
    """Mode 6: 7-bit RGBA endpoints + one p-bit each (so 8-bit endpoints), 4-bit indices (texel 0: 3 bits)."""
    a0, p0 = alpha0 >> 1, alpha0 & 1
    a1, p1 = alpha1 >> 1, alpha1 & 1
    f = [(1 << 6, 7)]
    for c in rgb:
        f += [(c >> 1, 7), (c >> 1, 7)]
    f += [(a0, 7), (a1, 7), (p0, 1), (p1, 1)]
    f += [(indices[0] & 7, 3)] + [(int(q), 4) for q in indices[1:]]
    return pack_bits(f)


def bc7_mode5(alpha0, alpha1, aidx, rot=0, rgb=(40, 80, 120)):
    """Mode 5: rotation, 7-bit RGB and 8-bit alpha endpoints, 2-bit colour and alpha indices (texel 0: 1 bit)."""
    f = [(1 << 5, 6), (rot, 2)]
    for c in rgb:
        f += [(c >> 1, 7), (c >> 1, 7)]
    f += [(alpha0, 8), (alpha1, 8)]
    f += [(0, 1)] + [(1, 2)] * 15
    f += [(aidx[0] & 1, 1)] + [(int(q), 2) for q in aidx[1:]]
    return pack_bits(f)


def bc7_mode7(a, p, idx):
    """Mode 7, shape 0 (second anchor texel 15): 5-bit RGBA endpoints (four of them) + one p-bit each, 2-bit indices (anchors 1 bit)."""
    f = [(1 << 7, 8), (0, 6)]
    for _ in range(3):
        f += [(17, 5)] * 4
    f += [(int(v), 5) for v in a] + [(int(v), 1) for v in p]
    f += [(int(q) & (1 if k in (0, 15) else 3), 1 if k in (0, 15) else 2) for k, q in enumerate(idx)]
    return pack_bits(f)


def bc3_block(a0, a1, indices, colour=(0xF800, 0x001F, 0)):
    """A BC3 block: alpha endpoints, sixteen 3-bit alpha indices, then a BC1 colour half."""
    bits = 0
    for k, q in enumerate(indices):
        bits |= int(q) << (3 * k)
    head = bytes([a0, a1]) + bits.to_bytes(6, "little")
    return np.frombuffer(head + struct.pack("<HHI", colour[0], colour[1], colour[2]), np.uint8)
