"""Helpers of the display-decompress / preview tests: the reference cut of DirectX::Decompress (oracle/build_ref_preview.py), the CPU
execution of the product's per-block display logic (tests/emu/display_emu.cpp), the input streams, and the preview oracle: the
plug-in's GetCompressedImageForPreview (IntelPlugin.cpp:957-1059, the cross at mip 0) composed from the handwritten oracle's front
end and encoder and the reference's own decompress."""
import ctypes
import functools
import os
import sys

import numpy as np

import itw_testlib as T

B = T.binding
# (source DXGI format, target) pairs of itw_decompress -> (decoder, rule of csrc/display.cuh)
PAIRS = {}
for src, dec in ((71, 71), (77, 77), (80, 80), (83, 83), (98, 98)):
    PAIRS[(src, 28)] = (dec, 0)
    PAIRS[(src, 29)] = (dec, 2)
for src, dec in ((72, 71), (78, 77), (99, 98)):
    PAIRS[(src, 28)] = (dec, 1)
    PAIRS[(src, 29)] = (dec, 0)
for src in (95, 96):
    PAIRS[(src, 28)] = (src, 3)
    PAIRS[(src, 2)] = (src, 4)
NAME = {71: "BC1", 72: "BC1", 77: "BC3", 78: "BC3", 80: "BC4", 83: "BC5", 95: "BC6H", 96: "BC6H", 98: "BC7", 99: "BC7"}


def bpb(src):
    return 8 if src in (71, 72, 80) else 16


def texel(target):
    return 16 if target == 2 else 4


def nblocks(w, h):
    return ((w + 3) // 4) * ((h + 3) // 4)


def empty(w, h, target):
    return np.zeros((h, w, 4), np.float32 if target == 2 else np.uint8)


@functools.lru_cache(None)
def ref():
    """oracle/_ref/libitw_ref_preview.so (None if it could not be built)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_preview
        try:
            path = build_ref_preview.build(verbose=False)
        except FileNotFoundError:
            return None
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_decompress.restype = ctypes.c_int
    lib.ref_decompress.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return lib


def ref_decompress(src, blocks, w, h, target):
    blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
    assert blocks.size == nblocks(w, h) * bpb(src)
    out = empty(w, h, target)
    assert ref().ref_decompress(src, blocks.ctypes.data, w, h, target, out.ctypes.data) == 0
    return out


@functools.lru_cache(None)
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_display_emu.so")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    lib.emu_display.restype = ctypes.c_int
    lib.emu_display.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    for n in ("emu_srgb_in_store", "emu_srgb_out_store"):
        getattr(lib, n).restype = ctypes.c_int
        getattr(lib, n).argtypes = [ctypes.c_float]
    return lib


def emu_decompress(src, blocks, w, h, target):
    dec, rule = PAIRS[(src, target)]
    blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
    out = empty(w, h, target)
    assert emu().emu_display(dec, rule, blocks.ctypes.data, w, h, out.ctypes.data) == 0
    return out


def random_blocks(src, n, seed):
    """Random bits, with the mode field of BC7 / BC6H cycled over every value (reserved ones included)."""
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 256, (n, bpb(src)), dtype=np.uint8)
    if src in (98, 99):
        for i in range(n):
            m = i % 9                                              # 8 = the reserved mode byte 0
            b[i, 0] = 0 if m == 8 else ((int(b[i, 0]) & ~((2 << m) - 1) & 0xFF) | (1 << m))
    elif src in (95, 96):
        b[:, 0] = (b[:, 0] & 0xE0) | (np.arange(n) % 32)
    return b.reshape(-1)


def encoded_streams(src, profiles):
    """(tag, blocks, 64, 64): the oracle encoder's output of the corpus images for each profile."""
    o = T.oracle()
    name = NAME[src]
    corpus = T.corpus_for(name)
    for prof in profiles:
        for key in sorted(corpus)[:3]:
            yield f"{prof}-{key}", T.run(o, name, corpus[key], prof), 64, 64


# ---- the preview oracle -------------------------------------------------------------------------------------------------------
CROSS = ((2, 1), (0, 1), (1, 0), (1, 2), (1, 1), (3, 1))          # +X,-X,+Y,-Y,+Z,-Z, IntelPlugin.cpp:1434


def shown_format(fmt, depth):
    """The format the dialog decompresses from (IntelPlugin.cpp:1024-1049) and its target (:1052-1055)."""
    if depth == 32:
        src = {71: 72, 77: 78, 98: 99}.get(fmt, fmt)
    else:
        src = {72: 71, 78: 77, 99: 98}.get(fmt, fmt)
    return src, (2 if (fmt in (95, 96) and depth == 32) else 28)


def oracle_cross(fmt, faces, flags):
    """The image CompressToScratchImage receives, unpadded: the handwritten oracle's front end of the one face, or of six faces in
    the horizontal cross (cells without a face hold the front end of an all-zero texel with alpha: the plug-in flips and
    normalises the zero-initialised cross after building it, IntelPlugin.cpp:975-1008)."""
    o = T.oracle()
    name = NAME[fmt]
    h, w = faces[0].shape[:2]
    conv = [o.convert_pixels(name, f, flags, pad=False) for f in faces]
    if len(faces) == 1:
        return conv[0]
    zero = np.zeros((1, 1, 4), np.uint8)
    blank = o.convert_pixels(name, zero, (flags | B.FRONT_HAS_ALPHA) & ~B.FRONT_GAMMA, pad=False)[0, 0]
    img = np.empty((3 * h, 4 * w, 4), conv[0].dtype)
    img[:] = blank
    for f, (cx, cy) in zip(conv, CROSS):
        img[cy * h:(cy + 1) * h, cx * w:(cx + 1) * w] = f
    return img


def oracle_preview(fmt, faces, flags, profile):
    """GetCompressedImageForPreview: oracle_cross, pad by edge replication, the handwritten oracle's encoder, DirectX::Decompress
    of the reference.  Returns (display image, compressed bytes)."""
    o = T.oracle()
    img = oracle_cross(fmt, faces, flags)
    H, W = img.shape[:2]
    padded = np.pad(img, ((0, (-H) % 4), (0, (-W) % 4), (0, 0)), mode="edge")
    settings = o.profile(profile) if profile else None
    blocks = o.encode(NAME[fmt], np.ascontiguousarray(padded), settings)
    src, target = shown_format(fmt, faces[0].itemsize * 8)
    return ref_decompress(src, blocks, W, H, target), blocks.size


def document(w, h, planes, depth, seed):
    """A Photoshop document: smooth gradients plus noise, in the element type of its depth."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 7 + y * 3 + 40 * c) % 256 for c in range(planes)], -1).astype(np.float64)
    base = np.clip(base + rng.normal(0, 12, base.shape), 0, 255)
    if depth == 8:
        return base.astype(np.uint8)
    if depth == 16:
        return (base * (32768 / 255)).astype(np.uint16)
    return (base / 255 * 1.25 - 0.05).astype(np.float32)         # a little outside [0, 1] on purpose
