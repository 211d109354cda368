"""Mip maps from layers (include/itw_bcn.h section 6, itw_dds_encode_layers): the save dialog's FROM_LAYERS option.

CPU: (1) the oracle restatement (oracle_copy_layer, oracle/itw_oracle_layers.cpp) against the reference's OWN bodies of
CopyLayersIntoMipMaps / CopyFromLayerChannelIntoImage / FillLayerDataToWhite (oracle/_ref/libitw_ref_layers.so, cut by
oracle/build_ref_layers.py), driven as DoWriteDDS drives them, and against committed digests of those bodies; (2) the kernel's
per-texel routine (layer_texel in csrc/frontend.cuh, through tests/emu) against the oracle.
GPU: itw_dds_encode_layers against the oracle pipeline composite convert -> layer 0 -> flip -> chain -> layers >= 1 ->
normalise -> pad -> encode; against itw_dds_encode_pixels where the two must agree; a round trip through the open path;
device-memory planes; rejections."""
import ctypes
import functools
import hashlib
import itertools
import json
import os
import sys

import numpy as np
import pytest

import itw_testlib as T

B = T.binding
HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"BC7": 98, "BC5": 83, "BC6H": 95}
SPECIALS32 = np.array([0.0, -0.0, 1.0, -1.0, 0.5, 1.0000001, 2.0, 1e-8, 65504.0, 70000.0, 1e9, -5.0, np.inf, -np.inf, np.nan,
                       0.21404114, 1 / 255], np.float32)
SPECIALS16 = np.array([0, 1, 2, 32768, 32767, 40000, 65535, 128, 15360], np.uint16)


def lvl(v, l):
    return max(1, v >> l)


def full_levels(w, h):
    return max(w, h).bit_length()


def plane(depth, w, h, rng, specials=True):
    """One document-sized channel of `depth` bits, with the 16- and 32-bit specials the front-end tests use."""
    if depth == 8:
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if depth == 16:
        a = rng.integers(0, 32769, (h, w), dtype=np.uint16)
        if specials:
            a.reshape(-1)[:SPECIALS16.size] = SPECIALS16[:a.size]
        return a
    a = (rng.random((h, w), dtype=np.float32) * 1.2 - 0.1).astype(np.float32)
    if specials:
        a.reshape(-1)[:SPECIALS32.size] = SPECIALS32[:a.size]
    return a


def make_layers(depth, w, h, count, channels, alpha, seed, specials=True):
    """`count` layers of `channels` channels; alpha planes when `alpha` (else None = white)."""
    rng = np.random.default_rng(seed)
    return [([plane(depth, w, h, rng, specials) for _ in range(channels)], plane(depth, w, h, rng, specials) if alpha else None)
            for _ in range(count)]


def before_levels(hdr, w, h, levels, seed):
    """What the scratch image holds before a copy (the composite's level 0, generated levels): random texels."""
    rng = np.random.default_rng(seed)
    if hdr:
        return [rng.integers(0, 0x7C00, (lvl(h, l), lvl(w, l), 4), dtype=np.uint16) for l in range(levels)]
    return [rng.integers(0, 256, (lvl(h, l), lvl(w, l), 4), dtype=np.uint8) for l in range(levels)]


def _ptrs(channels, alpha):
    arr = (ctypes.c_void_p * 4)()
    for c, p in enumerate(channels):
        arr[c] = p.ctypes.data
    arr[3] = alpha.ctypes.data if alpha is not None else None
    return arr


@functools.lru_cache(None)
def layers_oracle():
    """oracle/libitw_oracle_layers.so (oracle/build_oracle_layers.py; rebuilt only when stale)."""
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_oracle_layers
        path = build_oracle_layers.build(verbose=False)
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    f = lib.oracle_copy_layer
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                  ctypes.c_void_p, ctypes.c_int, ctypes.c_uint]
    return lib


def oracle_copy(level, depth, doc_w, layer, has_alpha, flip=0):
    """oracle_copy_layer on one tight level (in place)."""
    channels, alpha = layer
    f = layers_oracle().oracle_copy_layer
    p = _ptrs(channels, alpha)
    assert level.flags.c_contiguous
    assert f(int(level.dtype == np.uint16), level.ctypes.data, level.shape[1], level.shape[0], depth, doc_w, p, len(channels),
             p[3], int(has_alpha), flip) == 0
    return level


def oracle_layers_into(levels, depth, doc_w, layers, has_alpha, flip0=0):
    """DoWriteDDS's two CopyLayersIntoMipMaps calls on a chain that already exists (flip on level 0 only)."""
    for l in range(min(len(layers), len(levels))):
        oracle_copy(levels[l], depth, doc_w, layers[l], has_alpha, flip0 if l == 0 else 0)
    return levels


@pytest.fixture(scope="module")
def ref_layers():
    sys.path.insert(0, os.path.join(T.ROOT, "oracle"))
    try:
        import build_ref_layers
        try:
            path = build_ref_layers.build(verbose=False)
        except FileNotFoundError:
            pytest.skip("reference layer copy not built (no reference tree and no prebuilt oracle/_ref)")
    finally:
        sys.path.pop(0)
    lib = ctypes.CDLL(path)
    lib.ref_copy_layers_into_mips.restype = ctypes.c_int
    return lib


def ref_copy(lib, fmt, depth, w, h, images, layers, has_alpha, start, end, mask_slot=0):
    n = len(layers)
    planes = (ctypes.c_void_p * (4 * n))()
    for i, (channels, alpha) in enumerate(layers):
        for c, p in enumerate(channels):
            planes[4 * i + c] = p.ctypes.data
        planes[4 * i + 3] = alpha.ctypes.data if alpha is not None else None
    rows = (ctypes.c_longlong * n)(*[w * depth // 8] * n)
    counts = (ctypes.c_int * n)(*[len(c) for c, _ in layers])
    slots = (ctypes.c_int * n)(*[mask_slot] * n)
    ptrs = (ctypes.c_void_p * len(images))(*[im.ctypes.data for im in images])
    assert lib.ref_copy_layers_into_mips(TARGETS[fmt], depth, w, h, ptrs, len(images), planes, rows, counts, slots, n, int(has_alpha),
                                         start, ctypes.c_int(end)) == 0


def ref_do_write_dds(lib, fmt, depth, w, h, before, layers, has_alpha, mask_slot=0):
    """CopyLayersIntoMipMaps(..., 0, 1) on a one-image scratch, then (..., 1) on the whole chain, as DoWriteDDS calls them."""
    out = [b.copy() for b in before]
    ref_copy(lib, fmt, depth, w, h, out[:1], layers, has_alpha, 0, 1, mask_slot)
    if len(layers) > 1:
        ref_copy(lib, fmt, depth, w, h, out, layers, has_alpha, 1, 2 ** 31 - 1, mask_slot)
    return out


W, H = 13, 7                                  # ragged document: levels 13x7, 6x3, 3x1, 1x1
GRID = list(itertools.product(TARGETS, (8, 16, 32), (1, 2, 3), (True, False), (0, 1), (2, 4, 6)))


def grid_case(fmt, depth, channels, alpha, has_alpha, count):
    seed = depth * 1000 + channels * 100 + alpha * 10 + has_alpha + count * 7 + list(TARGETS).index(fmt) * 10000
    layers = make_layers(depth, W, H, count, channels, alpha, seed)
    before = before_levels(fmt == "BC6H", W, H, full_levels(W, H), seed + 1)
    return layers, before


@pytest.mark.parametrize("fmt,depth,channels", list(itertools.product(TARGETS, (8, 16, 32), (1, 2, 3))))
def test_oracle_matches_reference_function_bodies(ref_layers, fmt, depth, channels):
    for alpha, has_alpha, count in itertools.product((True, False), (0, 1), (2, 4, 6)):
        layers, before = grid_case(fmt, depth, channels, alpha, has_alpha, count)
        want = ref_do_write_dds(ref_layers, fmt, depth, W, H, before, layers, has_alpha, mask_slot=count & 2)
        got = oracle_layers_into([b.copy() for b in before], depth, W, layers, has_alpha)
        for l, (g, r) in enumerate(zip(got, want)):
            assert np.array_equal(g, r), (alpha, has_alpha, count, l)


def grid_digest(fmt, depth, channels, alpha, has_alpha, count, levels):
    return hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in levels)).hexdigest()


def test_oracle_matches_committed_reference_digests():
    """The digests were produced by the reference's own bodies (tests/golden/make_golden_layers.py); they keep the oracle
    pinned where neither the reference tree nor a prebuilt oracle/_ref exists."""
    golden = json.load(open(os.path.join(HERE, "golden", "layers_digests.json")))["levels"]
    for case in GRID:
        layers, before = grid_case(*case)
        got = oracle_layers_into([b.copy() for b in before], case[1], W, layers, case[4])
        assert grid_digest(*case, got) == golden[":".join(str(int(x) if isinstance(x, bool) else x) for x in case)], case
    assert len(golden) == len(GRID)


def test_depth16_white_alpha_is_the_plugins_15360():
    """FillLayerDataToWhite at depth 16 stores ConvertTo16Bit((unsigned8)255) = 15360, read back as 15360 / 32768."""
    rng = np.random.default_rng(1)
    layer = ([plane(16, 8, 4, rng, False)], None)
    ldr = oracle_copy(np.zeros((4, 8, 4), np.uint8), 16, 8, layer, False)
    hdr = oracle_copy(np.zeros((4, 8, 4), np.uint16), 16, 8, layer, True)          # hasAlpha with no alpha plane: white too
    assert (ldr[..., 3] == 119).all() and (hdr[..., 3] == 0x3780).all()
    for depth, want8, want16 in ((8, 255, 0x3C00), (32, 255, 0x3C00)):
        layer = ([plane(depth, 8, 4, rng, False)], None)
        assert (oracle_copy(np.zeros((4, 8, 4), np.uint8), depth, 8, layer, False)[..., 3] == want8).all()
        assert (oracle_copy(np.zeros((4, 8, 4), np.uint16), depth, 8, layer, False)[..., 3] == want16).all()


# ---- the kernel's per-texel routine on the CPU ----
@pytest.fixture(scope="module")
def emu_layers():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_layers_emu.so")
    src = os.path.join(T.ROOT, "tests", "emu", "layers_emu.cpp")
    deps = [src, os.path.join(T.ROOT, "intel-texture-works-plugin_b200", "csrc", "frontend.cuh")]
    if not os.path.exists(path) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(path):
        T.build_emu().compile_cpu(src, path)              # __graft_entry__.build() made it; rebuilt only when stale
    lib = ctypes.CDLL(path)
    lib.emu_layer_level.restype = ctypes.c_int
    return lib


def pad4(level):
    return T.synth.pad_to_4(level)


def stage(a, lw, lh):
    """The host's staging: the lw x lh top-left rectangle of a plane, tight."""
    return None if a is None else np.ascontiguousarray(a[:lh, :lw])


def emu_level(lib, level_padded, lw, lh, depth, layer, has_alpha, flip=0):
    channels, alpha = layer
    staged = [stage(c, lw, lh) for c in channels]
    p = _ptrs(staged, stage(alpha, lw, lh) if has_alpha else None)
    ph, pw = level_padded.shape[:2]
    assert lib.emu_layer_level(int(level_padded.dtype == np.uint16), level_padded.ctypes.data, lw, lh, pw, ph, depth, p, len(channels),
                               flip) == 0
    return level_padded


@pytest.mark.parametrize("fmt,depth,channels", list(itertools.product(TARGETS, (8, 16, 32), (1, 2, 3))))
def test_emulated_routine_matches_oracle(emu_layers, fmt, depth, channels):
    for alpha, has_alpha, count in itertools.product((True, False), (0, 1), (2, 6)):
        layers, before = grid_case(fmt, depth, channels, alpha, has_alpha, count)
        for l in range(min(count, len(before))):
            flip = (4 | 8) if (l == 0 and count == 6) else (4 if l == 0 else 0)
            lh, lw = before[l].shape[:2]
            want = oracle_copy(before[l].copy(), depth, W, layers[l], has_alpha, flip)
            got = emu_level(emu_layers, np.ascontiguousarray(pad4(before[l])), lw, lh, depth, layers[l], has_alpha, flip)
            assert np.array_equal(got, pad4(want)), (alpha, has_alpha, count, l)
            if l == 0:                                   # level 0 is written unpadded (the chain pads it)
                got = emu_level(emu_layers, before[0].copy(), lw, lh, depth, layers[0], has_alpha, flip)
                assert np.array_equal(got, want)


# ---- GPU ----
def oracle_file_levels(fmt, dxgi, prof, composite, layers, flags, levels):
    """The oracle pipeline: composite convert -> layer 0 -> flip -> chain -> layers >= 1 -> normalise -> pad -> encode."""
    import test_mips_f16 as HM
    o = T.oracle()
    hdr = fmt == "BC6H"
    h, w = composite.shape[:2]
    depth = composite.itemsize * 8
    flip = flags & (B.FRONT_FLIP_X | B.FRONT_FLIP_Y)
    has_alpha = flags & B.FRONT_HAS_ALPHA
    top = np.ascontiguousarray(o.convert_pixels(fmt, composite, flags & ~(B.FRONT_NORMALIZE | flip), pad=False))
    if layers:
        oracle_copy(top, depth, w, layers[0], has_alpha, flip)
    else:
        top = np.ascontiguousarray(o.convert_pixels(fmt, composite, flags & ~B.FRONT_NORMALIZE, pad=False))
    srgb = 1 if dxgi in (72, 78, 99) else 0
    chain = HM.oracle_chain(top, levels) if hdr else T.oracle_mip_chain_rgba8(top, srgb, levels, pad=False)
    chain = [np.ascontiguousarray(c) for c in chain]
    for l in range(1, min(len(layers), levels)):
        oracle_copy(chain[l], depth, w, layers[l], has_alpha)
    out = []
    for lv in chain:
        if flags & B.FRONT_NORMALIZE:                    # the oracle's normalise pass through an identity conversion
            if hdr:
                rgb = o.convert_pixels(fmt, lv.view(np.float16).astype(np.float32), B.FRONT_NORMALIZE, pad=False)
                lv = np.concatenate([rgb[..., :3], lv[..., 3:]], axis=2)
            else:
                lv = o.convert_pixels(fmt, lv, B.FRONT_NORMALIZE | B.FRONT_HAS_ALPHA, pad=False)
        out.append(o.encode(fmt, np.ascontiguousarray(HM.pad4(lv)), o.profile(prof) if prof else None))
    return out


def check_file(p, blob, d, want_levels):
    for l, want in enumerate(want_levels):
        off = p.lib.itw_dds_image_offset(ctypes.byref(d), 0, l)
        assert np.array_equal(blob[off:off + want.size], want), l


def composite_of(depth, w, h, planes, seed):
    rng = np.random.default_rng(seed)
    px = np.stack([plane(depth, w, h, rng, specials=False) for _ in range(planes)], axis=2)
    return np.ascontiguousarray(px)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,dxgi,prof,depth,channels,alpha,flags,w,h,count", [
    ("BC3", 77, None, 16, 3, False, 0, 64, 32, 7),                       # depth 16 without alpha: the 119 quirk
    ("BC3", 77, None, 16, 2, True, 1, 64, 32, 3),
    ("BC5", 83, None, 8, 3, False, 4 | 8 | 16, 64, 64, 3),               # flipped generated levels next to unflipped layer levels
    ("BC5", 83, None, 8, 2, False, 4 | 16, 32, 32, 2),
    ("BC7", 99, "veryfast", 8, 3, True, 1, 64, 32, 4),                   # _SRGB: sRGB chain, raw layer bytes
    ("BC7", 98, "veryfast", 32, 1, True, 1 | 2, 50, 27, 9),              # 50x27, 1-channel layers, extra layers
    ("BC6H", 95, "bc6h_veryfast", 8, 3, True, 1, 32, 16, 6),
    ("BC6H", 95, "bc6h_veryfast", 32, 2, False, 4 | 16, 50, 27, 3),
    ("BC1", 71, None, 8, 1, False, 0, 50, 27, 6)])
def test_gpu_encode_layers_matches_oracle_pipeline(fmt, dxgi, prof, depth, channels, alpha, flags, w, h, count):
    p = T.product()
    planes = 4 if (flags & B.FRONT_HAS_ALPHA) else 3
    composite = composite_of(depth, w, h, planes, seed=w + depth)
    if depth == 32:
        composite = np.clip(composite, 0, 4).astype(np.float32)
    layers = make_layers(depth, w, h, count, channels, alpha, seed=count + depth, specials=(depth != 32 or fmt != "BC6H"))
    if depth == 32 and fmt == "BC6H":
        layers = [([np.clip(c, 0, 4) for c in ch], None if a is None else np.clip(a, 0, 4)) for ch, a in layers]
    levels = full_levels(w, h)
    d = B.DdsDesc(w, h, levels, 1, dxgi, 0)
    s = p.profile(prof) if prof else None
    blob = p.dds_encode_layers(d, composite, layers, flags, s)
    check_file(p, blob, d, oracle_file_levels(fmt, dxgi, prof, composite, layers, flags, levels))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,dxgi,prof,w,h", [("BC7", 98, "veryfast", 64, 32), ("BC1", 71, None, 50, 27), ("BC3", 77, None, 32, 32)])
def test_gpu_layers_holding_the_generated_chain_give_encode_pixels_file(fmt, dxgi, prof, w, h):
    """Depth-8 RGBA layers that hold the library's own chain (de-padded) reproduce itw_dds_encode_pixels byte for byte; so does
    an empty layer list."""
    p = T.product()
    composite = composite_of(8, w, h, 4, seed=5)
    levels = full_levels(w, h)
    d = B.DdsDesc(w, h, levels, 1, dxgi, 0)
    s = p.profile(prof) if prof else None
    flags = B.FRONT_HAS_ALPHA
    want = p.dds_encode_pixels(d, [composite], flags, s)
    chain = T.oracle_mip_chain_rgba8(composite, 1 if dxgi in (72, 78, 99) else 0, levels, pad=False)
    layers = []
    for lv in chain:
        doc = np.zeros((h, w, 4), np.uint8)
        doc[:lv.shape[0], :lv.shape[1]] = lv
        layers.append(([doc[..., 0], doc[..., 1], doc[..., 2]], doc[..., 3]))
    assert np.array_equal(p.dds_encode_layers(d, composite, layers, flags, s), want)
    assert np.array_equal(p.dds_encode_layers(d, composite, [], flags, s), want)
    assert np.array_equal(p.dds_encode_layers(d, composite, [], 4 | 8, s), p.dds_encode_pixels(d, [composite], 4 | 8, s))


@pytest.mark.gpu
def test_gpu_round_trip_through_the_open_path():
    """itw_dds_open + ITW_OPEN_MIPS + itw_dds_read_layer per level, de-interleaved into planes, then itw_dds_encode_layers: level l
    of the new file is the oracle encode of the padded decoded level l."""
    p, o = T.product(), T.oracle()
    w, h = 64, 32
    levels = full_levels(w, h)
    d = B.DdsDesc(w, h, levels, 1, 77, 0)
    src = p.dds_encode_pixels(d, [composite_of(8, w, h, 4, seed=9)], B.FRONT_HAS_ALPHA)
    info, decoded = p.dds_open_layers(src, B.OPEN_MIPS)
    assert len(decoded) == levels and decoded[0].dtype == np.uint8
    layers = [([L[..., 0], L[..., 1], L[..., 2]], L[..., 3] if L.shape[2] == 4 else None) for L in decoded]
    flags = B.FRONT_HAS_ALPHA if decoded[0].shape[2] == 4 else 0
    blob = p.dds_encode_layers(d, decoded[0], layers, flags)
    want = []
    for l, L in enumerate(decoded):
        lv = np.ascontiguousarray(L[:lvl(h, l), :lvl(w, l)])
        if lv.shape[2] == 3:
            lv = np.concatenate([lv, np.full(lv.shape[:2] + (1,), 255, np.uint8)], axis=2)
        want.append(o.encode("BC3", np.ascontiguousarray(pad4(lv))))
    check_file(p, blob, d, want)


def _layer_structs(layers, row_bytes, ptr_of):
    arr = (B.LayerSource * max(1, len(layers)))()
    for i, (channels, alpha) in enumerate(layers):
        arr[i].channel_count = len(channels)
        for c, pl in enumerate(channels):
            arr[i].channels[c] = ptr_of(pl)
        arr[i].alpha = ptr_of(alpha) if alpha is not None else None
        arr[i].row_bytes = row_bytes
    return arr


@pytest.mark.gpu
def test_gpu_device_planes_and_wide_rows():
    import torch
    p = T.product()
    w, h, depth, count = 50, 27, 16, 4
    levels = full_levels(w, h)
    d = B.DdsDesc(w, h, levels, 1, 77, 0)
    composite = composite_of(depth, w, h, 4, seed=3)
    layers = make_layers(depth, w, h, count, 3, True, seed=4)
    want = p.dds_encode_layers(d, composite, layers, B.FRONT_HAS_ALPHA)
    pitch = 64                                                   # elements per row: wider than the document
    keep = []

    def wide(a, device):
        buf = np.zeros((h, pitch), a.dtype)
        buf[:, :w] = a
        t = torch.from_numpy(buf.view(np.int16)).cuda() if device else buf
        keep.append(t)
        return t.data_ptr() if device else t.ctypes.data
    for device in (False, True):
        arr = _layer_structs(layers, pitch * 2, lambda a: wide(a, device))
        d_comp = torch.from_numpy(composite.view(np.int16)).cuda() if device else composite
        keep.append(d_comp)
        src = B.PixelSource(d_comp.data_ptr() if device else composite.ctypes.data, w, h, 4, depth, 0)
        n = p.lib.itw_dds_file_bytes(ctypes.byref(d))
        out = np.zeros(n, np.uint8)
        got = p.dds_encode_layers_raw(d, src, arr, count, B.FRONT_HAS_ALPHA, None, out.ctypes.data, n)
        assert got == n, p.last_error()
        assert np.array_equal(out, want), device


@pytest.mark.gpu
def test_gpu_rejections_enqueue_nothing():
    p = T.product()
    w, h = 32, 16
    levels = full_levels(w, h)
    composite = composite_of(8, w, h, 4, seed=1)
    layers = make_layers(8, w, h, 3, 3, True, seed=2)
    good = B.DdsDesc(w, h, levels, 1, 71, 0)
    n = p.lib.itw_dds_file_bytes(ctypes.byref(good))
    p.dds_encode_layers(good, composite, layers, 1)             # warm: the context exists
    src = B.PixelSource(composite.ctypes.data, w, h, 4, 8, 0)

    def call(desc=good, source=src, arr=None, count=3, flags=1):
        arr = arr if arr is not None else _layer_structs(layers, 0, lambda a: a.ctypes.data)
        out = np.full(n, 0xAB, np.uint8)
        before = p.launch_count()
        got = p.dds_encode_layers_raw(desc, source, arr, count, flags, None, out.ctypes.data, n)
        assert got == 0 and p.last_error() != ""
        assert (out == 0xAB).all() and p.launch_count() == before
    call(desc=B.DdsDesc(w, h, levels + 3, 1, 71, 0))                        # the description
    call(desc=B.DdsDesc(w, h, levels, 6, 71, 1))                             # a cube map
    call(source=B.PixelSource(composite.ctypes.data, w + 4, h, 4, 8, 0))     # composite size against the description
    bad = _layer_structs(layers, 0, lambda a: a.ctypes.data)
    bad[1].channel_count = 4
    call(arr=bad)
    bad = _layer_structs(layers, 0, lambda a: a.ctypes.data)
    bad[2].channels[1] = None
    call(arr=bad)
    call(arr=_layer_structs(layers, w - 1, lambda a: a.ctypes.data))         # row_bytes too small
    call(flags=1 | 64)                                                       # unknown flag bits
    bad = _layer_structs(layers, 0, lambda a: a.ctypes.data)                 # a layer that is never read is not checked
    bad[2].channel_count = 0
    out = np.zeros(n, np.uint8)
    assert p.dds_encode_layers_raw(B.DdsDesc(w, h, 2, 1, 71, 0), src, bad, 3, 1, None, out.ctypes.data, n) != 0
