"""The BC6H save and preview paths on HDR values (tests/hdr_corpus.py): float planes -> front end -> RGBA16F mip chain ->
normal-map pass -> pad -> BC6H -> DDS, and the preview.

A. PINNED domain: every half is at most 65504 in magnitude, signs and denormals included.  CPU: the oracle against the
   reference's own bodies (oracle/_ref, when built) and against their committed digests (tests/golden/hdr_digests.json); the
   kernels' per-texel routines (tests/emu) against the oracle.  GPU: every save / preview entry point against the oracle.
B. PRODUCT-DEFINED domain: values above 65504, +-Inf, NaN, exponent-31 halves.  The same paths against the oracle only: this pins
   the product to its DirectXMath 3.06 restatement (csrc/frontend.cuh), not to the reference, whose SDK half conversions are
   not in its tree.  A change of DirectXMath generation edits these tests alone."""
import ctypes
import functools

import numpy as np
import pytest

import hdr_corpus as H
import itw_testlib as T
import test_frontend as F
import test_mips_f16 as M

B = T.binding
CHAIN_SHAPES = M.SIZES + H.EXTRA_CHAIN_SHAPES


@functools.lru_cache(None)
def golden():
    import json
    import os
    return json.load(open(os.path.join(os.path.dirname(__file__), "golden", "hdr_digests.json")))


def chain_sha(chain):
    return H.sha(np.concatenate([l.reshape(-1) for l in chain]))


def emu_chain(img, levels):
    """Levels 1 ... levels-1, padded, from the kernel's per-texel routine with the host's stale-row rule (as test_mips_f16)."""
    emu = T.emu().lib
    h, w = img.shape[:2]
    box = (w & (w - 1)) == 0 and (h & (h - 1)) == 0
    cur, keep, out, stale_ptr = np.ascontiguousarray(img), [], [], None
    for dh, dw in M.level_dims(w, h, levels)[1:]:
        ph, pw = dh + (-dh) % 4, dw + (-dw) % 4
        got = np.zeros((ph, pw, 4), np.uint16)
        if cur.shape[0] > 1:
            stale_ptr = cur.ctypes.data + (cur.shape[0] - 1) * cur.strides[0]
            keep.append(cur)
        emu.emu_mip_level_f16(ctypes.c_void_p(cur.ctypes.data), cur.shape[1], cur.shape[0], cur.strides[0], got.ctypes.data_as(ctypes.c_void_p),
                              dw, dh, pw, ph, 1 if box else 0, ctypes.c_void_p(stale_ptr))
        out.append(got)
        cur = np.ascontiguousarray(got[:dh, :dw])
    return out


def first_difference(got, want):
    """(y, x, channel, got, want) of the first differing half, for the assertion message."""
    i = tuple(int(v) for v in np.argwhere(got != want)[0])
    return i, hex(int(got[i])), hex(int(want[i]))


# ================================================= corpus power (CPU) =================================================
def test_corpus_reaches_every_order_and_conversion_class():
    """The corpus must keep seeing what it was built for: on the level 0 -> 1 step the reference's summation order differs from
    each other order in >= 100 stored halves per chain, and every conversion class occurs often enough."""
    power = {}
    for fam in ("order_cells", "boundary"):
        img = H.family(fam, 64, 64)
        ref = H.box_level1(img)
        for order in H.BOX_ORDERS[1:]:
            power[(fam, "box", order)] = int((H.box_level1(img, order) != ref).sum())
        img = H.family(fam, 48, 96)                                  # even, not a power of two: linear taps on the 2x2 grid
        power[(fam, "linear", "columns_first")] = int((H.linear_level1(img, "columns_first") != H.linear_level1(img)).sum())
    assert all(n >= 100 for n in power.values()), power

    bits = np.concatenate([H.family(f, 64, 64).reshape(-1, 4) for f in H.FAMILIES])
    lvl1 = np.concatenate([H.box_level1(H.family(f, 64, 64)).reshape(-1, 4) for f in H.FAMILIES])
    vals, out = H.float_from_half(bits), H.float_from_half(lvl1)
    bplanes = H.boundary_planes(64, 64).reshape(-1)
    nv = H.family("normal_vectors", 64, 64)
    prod = H.product_defined(64, 64)
    classes = {
        "negative halves into the filter": int((vals < 0).sum()),
        "half denormals made by averaging": int(((out != 0) & (np.abs(out) < 2.0 ** -14)).sum()),
        "truncating denormal shift != IEEE": int((H.half_from_float(bplanes) != H.half_from_float_ieee(bplanes)).sum()),
        "65504 ... 65519 -> 0x7BFF": int(((np.abs(bplanes) >= 65504) & (np.abs(bplanes) < 65520)).sum()),
        "exponent-31 halves": int(((prod & 0x7C00) == 0x7C00).sum()),
        "x / m != x * (1 / m)": int((H.normalize(nv) != H.normalize(nv, reciprocal=False)).sum()),
        "zero normal vectors": int((np.abs(H.float_from_half(nv[..., :3])).max(-1) == 0).sum()),
        "single-axis normal vectors": int(((H.float_from_half(nv[..., :3]) != 0).sum(-1) == 1).sum()),
        "huge normal vectors": int((np.abs(H.float_from_half(nv[..., :3])).max(-1) > 8192).sum()),
    }
    assert all(n >= 100 for n in classes.values()), classes


# ================================================= A. pinned domain, CPU =================================================
@pytest.mark.parametrize("h,w", CHAIN_SHAPES)
def test_chain_oracle_matches_reference_bodies_and_digests(h, w):
    """oracle_mip_chain_f16 == the reference's _Generate2DMips{Box,Linear}Filter (when oracle/_ref is built) == the committed
    digests, for every pinned family: 256x256 box, 129x255 linear, 8x512 / 512x8 (the stale fourth tap), 1x256 / 256x1."""
    lib = T.ref_frontend()
    levels = M.full_levels(w, h)
    for fam in H.FAMILIES:
        img = H.family(fam, h, w)
        assert H.sha(img) == golden()["inputs"][H.key(fam, h, w)], fam
        got = M.oracle_chain(img, levels)
        if lib is not None:
            want = M.chain_with(lib.ref_mip_chain_f16, img, levels)
            for l in range(levels):
                assert np.array_equal(got[l], want[l]), (fam, l, first_difference(got[l], want[l]))
        assert chain_sha(got) == golden()["chain_f16"][H.key(fam, h, w)], fam


@pytest.mark.parametrize("h,w", CHAIN_SHAPES)
def test_emulated_chain_matches_oracle(h, w):
    levels = M.full_levels(w, h)
    for fam in H.FAMILIES:
        img = H.family(fam, h, w)
        want = M.oracle_chain(img, levels)
        for l, got in enumerate(emu_chain(img, levels), 1):
            exp = M.pad4(want[l])
            assert np.array_equal(got, exp), (fam, l, first_difference(got, exp))


@pytest.mark.parametrize("planes", [1, 2, 3, 4])
def test_convert_oracle_matches_reference_bodies_and_digests(planes):
    """BC6H front end, every flag set: unclipped 32-bit planes of every pinned family, and 16-bit planes holding every value."""
    lib, o = T.ref_frontend(), T.oracle()
    h, w = H.CONVERT_SHAPE
    cases = [(H.key(fam, planes, f), np.ascontiguousarray(H.family_planes(fam, h, w)[..., :planes]), f, "convert32")
             for fam in H.FAMILIES for f in F.flag_sets("BC6H", 32, planes)]
    px16 = H.sixteen_bit_planes(planes)
    assert H.sha(px16) == golden()["inputs"][H.key("u16", planes)]
    cases += [(H.key(planes, f), px16, f, "convert16") for f in F.flag_sets("BC6H", 16, planes)]
    for k, px, flags, table in cases:
        got = o.convert_pixels("BC6H", px, flags)
        if lib is not None:
            want = F.ref_convert(lib, "BC6H", px, flags)
            assert np.array_equal(got, want), (k, first_difference(got, want))
        assert H.sha(got) == golden()[table][k], k


@pytest.mark.parametrize("planes", [1, 2, 3, 4])
def test_emulated_convert_matches_oracle(planes):
    o, e = T.oracle(), T.emu()
    h, w = H.CONVERT_SHAPE
    srcs = [np.ascontiguousarray(H.family_planes(fam, h, w)[..., :planes]) for fam in H.FAMILIES] + [H.sixteen_bit_planes(planes)]
    for px in srcs:
        for flags in F.flag_sets("BC6H", px.itemsize * 8, planes):
            for pad in (True, False):
                got, want = e.convert_pixels("BC6H", px, flags, pad=pad), o.convert_pixels("BC6H", px, flags, pad=pad)
                assert np.array_equal(got, want), (px.dtype, flags, pad, first_difference(got, want))


@pytest.mark.parametrize("fam,h,w", H.BC6H_CHAINS)
def test_oracle_bc6h_matches_reference_build_and_digests(fam, h, w):
    """The oracle's BC6H blocks of every padded chain level == oracle/_ref/libitw_ref.so (when built) == the digests, all presets."""
    o, ref = T.oracle(), T.ref()
    levels = M.full_levels(w, h)
    chain = [np.ascontiguousarray(M.pad4(l)) for l in M.oracle_chain(H.family(fam, h, w), levels)]
    for preset in B.BC6H_PROFILES:
        got = [o.encode("BC6H", l, o.profile(preset)) for l in chain]
        if ref is not None:
            for l, lv in enumerate(chain):
                assert np.array_equal(got[l], ref.encode("BC6H", lv, ref.profile(preset))), (preset, l)
        assert H.sha(np.concatenate(got)) == golden()["bc6h"][H.key(fam, h, w, preset)], preset


# ================================================= B. product-defined domain, CPU ==========================================
PRODUCT_CHAIN_SHAPES = [(64, 64), (8, 64), (16, 1), (27, 50), (5, 3), (1, 9)]


@pytest.mark.parametrize("h,w", PRODUCT_CHAIN_SHAPES)
def test_product_defined_emulated_chain_matches_oracle(h, w):
    """Exponent-31 halves, 0x7FFF saturation, NaN / Inf bit patterns: the kernel's routine == the oracle's DirectXMath 3.06
    restatement (not the reference's: its SDK conversions are outside its tree)."""
    levels = M.full_levels(w, h)
    img = H.product_defined(h, w)
    want = M.oracle_chain(img, levels)
    for l, got in enumerate(emu_chain(img, levels), 1):
        exp = M.pad4(want[l])
        assert np.array_equal(got, exp), (l, first_difference(got, exp))


def test_product_defined_emulated_convert_matches_oracle():
    o, e = T.oracle(), T.emu()
    px = H.product_defined_planes(*H.CONVERT_SHAPE)
    for planes in (1, 2, 3, 4):
        sub = np.ascontiguousarray(px[..., :planes])
        for flags in F.flag_sets("BC6H", 32, planes):
            got, want = e.convert_pixels("BC6H", sub, flags), o.convert_pixels("BC6H", sub, flags)
            assert np.array_equal(got, want), (planes, flags, first_difference(got, want))


# ================================================= GPU =================================================
NORM = B.FRONT_NORMALIZE


def gpu_chain(img, levels):
    """itw_generate_mips_device_f16 from a device copy of `img`: the padded levels (level 0 only when it needed padding)."""
    import torch
    lib = T.product()
    h, w = img.shape[:2]
    d_img = torch.from_numpy(np.ascontiguousarray(img).view(np.int16).reshape(-1)).cuda()
    pad0 = (w % 4 != 0) or (h % 4 != 0)
    scratch = torch.zeros(max(2 * lib.lib.itw_mip_scratch_bytes(w, h, levels, 0 if pad0 else 1), 32), dtype=torch.uint8, device="cuda")
    outs = (B.RgbaSurface * levels)()
    top = B.RgbaSurface(d_img.data_ptr(), w, h, w * 8)
    f = lib.lib.itw_generate_mips_device_f16
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.POINTER(B.RgbaSurface), ctypes.c_int, ctypes.POINTER(B.RgbaSurface), ctypes.c_void_p, ctypes.c_void_p]
    assert f(ctypes.byref(top), levels, outs, ctypes.c_void_p(scratch.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    base, host = scratch.data_ptr(), scratch.cpu().numpy()
    res = {}
    for l in range(0 if pad0 else 1, levels):
        off = outs[l].ptr - base
        res[l] = host[off:off + outs[l].height * outs[l].stride].view(np.uint16).reshape(outs[l].height, outs[l].width, 4)
    return res


def check_gpu_chain(img):
    h, w = img.shape[:2]
    levels = M.full_levels(w, h)
    want = M.oracle_chain(img, levels)
    for l, got in gpu_chain(img, levels).items():
        exp = M.pad4(want[l])
        assert np.array_equal(got, exp), (l, first_difference(got, exp))


def oracle_save_path(srcs, flags, levels, prof):
    """itw_dds_encode_pixels for BC6H restated: oracle convert (+ flip) -> oracle chain -> oracle normalise of every level ->
    pad -> oracle encode; {(item, mip): blocks}.  The normal-map pass re-reads the stored halves through the 3.06 decode."""
    o = T.oracle()
    out = {}
    for item, px in enumerate(srcs):
        top = o.convert_pixels("BC6H", px, flags & ~NORM, pad=False)
        for mip, lv in enumerate(M.oracle_chain(top, levels)):
            if flags & NORM:
                rgb = o.convert_pixels("BC6H", np.ascontiguousarray(H.planes(lv)), NORM, pad=False)
                lv = np.concatenate([rgb[..., :3], lv[..., 3:]], axis=2)
            out[(item, mip)] = o.encode("BC6H", np.ascontiguousarray(M.pad4(lv)), o.profile(prof))
    return out


def check_dds(blob, d, want):
    lib = T.product()
    for (item, mip), blocks in want.items():
        off = lib.lib.itw_dds_image_offset(ctypes.byref(d), item, mip)
        got = blob[off:off + blocks.size]
        assert np.array_equal(got, blocks), (item, mip, int((got.reshape(-1, 16) != blocks.reshape(-1, 16)).any(1).argmax()))


def sources(kind, planes, w, h, items):
    if kind == "u16":
        return [np.ascontiguousarray(H.sixteen_bit_planes(planes, seed=i)[:h, :w]) for i in range(items)]
    if kind == "product_defined":
        return [np.ascontiguousarray(H.product_defined_planes(h, w, seed=i)[..., :planes]) for i in range(items)]
    return [np.ascontiguousarray(H.family_planes(kind, h, w, seed=i)[..., :planes]) for i in range(items)]


DDS_PIXEL_CASES = [  # dxgi, preset, source, planes, flags, w, h, items, cube
    (95, "bc6h_veryfast", "log_uniform", 3, 0, 64, 64, 1, 0),
    (96, "bc6h_fast", "order_cells", 4, B.FRONT_HAS_ALPHA, 60, 36, 1, 0),
    (95, "bc6h_basic", "normal_vectors", 3, B.FRONT_FLIP_X | B.FRONT_FLIP_Y | NORM, 32, 16, 1, 0),
    (96, "bc6h_slow", "boundary", 4, B.FRONT_HAS_ALPHA | NORM, 27, 13, 1, 0),
    (95, "bc6h_veryslow", "u16", 4, B.FRONT_HAS_ALPHA | B.FRONT_FLIP_Y, 20, 12, 1, 0),
    (95, "bc6h_basic", "exposure_ramp", 3, B.FRONT_FLIP_X, 32, 32, 6, 1),
    (96, "bc6h_veryfast", "real_hdr", 4, B.FRONT_HAS_ALPHA, 128, 128, 1, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(256, 256), (16, 128), (128, 16), (37, 61), (4, 4), (1, 16), (64, 200), (2048, 2048), (1023, 2047)])
def test_gpu_chain_matches_oracle(h, w):
    """Every pinned family through itw_generate_mips_device_f16; 2048^2 (box, multi-row grids) and 2047x1023 (linear, long rows)
    with the order-sensitive and log-uniform families."""
    for fam in (("order_cells", "log_uniform") if h * w > 1 << 20 else H.FAMILIES):
        check_gpu_chain(H.family(fam, h, w))


@pytest.mark.gpu
@pytest.mark.parametrize("dxgi,prof,kind,planes,flags,w,h,items,cube", DDS_PIXEL_CASES)
def test_gpu_dds_encode_pixels_matches_oracle(dxgi, prof, kind, planes, flags, w, h, items, cube):
    """The whole save path from unclipped 32-bit planes (and full-range 16-bit ones), BC6H_UF16 and BC6H_SF16 (both take the
    unsigned encoder), every BC6H preset on one shape."""
    p = T.product()
    srcs = sources(kind, planes, w, h, items)
    levels = M.full_levels(w, h)
    d = B.DdsDesc(w, h, levels, items, dxgi, cube)
    blob = p.dds_encode_pixels(d, srcs, flags, p.profile(prof))
    check_dds(blob, d, oracle_save_path(srcs, flags, levels, prof))


@pytest.mark.gpu
@pytest.mark.parametrize("fam,prof,w,h,items,cube", [("log_uniform", "bc6h_veryfast", 64, 64, 1, 0), ("order_cells", "bc6h_fast", 60, 36, 1, 0),
                                                     ("boundary", "bc6h_basic", 32, 32, 6, 1), ("normal_vectors", "bc6h_veryfast", 64, 16, 1, 0)])
def test_gpu_dds_encode_texture_matches_oracle(fam, prof, w, h, items, cube):
    """RGBA16F tops that keep their sign bits and denormals: itw_dds_encode_texture == oracle chain + pad + encode."""
    p, o = T.product(), T.oracle()
    tops = [H.family(fam, h, w, seed=i) for i in range(items)]
    levels = M.full_levels(w, h)
    d = B.DdsDesc(w, h, levels, items, 95, cube)
    blob = p.dds_encode_texture(d, tops, p.profile(prof))
    want = {(i, m): o.encode("BC6H", np.ascontiguousarray(M.pad4(lv)), o.profile(prof))
            for i, t in enumerate(tops) for m, lv in enumerate(M.oracle_chain(t, levels))}
    check_dds(blob, d, want)


ENCODE_PIXEL_CASES = [("BC6H", "bc6h_basic", 3, 0), ("BC6H", "bc6h_veryfast", 4, B.FRONT_HAS_ALPHA | NORM),
                      ("BC1", None, 3, B.FRONT_GAMMA), ("BC3", None, 4, B.FRONT_GAMMA | B.FRONT_HAS_ALPHA), ("BC7", "basic", 4, B.FRONT_GAMMA)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,prof,planes,flags", ENCODE_PIXEL_CASES)
def test_gpu_encode_pixels_unclipped_planes(fmt, prof, planes, flags):
    """itw_encode_pixels from the unclipped HDR planes that test_frontend clips to [0, 4]: == oracle convert + oracle encode."""
    o, p = T.oracle(), T.product()
    for fam in ("log_uniform", "boundary", "exposure_ramp", "normal_vectors"):
        px = np.ascontiguousarray(H.family_planes(fam, 27, 50)[..., :planes])
        want = o.encode(fmt, o.convert_pixels(fmt, px, flags), o.profile(prof) if prof else None)
        assert np.array_equal(p.encode_pixels(fmt, px, flags, p.profile(prof) if prof else None), want), fam


def check_preview(fmt, faces, flags, prof):
    import preview_lib as P
    if P.ref() is None:
        pytest.skip("oracle/_ref/libitw_ref_preview.so unavailable")
    p = T.product()
    want, nbytes = P.oracle_preview(fmt, faces, flags, prof)
    got, n = p.preview_pixels(fmt, faces, flags, p.profile(prof))
    assert n == nbytes and got.tobytes() == want.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,faces", [(32, 1), (32, 6), (16, 1), (16, 6)])
def test_gpu_preview_bc6h(depth, faces):
    """itw_preview_pixels for BC6H: float display at depth 32, saturated UNORM8 at depth 16; one face and the cube cross."""
    w, h = (37, 22) if faces == 1 else (9, 7)
    src = [s for i in range(faces) for s in sources("u16" if depth == 16 else ("log_uniform", "exposure_ramp")[i % 2], 4, w, h, 1)]
    check_preview(95, src, B.FRONT_HAS_ALPHA if faces == 1 else B.FRONT_FLIP_Y, "bc6h_basic")


# ================================================= B. product-defined domain, GPU ==========================================
@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(256, 256), (37, 61), (1, 16), (64, 200)])
def test_gpu_product_defined_chain_matches_oracle(h, w):
    """Exponent-31 halves and saturated values through the device chain == the oracle's 3.06 restatement (not the reference)."""
    check_gpu_chain(H.product_defined(h, w))


@pytest.mark.gpu
@pytest.mark.parametrize("dxgi,prof,planes,flags,w,h", [(95, "bc6h_veryfast", 3, 0, 64, 64), (96, "bc6h_basic", 4, B.FRONT_HAS_ALPHA | NORM, 27, 13),
                                                        (95, "bc6h_fast", 3, B.FRONT_FLIP_X | B.FRONT_FLIP_Y, 60, 36)])
def test_gpu_product_defined_save_path_matches_oracle(dxgi, prof, planes, flags, w, h):
    """+-Inf, NaN, 1e9, 70000, 131008 planes through itw_dds_encode_pixels, and exponent-31 tops through itw_dds_encode_texture,
    against the oracle's 3.06 restatement."""
    p, o = T.product(), T.oracle()
    levels = M.full_levels(w, h)
    srcs = sources("product_defined", planes, w, h, 1)
    d = B.DdsDesc(w, h, levels, 1, dxgi, 0)
    check_dds(p.dds_encode_pixels(d, srcs, flags, p.profile(prof)), d, oracle_save_path(srcs, flags, levels, prof))
    top = H.product_defined(h, w)
    d = B.DdsDesc(w, h, levels, 1, 95, 0)
    check_dds(p.dds_encode_texture(d, [top], p.profile(prof)), d,
              {(0, m): o.encode("BC6H", np.ascontiguousarray(M.pad4(lv)), o.profile(prof)) for m, lv in enumerate(M.oracle_chain(top, levels))})


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,prof,planes,flags", ENCODE_PIXEL_CASES)
def test_gpu_product_defined_encode_pixels(fmt, prof, planes, flags):
    o, p = T.oracle(), T.product()
    px = np.ascontiguousarray(H.product_defined_planes(27, 50)[..., :planes])
    want = o.encode(fmt, o.convert_pixels(fmt, px, flags), o.profile(prof) if prof else None)
    assert np.array_equal(p.encode_pixels(fmt, px, flags, p.profile(prof) if prof else None), want)


@pytest.mark.gpu
@pytest.mark.parametrize("faces", [1, 6])
def test_gpu_product_defined_preview_bc6h(faces):
    w, h = (37, 22) if faces == 1 else (9, 7)
    check_preview(95, sources("product_defined", 4, w, h, faces), B.FRONT_HAS_ALPHA, "bc6h_basic")
