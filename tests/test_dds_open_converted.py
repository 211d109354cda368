"""The converted open path on the CPU (include/itw_bcn.h section 14): the per-texel chain of the layer kernel (emulated) against the
reference's own _LoadScanline / _ConvertScanline / _StoreScanline over whole value domains, the alpha predicate of the scan against the
cut IsAlphaAllOpaque branch for every alpha value, header parsing against _DecodeDDSHeader, the refusals (all before any CUDA call)
and the layout."""
import numpy as np
import pytest

import itw_testlib as T
import open_converted_lib as C
import open_uncompressed_lib as U
import test_dds_open_uncompressed as TU       # section 13's g_LegacyDDSMap headers and ambiguous headers

B = T.binding

pytestmark = pytest.mark.skipif(C.ref() is None or U.ref() is None, reason="oracle/_ref/libitw_ref_open_converted.so not built")

RNG = np.random.default_rng(14)


def domain(fmt):
    """Source texels of `fmt` covering its domain: every value of every channel where the domain allows."""
    if fmt in (10, 13):                    # every half / SNORM16 pattern in every channel position
        v = np.arange(65536, dtype=np.uint16)
        return np.stack([v, np.roll(v, 1), np.roll(v, 7), np.roll(v, 13)], -1).tobytes()
    if fmt in (54, 58):
        return np.arange(65536, dtype=np.uint16).tobytes()
    if fmt in (34, 35, 37):
        v = np.arange(65536, dtype=np.uint16)
        return np.stack([v, np.roll(v, 5)], -1).tobytes()
    if fmt == 115:
        return np.arange(65536, dtype=np.uint16).tobytes()
    if fmt in (49, 51):
        v = np.arange(65536, dtype=np.uint16)
        return v.tobytes()
    if fmt in (63, 65):
        return np.arange(256, dtype=np.uint8).tobytes()
    if fmt == 31:
        v = np.arange(256, dtype=np.uint32)
        return (v | (np.roll(v, 3) << 8) | (np.roll(v, 101) << 16) | (np.roll(v, 200) << 24)).astype(np.uint32).tobytes()
    if fmt == 26:                          # every 11-bit field of red and green, every 10-bit field of blue
        f11 = np.arange(2048, dtype=np.uint32)
        r = f11 | (np.roll(f11, 3) << 11) | ((np.arange(2048, dtype=np.uint32) % 1024) << 22)
        b = RNG.integers(0, 2048, 1024).astype(np.uint32) | (RNG.integers(0, 2048, 1024).astype(np.uint32) << 11) | \
            (np.arange(1024, dtype=np.uint32) << 22)
        return np.concatenate([r, b]).astype(np.uint32).tobytes()
    if fmt == 67:                          # every (mantissa, exponent) pair, in every channel, the other channels random
        m, e = np.meshgrid(np.arange(512, dtype=np.uint32), np.arange(32, dtype=np.uint32))
        m, e = m.ravel(), e.ravel()
        out = []
        for ch in range(3):
            w = RNG.integers(0, 1 << 27, m.size).astype(np.uint32) & ~np.uint32(0x1FF << (9 * ch))
            out.append(w | (m << (9 * ch)) | (e << 27))
        return np.concatenate(out).astype(np.uint32).tobytes()
    if fmt == 16:                          # float edges: zeros, denormals, infinities, NaNs, values around 1, random bits
        edge = np.array([0, 0x80000000, 1, 0x807FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFFFFFFF, 0x3F800000,
                         0x3F7FFFFF, 0x3F800001, 0xBF800000, 0x00800000, 0x7F7FFFFF], np.uint32)
        r = RNG.integers(0, 1 << 32, 4096, dtype=np.uint64).astype(np.uint32)
        v = np.concatenate([edge, r])
        return np.stack([v, np.roll(v, 3)], -1).astype(np.uint32).tobytes()
    raise KeyError(fmt)


@pytest.mark.parametrize("fmt", sorted(C.LOADED))
def test_per_texel_chain_against_the_reference(fmt):
    src = domain(fmt)
    kind = C.LOADED[fmt][0]
    want = C.ref_convert(fmt, src)
    got = C.emu_texels(kind, 4, src)
    assert np.array_equal(got, want), f"{int((got != want).sum())} bytes differ"
    plane = len(got) // (len(src) // C.LOADED[fmt][1]) // 4
    three = C.emu_texels(kind, 3, src)
    assert np.array_equal(three.reshape(-1, 3 * plane), got.reshape(-1, 4 * plane)[:, :3 * plane])


def test_x4r4g4b4_sets_alpha():
    src = np.arange(65536, dtype=np.uint16).tobytes()
    want = C.ref_convert(115, C.set_alpha_4444(src))
    assert np.array_equal(C.emu_texels(C.KIND_BGRX4, 4, src), want)


@pytest.mark.parametrize("fmt", [f for f in sorted(C.LOADED) if C.LOADED[f][4]])
def test_alpha_predicate_for_every_alpha_value(fmt):
    kind, tb = C.LOADED[fmt][0], C.LOADED[fmt][1]
    if fmt == 65:
        src = np.arange(256, dtype=np.uint8).tobytes()
    elif fmt == 31:
        src = (np.arange(256, dtype=np.uint32) << 24 | 0x00808080).astype(np.uint32).tobytes()
    elif fmt == 115:
        src = np.arange(65536, dtype=np.uint16).tobytes()
    else:                                  # every alpha ushort, colour random
        a = np.arange(65536, dtype=np.uint64)
        src = (RNG.integers(0, 1 << 48, 65536, dtype=np.uint64) | (a << 48)).astype(np.uint64).tobytes()
    want = 1 - C.ref_opaque(fmt, src)
    for slot in range(4 // tb if tb < 4 else 1):    # every alpha slot of the scan's word: byte 0..3 (A8), ushort 0..1 (4444)
        assert np.array_equal(C.emu_below(kind, src, tb, slot), want), slot


def verdict(file):
    """Open the header alone (every accepted header then fails at its size check, before any CUDA call)."""
    lib = T.product()
    dx10 = file.size >= 148 and bytes(file[84:88]) == b"DX10"
    f = np.ascontiguousarray(file[:min(file.size, 148 if dx10 else 128)])
    info = B.DdsConvertedInfo()
    before = bytes(info)
    assert lib.dds_open_converted_raw(f.ctypes.data, f.size, info) != 0
    assert bytes(info) == before
    msg = lib.last_error()
    assert msg.startswith("itw_dds_open_converted: "), msg
    if "truncated file" in msg:
        return True, int(msg.split("needs ")[1].rstrip(")")), msg
    return False, None, msg


def check_header(file):
    """The product's verdict on `file` against _DecodeDDSHeader: accepted iff the loaded format is served and the loader does not
    expand it (CONV_FLAGS_EXPAND: the palettised and 3:3:2 / 4:4 forms, A4L4 loading as B4G4R4A4 among them); an accepted header needs
    exactly the file's size, and when the loaded format has no alpha (the open is then host-only) the product's description and
    header form are the reference's."""
    m = U.ref_header(file)
    ok, need, msg = verdict(file)
    assert ok == (m is not None and m["format"] in C.LOADED and not m["conv"] & 0x1), msg
    if not ok:
        return m, msg
    assert need == file.size
    if not C.LOADED[m["format"]][4]:
        lib = T.product()
        info = lib.dds_open_converted(file.ctypes.data, file.size)
        d = info.desc
        assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
            (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
        assert info.payload_offset == m["offset"]
        forms = {v[2]: v[1] for v in C.LEGACY.values() if v[1] != B.CONV_X4R4G4B4}
        want_form = B.CONV_DX10 if m["offset"] == 148 else forms[m["format"]]
        assert info.form == want_form
    return m, msg


@pytest.mark.parametrize("label,writer", C.FORMS, ids=[f[0] for f in C.FORMS])
@pytest.mark.parametrize("w,h,mips,cube", [(1, 1, 1, False), (5, 3, 3, False), (4, 4, 3, True)])
def test_header_forms_against_decode_header(label, writer, w, h, mips, cube):
    m, msg = check_header(writer(w, h, mips, cube))
    assert m is not None and m["format"] in C.LOADED, msg


def ambiguous():
    """Legacy headers whose flags or masks make g_LegacyDDSMap's order matter for the converted forms, plus section 13's set."""
    return TU.ambiguous() + [
        (U.RGB | U.FOURCC, 112, 32, 0xffff, 0xffff0000, 0, 0),      # G16R16's masks come before FourCC 112
        (U.RGB | U.FOURCC, 113, 32, 0xff0000, 0xff00, 0xff, 0xff000000),   # A8R8G8B8's masks (WIC) win over FourCC 113
        (U.RGB | U.FOURCC, 113, 16, 0x1, 0x2, 0x4, 0x8),             # masks of no entry: FourCC 113
        (U.RGBA, 0, 16, 0xf00, 0xf0, 0xf, 0),                         # X4R4G4B4's masks under RGBA: X4R4G4B4
        (U.RGB, 0, 16, 0xf00, 0xf0, 0xf, 0xf000),                     # A4R4G4B4's masks under RGB: A4R4G4B4 (flags intersect)
        (U.LUMA | U.ALPHA, 0, 8, 0, 0, 0, 0xff),                      # A8's masks under LUMINANCE | ALPHA: A8
        (U.LUM | U.ALPHA, 0, 16, 0xff, 0, 0, 0xff00),                 # A8L8's masks without ALPHAPIXELS: A8L8
        (U.RGB | U.LUM, 0, 32, 0xffff, 0xffff0000, 0, 0)]             # G16R16's masks under RGB | LUMINANCE


@pytest.mark.parametrize("cube", [False, True])
def test_legacy_headers_in_table_order(cube):
    """Every g_LegacyDDSMap entry and the ambiguous headers resolve as _GetDXGIFormat resolves them."""
    seen = set()
    for pf in TU.legacy_table() + ambiguous():
        m = U.ref_header(np.frombuffer(U.header(4, 4, 1, pf, cube), np.uint8).copy())
        fmt = None if m is None else m["format"]
        tb = C.LOADED[fmt][1] if fmt in C.LOADED else 16
        file = np.frombuffer(U.header(4, 4, 1, pf, cube) + bytes(U.payload_bytes(4, 4, 1, 6 if cube else 1, tb)), np.uint8).copy()
        check_header(file)
        seen.add(fmt)
    assert set(C.LOADED) - {16, 10, 54, 34, 13, 35, 49, 65, 115} == {37, 58, 26, 67, 51, 31, 63}   # the DX10-only formats
    assert {35, 49, 65, 115, 13, 54, 34, 10, 16} <= seen


def expected_refusal(loaded):
    """The reason the product must give for a loaded format it does not serve, from the compiled reference functions."""
    if (70 <= loaded <= 84) or (94 <= loaded <= 99):
        return "itw_dds_open"
    target, _ = C.ref_target(loaded)
    if loaded == target:
        return "itw_dds_open_uncompressed"
    if C.ref().ref_use_wic(loaded, target):
        return "WIC"
    if loaded == 6:
        return "runtime"
    return "not opened here"


def test_scope_against_use_wic_conversion():
    """For every DXGI id a 'DX10' header can name and every legacy form: the product opens the file iff its loaded format is one of
    the served formats; every served (loaded, DoReadStart target) pair is non-WIC by the compiled _UseWICConversion; the product's
    target, depth and alpha decision are the reference's BitsPerColor / IsSRGB rule and HasAlpha; every refusal names its reason."""
    for f in range(1, 121):
        file = np.frombuffer(U.header(4, 4, dx10=(f, 3, 0, 1)) + bytes(4 * 4 * 16), np.uint8).copy()
        m = U.ref_header(file)
        ok, _, msg = verdict(file)
        served = m is not None and f in C.LOADED
        assert ok == served, (f, msg)
        kind, target, depth, has_alpha = C.emu_scope(f)
        assert (kind >= 0) == (f in C.LOADED), f
        if served:
            want_target, want_depth = C.ref_target(f)
            assert f != want_target and not C.ref().ref_use_wic(f, want_target), f
            assert (target, depth, has_alpha) == (want_target, want_depth, C.ref().ref_has_alpha(f)), f
        elif m is not None:
            assert expected_refusal(f) in msg, (f, msg)
    for pf in TU.legacy_table():
        head = U.header(4, 4, 1, pf)
        m = U.ref_header(np.frombuffer(head, np.uint8).copy())
        ok, _, msg = verdict(np.frombuffer(head + bytes(4 * 4 * 16), np.uint8).copy())
        if m is None:
            assert not ok, (pf, msg)
            continue
        loaded = m["format"]
        assert ok == (loaded in C.LOADED and not m["conv"] & 0x1), (pf, msg)
        if ok:
            assert not C.ref().ref_use_wic(loaded, C.ref_target(loaded)[0]), pf
        elif (70 <= loaded <= 84) or (94 <= loaded <= 99):
            assert "itw_dds_open" in msg, (pf, msg)
        elif m["conv"] & 0x1:                                          # CONV_FLAGS_EXPAND
            assert "expansion" in msg or "itw_dds_open_uncompressed" in msg, (pf, msg)
        else:
            assert expected_refusal(loaded) in msg, (pf, msg)


REFUSED_DX10 = {2: "itw_dds_open_uncompressed", 11: "itw_dds_open_uncompressed", 28: "itw_dds_open_uncompressed",
                29: "itw_dds_open_uncompressed", 71: "itw_dds_open", 98: "itw_dds_open", 6: "runtime", 87: "WIC", 88: "WIC", 91: "WIC",
                93: "WIC", 85: "WIC", 86: "WIC", 24: "WIC", 89: "WIC", 61: "WIC", 56: "WIC", 41: "WIC", 40: "WIC", 55: "WIC", 42: "not opened here",
                12: "not opened here", 107: "not opened here", 68: "not opened here", 113: "palettised"}


@pytest.mark.parametrize("fmt,text", sorted(REFUSED_DX10.items()))
def test_dx10_refusals(fmt, text):
    file = np.frombuffer(U.header(4, 4, dx10=(fmt, 3, 0, 1)) + b"\0" * 256, np.uint8).copy()
    ok, _, msg = verdict(file)
    assert not ok and text in msg, msg


LEGACY_REFUSED = {"A8R8G8B8": ((U.RGBA, 0, 32, 0xff0000, 0xff00, 0xff, 0xff000000), "WIC"),
                  "R5G6B5": ((U.RGB, 0, 16, 0xf800, 0x07e0, 0x001f, 0), "WIC"),
                  "L8": ((U.LUM, 0, 8, 0xff, 0, 0, 0), "WIC"),
                  "L16": ((U.LUM, 0, 16, 0xffff, 0, 0, 0), "WIC"),
                  "R32F": ((U.FOURCC, 114, 0, 0, 0, 0, 0), "WIC"),
                  "A2B10G10R10": ((U.RGB, 0, 32, 0x3ff00000, 0xffc00, 0x3ff, 0xc0000000), "WIC"),
                  "A8B8G8R8": (U.PF["A8B8G8R8"], "itw_dds_open_uncompressed"),
                  "FourCC36": (U.PF["A16B16G16R16"], "itw_dds_open_uncompressed"),
                  "DXT5": ((U.FOURCC, U.fourcc("DXT5"), 0, 0, 0, 0, 0), "itw_dds_open"),
                  "YUY2": ((U.FOURCC, U.fourcc("YUY2"), 0, 0, 0, 0, 0), "not opened here"),
                  "P8": ((0x20, 0, 8, 0, 0, 0, 0), "expansion")}


@pytest.mark.parametrize("name", sorted(LEGACY_REFUSED))
def test_legacy_refusals(name):
    pf, text = LEGACY_REFUSED[name]
    file = np.frombuffer(U.header(4, 4, pf=pf) + b"\0" * 256, np.uint8).copy()
    ok, _, msg = verdict(file)
    assert not ok and text in msg, msg


def test_shape_refusals():
    for file, text in [(np.frombuffer(U.header(4, 4, dx10=(10, 4, 0, 1)), np.uint8).copy(), "volume"),
                       (np.frombuffer(U.header(4, 4, dx10=(10, 3, 0, 2)), np.uint8).copy(), "array"),
                       (np.frombuffer(U.header(4, 4, pf=C.LEGACY["A8L8"][0], caps2=0x600), np.uint8).copy(), "six faces"),
                       (C.legacy_file("A8L8", 8, 8)[:-1], "truncated")]:
        info = B.DdsConvertedInfo()
        assert T.product().dds_open_converted_raw(file.ctypes.data, file.size, info) != 0
        assert text in T.product().last_error()
        assert bytes(info) == bytes(B.DdsConvertedInfo())


@pytest.mark.parametrize("options", C.OPTIONS)
@pytest.mark.parametrize("name,cube", [("G16R16", False), ("A8L8", True), ("FourCC115", False), ("FourCC111", True)])
def test_layout_for_every_option(name, cube, options):
    """Formats without alpha: the open is host-only (no scan), so the layout can be checked on the CPU."""
    lib = T.product()
    file = C.legacy_file(name, 6, 5, 3 if not cube else 1, cube)
    info = lib.dds_converted_layout(lib.dds_open_converted(file.ctypes.data, file.size), options)
    m = U.ref_header(file)
    proxy = B.DdsDesc(m["width"], m["height"], m["mip_levels"], m["array_size"], 77, 1 if m["cube"] else 0)
    want = U.open_lib.read_start(proxy, True, options)
    _, _, target, depth, _ = C.LOADED[m["format"]]
    want["target_dxgi"], want["depth"] = target, depth
    assert C.info_fields(info) == {k: want[k] for k in C.info_fields(info)}
    assert info.form == C.LEGACY[name][1] and info.desc.dxgi_format == C.LEGACY[name][2]
