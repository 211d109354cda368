"""The uncompressed open path on the CPU (include/itw_bcn.h section 13): header parsing against the reference's own _DecodeDDSHeader,
the refusals (all before any CUDA call), the layout, the alpha thresholds against the cut IsAlphaAllOpaque branch, and the per-texel
rule of the layer kernel (emulated) against the reference's row copies."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import open_uncompressed_lib as U

B = T.binding

pytestmark = pytest.mark.skipif(U.ref() is None, reason="oracle/_ref/libitw_ref_open_uncompressed.so not built")

ACCEPTED_CONV = (0x0, 0x2, 0x13)          # none, NOALPHA (X8B8G8R8), EXPAND | NOALPHA | 888 (R8G8B8); CONV_FLAGS_DX10 masked
SHAPES = [(1, 1, 1, False), (5, 3, 3, False), (7, 9, 1, False), (4, 4, 3, True), (3, 2, 1, True)]


def product():
    return T.product()


def verdict(file):
    """Open the header of `file` alone: an accepted header fails only at the size check, whose message states the size the header
    needs (no CUDA call is reached either way).  Returns (accepted, needed size or None, message)."""
    lib = product()
    dx10 = file.size >= 148 and bytes(file[84:88]) == b"DX10"
    f = np.ascontiguousarray(file[:min(file.size, 148 if dx10 else 128)])
    info = B.DdsUncompressedInfo()
    assert lib.dds_open_uncompressed_raw(f.ctypes.data, f.size, info) != 0
    msg = lib.last_error()
    assert msg.startswith("itw_dds_open_uncompressed: "), msg
    if "truncated file" in msg:
        return True, int(msg.split("needs ")[1].rstrip(")")), msg
    return False, None, msg


def ref_accepts(file):
    m = U.ref_header(file)
    return m is not None and m["format"] in U.TARGETS and (m["conv"] & ~0x10000) in ACCEPTED_CONV and m["dimension"] == 3 and \
        (m["array_size"] == 1 or (m["cube"] and m["array_size"] == 6))


def all_forms(w, h, mips, cube, seed=0):
    files = [(n, U.legacy_file(n, w, h, mips, cube, seed=seed)) for n in U.PF]
    files += [(f"DX10-{f}", U.dx10_file(f, w, h, mips, cube, seed=seed)) for f in (2, 11, 28, 29)]
    return files


@pytest.mark.parametrize("w,h,mips,cube", SHAPES)
def test_accepted_headers_parse_as_the_reference(w, h, mips, cube):
    for name, f in all_forms(w, h, mips, cube):
        m = U.ref_header(f)
        assert m is not None and ref_accepts(f), name
        ok, need, msg = verdict(f)
        assert ok and need == f.size, (name, msg)
        # the size the header needs is the payload offset plus the payload of the loaded description
        src = U.SRC_BYTES.get(name, U.TEXEL[m["format"]])
        assert need == m["offset"] + U.payload_bytes(w, h, m["mip_levels"], m["array_size"], src)


@pytest.mark.parametrize("name", ["X8B8G8R8", "R8G8B8"])
@pytest.mark.parametrize("w,h,mips,cube", SHAPES)
def test_opaque_forms_open_without_a_scan(name, w, h, mips, cube):
    """X8B8G8R8 and R8G8B8 load with alpha 255: itw_dds_open_uncompressed needs no CUDA call for them."""
    f = U.legacy_file(name, w, h, mips, cube)
    m = U.ref_header(f)
    info = product().dds_open_uncompressed(f.ctypes.data, f.size)
    d = info.desc
    assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
        (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
    assert info.source == U.SOURCES[name] and info.payload_offset == m["offset"] == 128
    assert info.has_alpha == 0 and info.has_mips == (mips > 1) and info.ask_user == (not cube and mips > 1)
    assert product().last_kernel_ms() < 0


def test_dx10_headers_on_legacy_formats_keep_their_offset():
    """28 behind a 'DX10' header (texconv -dx10): the payload starts at 148, not where the library would write it."""
    f = U.dx10_file(28, 6, 5, 3)
    assert U.ref_header(f)["offset"] == 148
    ok, need, _ = verdict(f)
    assert ok and need == 148 + U.payload_bytes(6, 5, 3, 1, 4)


def legacy_table():
    """Every g_LegacyDDSMap entry's pixel format (DDS.h and the table's inline entries)."""
    cc = U.fourcc
    pfs = [(U.FOURCC, cc(s), 0, 0, 0, 0, 0) for s in ("DXT1", "DXT3", "DXT5", "DXT2", "DXT4", "BC4U", "BC4S", "BC5U", "BC5S", "ATI1", "ATI2",
                                                      "RGBG", "GRGB", "YUY2", "UYVY")]
    pfs += [(U.FOURCC, v, 0, 0, 0, 0, 0) for v in (36, 110, 111, 112, 113, 114, 115, 116)]
    pfs += [(U.RGBA, 0, 32, 0xff0000, 0xff00, 0xff, 0xff000000), (U.RGB, 0, 32, 0xff0000, 0xff00, 0xff, 0),
            U.PF["A8B8G8R8"], U.PF["X8B8G8R8"], (U.RGB, 0, 32, 0xffff, 0xffff0000, 0, 0),
            (U.RGB, 0, 32, 0x3ff, 0xffc00, 0x3ff00000, 0xc0000000), (U.RGB, 0, 32, 0x3ff00000, 0xffc00, 0x3ff, 0xc0000000),
            U.PF["R8G8B8"], (U.RGB, 0, 16, 0xf800, 0x7e0, 0x1f, 0), (U.RGBA, 0, 16, 0x7c00, 0x3e0, 0x1f, 0x8000),
            (U.RGB, 0, 16, 0x7c00, 0x3e0, 0x1f, 0), (U.RGB, 0, 16, 0xe0, 0x1c, 0x3, 0xff00), (U.RGB, 0, 8, 0xe0, 0x1c, 0x3, 0),
            (U.LUM, 0, 8, 0xff, 0, 0, 0), (U.LUM, 0, 16, 0xffff, 0, 0, 0), (U.LUMA, 0, 16, 0xff, 0, 0, 0xff00), (U.ALPHA, 0, 8, 0, 0, 0, 0xff),
            (U.RGB, 0, 32, 0xffffffff, 0, 0, 0), (U.PAL8, 0, 16, 0, 0, 0, 0), (U.PAL8, 0, 8, 0, 0, 0, 0),
            (U.RGBA, 0, 16, 0xf00, 0xf0, 0xf, 0xf000), (U.RGB, 0, 16, 0xf00, 0xf0, 0xf, 0), (U.LUM, 0, 8, 0xf, 0, 0, 0xf0)]
    return pfs


def ambiguous():
    """Headers whose flags or masks make the table's order matter."""
    a8b8 = U.PF["A8B8G8R8"][1:]
    return [(0x1,) + a8b8,                       # DDPF_ALPHAPIXELS alone intersects every RGBA / LUMINANCEA entry
            (U.RGB,) + a8b8,                     # DDS_RGB with an alpha mask: A8B8G8R8's masks
            (U.RGB | U.FOURCC, 36, 32, 0xff, 0xff00, 0xff0000, 0xff000000),   # both: the FourCC entry comes later than A8B8G8R8
            (U.RGB | U.FOURCC, 113, 32, 0xff, 0xff00, 0xff0000, 0),           # X8B8G8R8's masks win over FourCC 113
            (U.RGBA | U.LUM, 0, 16, 0xff, 0, 0, 0xff00),                      # A8L8's masks under RGBA | LUMINANCE
            (U.RGB, 0, 24, 0xff0000, 0xff00, 0xff, 0xff),                     # 24 bits with an alpha mask: no entry
            (U.RGB, 0, 32, 0xff, 0xff00, 0xff0000, 0x1),                      # an odd alpha mask: no entry
            (U.PAL8 | U.RGB, 0, 24, 0xff0000, 0xff00, 0xff, 0),               # PAL8 entries compare the bit count only
            (U.PAL8, 0, 8, 0xff, 0xff, 0xff, 0xff),
            (U.FOURCC, U.fourcc("DX11"), 0, 0, 0, 0, 0), (0x0,) + a8b8]


@pytest.mark.parametrize("cube", [False, True])
def test_legacy_pixel_formats_follow_the_table_order(cube):
    seen = set()
    for pf in legacy_table() + ambiguous():
        bits = pf[2] if pf[2] in (24, 32) else 32
        payload = b"\0" * (U.payload_bytes(3, 2, 1, 6 if cube else 1, max(bits // 8, 16)))
        f = np.frombuffer(U.header(3, 2, 1, pf, cube) + payload, np.uint8).copy()
        want = ref_accepts(f)
        ok, need, msg = verdict(f)
        assert ok == want, (hex(pf[0]), pf[1:], msg)
        if not ok:
            seen.add(msg)
    assert len(seen) >= 30                       # every refused form says what it is


REFUSED_DX10 = [0, 1, 3, 10, 13, 24, 41, 54, 61, 65, 85, 87, 88, 91, 107, 111, 113, 114, 115, 121, 200, 71, 72, 77, 80, 83, 95, 96, 98, 99]


def refused_files():
    out = [(f"dx10-{f}", np.frombuffer(U.header(4, 4, dx10=(f, 3, 0, 1)) + b"\0" * 256, np.uint8).copy()) for f in REFUSED_DX10]
    out += [("dx10-1d", np.frombuffer(U.header(4, 1, dx10=(28, 2, 0, 1)) + b"\0" * 64, np.uint8).copy()),
            ("dx10-volume", np.frombuffer(U.header(4, 4, hflags=0x801007, dx10=(28, 4, 0, 1)) + b"\0" * 64, np.uint8).copy()),
            ("dx10-array", np.frombuffer(U.header(4, 4, dx10=(28, 3, 0, 2)) + b"\0" * 128, np.uint8).copy()),
            ("dx10-cube-array", np.frombuffer(U.header(4, 4, dx10=(28, 3, 4, 2)) + b"\0" * 768, np.uint8).copy()),
            ("dx10-array-0", np.frombuffer(U.header(4, 4, dx10=(28, 3, 0, 0)) + b"\0" * 64, np.uint8).copy()),
            ("legacy-volume", np.frombuffer(U.header(4, 4, hflags=0x801007) + b"\0" * 64, np.uint8).copy()),
            ("partial-cube", np.frombuffer(U.header(4, 4, caps2=0x0600) + b"\0" * 64, np.uint8).copy()),
            ("too-many-mips", np.frombuffer(U.header(4, 4, 4) + b"\0" * 128, np.uint8).copy()),
            ("zero-width", np.frombuffer(U.header(0, 4) + b"\0" * 64, np.uint8).copy()),
            ("huge", np.frombuffer(U.header(1 << 25, 1), np.uint8).copy()),
            ("not-dds", np.frombuffer(b"DDX " + U.header(4, 4)[4:] + b"\0" * 64, np.uint8).copy()),
            ("short", np.frombuffer(U.header(4, 4)[:100], np.uint8).copy()),
            ("dx10-short", np.frombuffer(U.header(4, 4, dx10=(28, 3, 0, 1))[:140], np.uint8).copy()),
            ("truncated", U.legacy_file("A8B8G8R8", 4, 4)[:-4].copy())]
    for name in ("A8R8G8B8", "X8R8G8B8", "R5G6B5", "A1R5G5B5", "A4R4G4B4", "L8", "L16", "A8L8", "A2B10G10R10", "G16R16", "P8", "A8P8",
                 "A8R3G3B2", "A4L4", "DXT1", "DXT5", "113"):
        pf = {"A8R8G8B8": (U.RGBA, 0, 32, 0xff0000, 0xff00, 0xff, 0xff000000), "X8R8G8B8": (U.RGB, 0, 32, 0xff0000, 0xff00, 0xff, 0),
              "R5G6B5": (U.RGB, 0, 16, 0xf800, 0x7e0, 0x1f, 0), "A1R5G5B5": (U.RGBA, 0, 16, 0x7c00, 0x3e0, 0x1f, 0x8000),
              "A4R4G4B4": (U.RGBA, 0, 16, 0xf00, 0xf0, 0xf, 0xf000), "L8": (U.LUM, 0, 8, 0xff, 0, 0, 0), "L16": (U.LUM, 0, 16, 0xffff, 0, 0, 0),
              "A8L8": (U.LUMA, 0, 16, 0xff, 0, 0, 0xff00), "A2B10G10R10": (U.RGB, 0, 32, 0x3ff00000, 0xffc00, 0x3ff, 0xc0000000),
              "G16R16": (U.RGB, 0, 32, 0xffff, 0xffff0000, 0, 0), "P8": (U.PAL8, 0, 8, 0, 0, 0, 0), "A8P8": (U.PAL8, 0, 16, 0, 0, 0, 0),
              "A8R3G3B2": (U.RGB, 0, 16, 0xe0, 0x1c, 0x3, 0xff00), "A4L4": (U.LUM, 0, 8, 0xf, 0, 0, 0xf0),
              "DXT1": (U.FOURCC, U.fourcc("DXT1"), 0, 0, 0, 0, 0), "DXT5": (U.FOURCC, U.fourcc("DXT5"), 0, 0, 0, 0, 0),
              "113": (U.FOURCC, 113, 0, 0, 0, 0, 0)}[name]
        out.append((name, np.frombuffer(U.header(4, 4, 1, pf) + b"\0" * 2048, np.uint8).copy()))
    return out


def test_refusals_touch_nothing_and_launch_nothing():
    lib = product()
    before = lib.launch_count()
    messages = {}
    for name, f in refused_files():
        info = B.DdsUncompressedInfo()
        ctypes.memset(ctypes.byref(info), 0x5A, ctypes.sizeof(info))
        snap = bytes(info)
        assert lib.dds_open_uncompressed_raw(f.ctypes.data, f.size, info) != 0, name
        msg = lib.last_error()
        assert msg.startswith("itw_dds_open_uncompressed: ") and bytes(info) == snap, (name, msg)
        messages[name] = msg
        # the read call parses the same header first: dst untouched
        dst = np.full(64, 0xA5, np.uint8)
        assert lib.dds_read_uncompressed_layer_raw(f.ctypes.data, f.size, good_info(), 0, dst.ctypes.data) != 0
        assert (dst == 0xA5).all() and lib.last_error().startswith("itw_dds_read_uncompressed_layer: ")
    assert lib.launch_count() == before
    for bc in ("dx10-71", "DXT1", "DXT5"):
        assert "itw_dds_open" in messages[bc]
    for conv in ("A8R8G8B8", "X8R8G8B8", "113", "dx10-87", "dx10-10"):
        assert "Convert" in messages[conv]
    for exp in ("P8", "A8P8", "A8R3G3B2", "A4L4"):
        assert "expansion" in messages[exp]
    assert "volume" in messages["legacy-volume"] and "volume" in messages["dx10-volume"]
    assert "six faces" in messages["partial-cube"] and "array" in messages["dx10-array"]
    assert "truncated" in messages["truncated"] and "16777216" in messages["huge"]
    distinct = {messages[n] for n in ("A8R8G8B8", "X8R8G8B8", "R5G6B5", "L8", "A8L8", "G16R16", "P8", "A8P8", "A4L4", "113")}
    assert len(distinct) == 10


def good_info(w=4, h=4, mips=1, fmt=28, source=B.RAW_A8B8G8R8, cube=False, has_alpha=0, options=0):
    info = B.DdsUncompressedInfo()
    info.desc = B.DdsDesc(w, h, mips, 6 if cube else 1, fmt, 1 if cube else 0)
    info.source, info.payload_offset, info.has_alpha, info.has_mips = source, 148 if source == B.RAW_DX10 else 128, has_alpha, mips > 1
    product().dds_uncompressed_layout(info, options)
    return info


LAYOUT_CASES = [(fmt, src) for fmt, src in ((28, B.RAW_A8B8G8R8), (28, B.RAW_X8B8G8R8), (28, B.RAW_R8G8B8), (11, B.RAW_A16B16G16R16),
                                            (2, B.RAW_A32B32G32R32F), (2, B.RAW_DX10), (11, B.RAW_DX10), (28, B.RAW_DX10), (29, B.RAW_DX10))]


@pytest.mark.parametrize("fmt,source", LAYOUT_CASES)
def test_layout_is_doreadstarts(fmt, source):
    for w, h, mips, cube in [(8, 4, 1, False), (8, 4, 4, False), (5, 5, 3, True), (5, 5, 1, True)]:
        for has_alpha in (0, 1):
            for options in U.OPTIONS:
                info = good_info(w, h, mips, fmt, source, cube, has_alpha, options)
                m = dict(width=w, height=h, mip_levels=mips, array_size=6 if cube else 1, format=fmt, cube=int(cube))
                want = U.read_start(m, not has_alpha, options)
                got = U.info_fields(info)
                for k in ("layers", "calls", "planes", "depth", "width", "height", "target_dxgi"):
                    assert got[k] == want[k], (k, fmt, source, w, h, mips, cube, has_alpha, options)


def test_layout_refusals():
    lib = product()
    bad = [B.DdsDesc(4, 4, 1, 1, 77, 0), B.DdsDesc(4, 4, 1, 2, 28, 0), B.DdsDesc(4, 4, 4, 1, 28, 0), B.DdsDesc(0, 4, 1, 1, 28, 0),
           B.DdsDesc(4, 4, 1, 6, 28, 0), B.DdsDesc(4, 4, 1, 1, 11, 0)]
    for d in bad:
        info = B.DdsUncompressedInfo()
        info.desc, info.source = d, B.RAW_A8B8G8R8
        snap = bytes(info)
        assert lib.dds_uncompressed_layout_raw(info, 0) != 0 and bytes(info) == snap
    info = good_info()
    assert lib.dds_uncompressed_layout_raw(info, 4) != 0 and "option" in lib.last_error()
    assert lib.dds_uncompressed_layout_raw(None, 0) != 0


def test_read_refusals_before_any_cuda_call():
    lib = product()
    f = U.legacy_file("X8B8G8R8", 4, 4, 3)
    info = lib.dds_uncompressed_layout(lib.dds_open_uncompressed(f.ctypes.data, f.size), B.OPEN_MIPS)
    dst = np.full(4 * 4 * 4 + 64, 0xA5, np.uint8)
    before = lib.launch_count()
    cases = [(f, info, 3, 0, "call out of range"), (f, info, -1, 0, "call out of range"), (f, info, 0, 8, "row_bytes"),
             (f, good_info(4, 4, 3, 28, B.RAW_A8B8G8R8, options=B.OPEN_MIPS), 0, 0, "does not match"),
             (U.legacy_file("X8B8G8R8", 4, 4, 2), info, 0, 0, "does not match")]
    for file, inf, call, rb, text in cases:
        assert lib.dds_read_uncompressed_layer_raw(file.ctypes.data, file.size, inf, call, dst.ctypes.data, rb) != 0
        assert text in lib.last_error()
    unlaid = B.DdsUncompressedInfo.from_buffer_copy(info)
    unlaid.planes = 2
    assert lib.dds_read_uncompressed_layer_raw(f.ctypes.data, f.size, unlaid, 0, dst.ctypes.data) != 0
    assert "not laid out" in lib.last_error()
    assert lib.dds_read_uncompressed_layer_raw(0, f.size, info, 0, dst.ctypes.data) != 0
    assert lib.dds_read_uncompressed_layer_raw(f.ctypes.data, f.size, info, 0, 0) != 0
    assert (dst == 0xA5).all() and lib.launch_count() == before


def float_edges():
    n = np.float32(0.99)
    vals = [n, np.nextafter(n, np.float32(0)), np.nextafter(n, np.float32(2)), np.float32(np.nan), np.float32(-np.nan), np.float32(0.0),
            np.float32(-0.0), np.float32(np.inf), np.float32(-np.inf), np.float32(1.0), np.float32(0.98999), np.float32(2.0)]
    raw = np.array(vals, np.float32).view(np.uint32)
    raw = np.concatenate([raw, np.array([0x7FC00001, 0xFFFFFFFF, 0x00000001, 0x80000001], np.uint32)])
    return raw.view(np.float32)


def test_alpha_thresholds_match_the_cut_branch():
    # UNORM8: every byte; UNORM16: every ushort; float: 0.99f, its neighbours and the specials
    for fmt, kind, alphas, texel in ((28, 0, np.arange(256, dtype=np.uint8), 4), (11, 3, np.arange(65536, dtype=np.uint16), 8),
                                     (2, 4, float_edges(), 16)):
        tex = np.zeros((alphas.size, 4), alphas.dtype)
        tex[:, :3] = np.asarray(1, alphas.dtype)
        tex[:, 3] = alphas
        raw = np.ascontiguousarray(tex).view(np.uint8).reshape(-1)
        want = np.zeros(alphas.size, np.uint8)
        U.ref().ref_texels_opaque(fmt, raw.ctypes.data, alphas.size, want.ctypes.data)
        got = np.zeros(alphas.size, np.uint8)
        assert U.emu().emu_raw_alpha_below(kind, raw.ctypes.data, alphas.size, got.ctypes.data) == 0
        assert np.array_equal(got, 1 - want), fmt
    # the thresholds hold whichever way the normalisation is written (v * (1/n) or v / n)
    for n, lo in ((255, 252), (65535, 64879)):
        for v, below in ((lo, True), (lo + 1, False)):
            assert (np.float32(v) * (np.float32(1) / np.float32(n)) < np.float32(0.99)) == below
            assert (np.float32(v) / np.float32(n) < np.float32(0.99)) == below
    assert U.ref().ref_convert_to_16bit_255() == 0x3C00


@pytest.mark.parametrize("name", list(U.PF))
def test_emulated_texel_rule_matches_the_reference(name):
    """The layer kernel's per-texel routines (emulated) against the reference's row path and the plug-in's copy loop."""
    rng = np.random.default_rng(7)
    n = 4096
    src = rng.integers(0, 256, n * U.SRC_BYTES[name], dtype=np.uint8)
    if name == "A32B32G32R32F":
        src = rng.normal(0.5, 2.0, n * 4).astype(np.float32).view(np.uint8)
        src[:64] = float_edges()[:16].view(np.uint8)
    f = U.legacy_file(name, n, 1, payload=src.tobytes())
    m, loaded = U.ref_load(f)
    fmt = m["format"]
    img = loaded.view(U.DTYPES[fmt]).reshape(n, 4)
    forced = {28: 255, 11: U.ref().ref_convert_to_16bit_255(), 2: np.float32(1.0)}[fmt]
    for planes in (3, 4):
        for force in (0, 1):
            want = img[:, :planes].copy()
            if force:
                want[:, planes - 1] = forced
            got = U.emu_texels(U.KIND[name], planes, src, force)
            assert got.tobytes() == np.ascontiguousarray(want).tobytes(), (name, planes, force)
