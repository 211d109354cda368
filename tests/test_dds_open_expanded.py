"""The expanded open path on the CPU (include/itw_bcn.h section 16): the per-texel rule of the layer kernel (emulated) against the
reference's own _LegacyExpandScanline (with a real palette) and, for A4L4, its non-WIC _Convert, over whole value domains; the scan's
alpha predicate against the cut IsAlphaAllOpaque branches for every alpha value in every slot of the scan's word; header parsing against
_DecodeDDSHeader and LoadFromDDSMemory's palette step; the scope over every legacy form and 'DX10' id; the refusals (all before any
CUDA call) and the layout."""
import numpy as np
import pytest

import itw_testlib as T
import open_converted_lib as C
import open_expanded_lib as E
import open_uncompressed_lib as U
import test_dds_open_uncompressed as TU       # section 13's g_LegacyDDSMap headers

B = T.binding

pytestmark = pytest.mark.skipif(not E.refs_ready(), reason="oracle/_ref/libitw_ref_open_expanded.so not built")

EXPAND, PAL8_FLAG, F44, F332, F8332 = 0x1, 0x8, 0x100, 0x200, 0x400
PALETTES = {"alpha00": E.random_palette(1, 0x00), "alphaFF": E.random_palette(2, 0xFF), "random": E.random_palette(3)}


def domain(name):
    """Every source texel of the form: every byte (P8, A4L4), every ushort (A8P8, A8R3G3B2)."""
    return np.arange(256 if E.FORMS[name][3] == 1 else 65536, dtype=np.uint8 if E.FORMS[name][3] == 1 else np.uint16).tobytes()


@pytest.mark.parametrize("name,pal", [("P8", p) for p in PALETTES] + [("A8P8", p) for p in PALETTES] + [("A8R3G3B2", None), ("A4L4", None)])
def test_per_texel_rule_against_the_reference(name, pal):
    src = domain(name)
    palette = None if pal is None else PALETTES[pal]
    want = E.ref_texels(name, src, palette)
    got = E.emu_texels(name, 4, src, palette)
    assert np.array_equal(got, want), f"{int((got != want).sum())} bytes differ"
    three = E.emu_texels(name, 3, src, palette)
    assert np.array_equal(three.reshape(-1, 3), got.reshape(-1, 4)[:, :3])
    forced = E.emu_texels(name, 4, src, palette, force=True).reshape(-1, 4)
    assert (forced[:, 3] == 255).all() and np.array_equal(forced[:, :3], got.reshape(-1, 4)[:, :3])


def test_a4l4_loads_as_b4g4r4a4():
    """The 4:4 expansion itself: the loaded 115 texel of every A4L4 byte."""
    src = domain("A4L4")
    l, a = np.arange(256) & 0xF, np.arange(256) >> 4
    want = (l | l << 4 | l << 8 | a << 12).astype("<u2")
    assert np.array_equal(E.ref_expand("A4L4", src).view("<u2"), want)


@pytest.mark.parametrize("name,pal", [("P8", p) for p in PALETTES] + [("A8P8", p) for p in PALETTES] + [("A8R3G3B2", None), ("A4L4", None)])
def test_alpha_predicate_for_every_alpha_value(name, pal):
    """The scan's predicate is IsAlphaAllOpaque's on the loaded texel, for every source texel in every slot of the scan's word."""
    _, _, loaded, tb, _ = E.FORMS[name]
    palette = None if pal is None else PALETTES[pal].copy()
    fill = 0xFF if tb == 1 else 0xFFFF             # an opaque neighbour: alpha nibble 15, alpha byte 255 (A8P8: ORed to 255)
    if name == "P8":
        palette[0xFF] |= np.uint32(0xFF000000)     # P8's neighbour is index 255, made opaque
    src = domain(name)
    want = 1 - E.ref_opaque(loaded, E.ref_expand(name, src, palette))
    for slot in range(4 // tb):
        assert np.array_equal(E.emu_below(name, src, slot, palette, fill), want), slot
    if name == "A8P8" and pal == "alphaFF":
        assert not want.any()                      # an opaque palette entry makes every A8P8 texel opaque
    if name == "A8P8" and pal == "alpha00":
        assert np.array_equal(want, (np.arange(65536) >> 8 <= 252).astype(np.uint8))


def test_unreferenced_palette_entries_do_not_count():
    """A P8 palette with transparent entries that no texel uses: every texel the payload holds is opaque to the scan and the cut."""
    pal = E.random_palette(7, 0x00)
    used = np.arange(0, 256, 3, dtype=np.uint8)
    pal[used] |= np.uint32(0xFF000000)
    payload = np.resize(used, 64 * 4 + 3).tobytes()
    m, loaded = E.ref_load(E.file_of("P8", 259, 1, payload=payload, palette=pal))
    assert U.ref().ref_is_alpha_all_opaque(28, loaded.ctypes.data, m["width"], m["height"], 1, 1) == 1
    for slot in range(4):
        assert not E.emu_below("P8", payload, slot, pal, fill=int(used[0])).any()


def verdict(file):
    """Open the file with its payload one byte short (every accepted header then fails at its size check, before any CUDA call)."""
    lib = T.product()
    f = np.ascontiguousarray(file[:-1])
    info = B.DdsExpandedInfo()
    before = bytes(info)
    launches = lib.launch_count()
    assert lib.dds_open_expanded_raw(f.ctypes.data, f.size, info) != 0
    assert bytes(info) == before and lib.launch_count() == launches
    msg = lib.last_error()
    assert msg.startswith("itw_dds_open_expanded: "), msg
    if "truncated file" in msg:
        return True, int(msg.split("needs ")[1].rstrip(")")), msg
    return False, None, msg


@pytest.mark.parametrize("name", sorted(E.FORMS))
@pytest.mark.parametrize("w,h,mips,cube", [(1, 1, 1, False), (5, 3, 3, False), (7, 9, 4, False), (4, 4, 3, True)])
def test_header_forms_against_load_from_dds_memory(name, w, h, mips, cube):
    """The product's verdict and size against LoadFromDDSMemory: the file loads, it needs exactly its bytes (palette included), and
    one byte less fails in both."""
    file = E.file_of(name, w, h, mips, cube, seed=w + h)
    m, loaded = E.ref_load(file)
    assert m is not None and m["format"] == E.FORMS[name][2] and m["offset"] == (1152 if E.has_palette(name) else 128)
    assert (m["width"], m["height"], m["mip_levels"], m["array_size"], m["cube"]) == (w, h, mips, 6 if cube else 1, int(cube))
    assert E.ref_load(file[:-1])[0] is None
    ok, need, msg = verdict(file)
    assert ok and need == file.size, msg
    form, fmt, pal, tb = E.emu_scope(E.FORMS[name][1])
    assert (form, fmt, pal, tb) == (E.FORMS[name][4], E.FORMS[name][2], int(E.has_palette(name)), E.FORMS[name][3])


def test_scope_over_every_legacy_form_and_dx10_id():
    """The call opens exactly P8, A8P8, A8R3G3B2 and A4L4; every other file is refused with the call that serves it or the reason.
    The compiled _UseWICConversion sends R3G3B2's 85 -> 28 to WIC and A4L4's 115 -> 28 to the non-WIC _Convert."""
    assert C.ref().ref_use_wic(85, 28) == 1 and C.ref().ref_use_wic(115, 28) == 0
    opened = set()
    for pf in TU.legacy_table():
        m = U.ref_header(np.frombuffer(U.header(4, 4, 1, pf), np.uint8).copy())
        pal = bytes(1024) if pf[0] == E.PAL8 else b""
        tight = 4 * 4 * (pf[2] // 8 if pf[2] else 16)            # the accepted forms' exact payload, which verdict() cuts short
        ok, _, msg = verdict(np.frombuffer(U.header(4, 4, 1, pf) + pal + bytes(tight), np.uint8).copy())
        if m is None:
            assert not ok, (pf, msg)
            continue
        conv = m["conv"]
        assert ok == bool(conv & EXPAND and conv & (PAL8_FLAG | F44 | F8332)), (pf, msg)
        if ok:
            opened.add(pf)
            continue
        fmt = m["format"]
        if conv & F332:
            assert "WIC" in msg and "R3G3B2" in msg, msg
        elif pf in (U.PF["A8B8G8R8"], U.PF["X8B8G8R8"], U.PF["R8G8B8"], U.PF["A16B16G16R16"], U.PF["A32B32G32R32F"]):
            assert "itw_dds_open_uncompressed" in msg, (pf, msg)
        elif fmt in (74, 81, 84) or (fmt == 77 and conv & 0x20000):            # DXT2 / DXT3 / BC4S / BC5S / DXT4 (premultiplied)
            assert "itw_dds_open_other_bc" in msg, (pf, msg)
        elif 70 <= fmt <= 99:
            assert "itw_dds_open" in msg and "other_bc" not in msg, (pf, msg)
        elif fmt in C.LOADED:
            assert "itw_dds_open_converted" in msg, (pf, msg)
        else:
            assert "WIC" in msg or "not opened here" in msg, (pf, msg)
    assert opened == {v[0] for v in E.FORMS.values()}
    for f in range(1, 121):
        file = np.frombuffer(U.header(4, 4, dx10=(f, 3, 0, 1)) + bytes(4 * 4 * 16), np.uint8).copy()
        ok, _, msg = verdict(file)
        assert not ok, f
        if f in (113, 114):
            assert U.ref_header(file) is None and "palettised" in msg and str(f) in msg, msg
        elif (70 <= f <= 84 or 94 <= f <= 99) and f not in (71, 72, 77, 78, 80, 83, 95, 96, 98, 99):
            assert "itw_dds_open_other_bc" in msg, (f, msg)
        elif 70 <= f <= 99 and (f <= 84 or f >= 94):
            assert "itw_dds_open" in msg and "other_bc" not in msg, (f, msg)
        elif f in (2, 11, 28, 29):
            assert "itw_dds_open_uncompressed" in msg, (f, msg)
        elif f in C.LOADED:
            assert "itw_dds_open_converted" in msg, (f, msg)
        elif U.ref_header(file) is not None:
            assert "WIC" in msg or "not opened here" in msg, (f, msg)


def refused(file, text):
    lib = T.product()
    info = B.DdsExpandedInfo()
    launches = lib.launch_count()
    assert lib.dds_open_expanded_raw(file.ctypes.data, file.size, info) != 0
    msg = lib.last_error()
    assert text in msg and msg.startswith("itw_dds_open_expanded: "), msg
    assert bytes(info) == bytes(B.DdsExpandedInfo()) and lib.launch_count() == launches
    return msg


def test_refusals_launch_nothing_and_leave_info_untouched():
    p8 = E.file_of("P8", 8, 8)
    refused(np.ascontiguousarray(p8[:1151]), "palette")
    refused(np.ascontiguousarray(p8[:1152 + 63]), "truncated")
    refused(np.ascontiguousarray(E.file_of("A4L4", 8, 8)[:-1]), "truncated")
    refused(np.frombuffer(U.header(8, 8, 1, E.R3G3B2) + bytes(64), np.uint8).copy(), "WIC")
    refused(np.frombuffer(U.header(4, 4, dx10=(113, 3, 0, 1)) + bytes(256), np.uint8).copy(), "palettised")
    refused(np.frombuffer(U.header(4, 4, dx10=(114, 3, 0, 1)) + bytes(256), np.uint8).copy(), "palettised")
    refused(np.frombuffer(U.header(4, 4, 1, E.FORMS["P8"][0], hflags=0x00801007) + bytes(2048), np.uint8).copy(), "volume")
    refused(np.frombuffer(U.header(4, 4, 1, E.FORMS["A8R3G3B2"][0], caps2=0x600) + bytes(256), np.uint8).copy(), "six faces")
    refused(np.frombuffer(U.header(0, 4, 1, E.FORMS["A4L4"][0]) + bytes(256), np.uint8).copy(), "width or height 0")
    refused(np.frombuffer(U.header((1 << 24) + 1, 1, 1, E.FORMS["A4L4"][0]) + bytes(256), np.uint8).copy(), "above 16777216")
    refused(np.frombuffer(U.header(4, 4, 4, E.FORMS["A8P8"][0]) + bytes(2048), np.uint8).copy(), "mip levels")
    refused(np.frombuffer(U.header(4, 4, 1, U.PF["A8B8G8R8"]) + bytes(256), np.uint8).copy(), "itw_dds_open_uncompressed")
    refused(np.frombuffer(U.header(4, 4, 1, C.LEGACY["A4R4G4B4"][0]) + bytes(256), np.uint8).copy(), "itw_dds_open_converted")
    refused(np.frombuffer(U.header(4, 4, 1, (U.FOURCC, U.fourcc("DXT3"), 0, 0, 0, 0, 0)) + bytes(256), np.uint8).copy(), "itw_dds_open_other_bc")
    refused(np.frombuffer(U.header(4, 4, 1, (U.FOURCC, U.fourcc("DXT1"), 0, 0, 0, 0, 0)) + bytes(256), np.uint8).copy(), "itw_dds_open")


def test_layer_reads_refuse_before_any_cuda_call():
    lib = T.product()
    file = E.file_of("A8P8", 8, 8)
    info = B.DdsExpandedInfo()
    info.desc = B.DdsDesc(8, 8, 1, 1, 28, 0)
    info.form, info.payload_offset = B.EXP_A8P8, 1152
    lib.dds_expanded_layout(info, 0)
    out = np.full((8, 8, 3), 0x5A, np.uint8)
    launches = lib.launch_count()
    for f, size, inf, call, text in [(file, file.size - 1, info, 0, "truncated"), (file, file.size, info, 1, "call out of range"),
                                     (E.file_of("P8", 8, 8), 8 * 8 + 1152, info, 0, "does not match")]:
        assert lib.dds_read_expanded_layer_raw(f.ctypes.data, size, inf, call, out.ctypes.data) != 0
        assert text in lib.last_error(), lib.last_error()
    bad = B.DdsExpandedInfo.from_buffer_copy(bytes(info))
    bad.payload_offset = 128
    assert lib.dds_read_expanded_layer_raw(file.ctypes.data, file.size, bad, 0, out.ctypes.data) != 0
    assert "not a description" in lib.last_error()
    assert lib.launch_count() == launches and (out == 0x5A).all()


@pytest.mark.parametrize("options", E.OPTIONS)
@pytest.mark.parametrize("name,w,h,mips,cube,alpha", [("P8", 6, 5, 3, False, 1), ("A8P8", 6, 5, 1, False, 0), ("A8R3G3B2", 4, 4, 1, True, 1),
                                                      ("A4L4", 9, 2, 4, False, 0), ("A4L4", 3, 3, 1, True, 0)])
def test_layout_for_every_option(name, w, h, mips, cube, alpha, options):
    """The layout is pure arithmetic on the description the open call gives (the header's, with has_alpha as the scan leaves it)."""
    lib = T.product()
    m, _ = E.ref_load(E.file_of(name, w, h, mips, cube))
    info = B.DdsExpandedInfo()
    info.desc = B.DdsDesc(w, h, mips, 6 if cube else 1, m["format"], int(cube))
    info.form, info.payload_offset, info.has_alpha = E.FORMS[name][1], m["offset"], alpha
    info.has_mips = int(mips > 1)
    info.ask_user = int(not cube and (alpha or mips > 1))
    wrong = B.DdsExpandedInfo.from_buffer_copy(bytes(info))
    wrong.desc.dxgi_format = 115 if m["format"] == 28 else 28
    assert lib.dds_expanded_layout_raw(wrong, options) != 0 and "not a description" in lib.last_error()
    lib.dds_expanded_layout(info, options)
    assert lib.last_error() == ""
    proxy = B.DdsDesc(w, h, mips, 6 if cube else 1, 77, int(cube))
    want = U.open_lib.read_start(proxy, not alpha, options)
    want["target_dxgi"], want["depth"] = 28, 8
    assert E.info_fields(info) == {k: want[k] for k in E.info_fields(info)}
