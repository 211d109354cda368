"""The expanded open path (include/itw_bcn.h section 16) on the GPU: every decision and every layer byte for byte against the reference
pipeline of tests/open_expanded_lib.py (the cut _DecodeDDSHeader, LoadFromDDSMemory's palette step, _LegacyExpandScanline with the
palette, the IsAlphaAllOpaque branches and, for A4L4, the non-WIC _Convert, with DoReadStart / DoReadContinue restated), for every
load-dialog answer.  Every form at 1x1, ragged sizes and 257x129 with and without chains, cubes with alpha, one transparent texel in
the deepest mip of a cube's last face, 4096² P8 and A8P8 files with full chains, host and device operands with wide rows, palettes
whose alpha bytes are all 0 or all 0xFF, unreferenced transparent palette entries, and refusals that launch nothing."""
import numpy as np
import pytest

import itw_testlib as T
import open_expanded_lib as E
import open_uncompressed_lib as U

B = T.binding

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if not E.refs_ready():
        pytest.skip("oracle/_ref/libitw_ref_open_expanded.so not built")
    return T.product()


def check_open(lib, file, options=E.OPTIONS):
    """Every option: info and every layer equal the oracle's."""
    file = np.ascontiguousarray(file)
    for opt in options:
        m, start, want = E.oracle_open(file, opt)
        info, got = lib.dds_open_expanded_layers(file, opt)
        d = info.desc
        assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
            (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
        assert info.payload_offset == m["offset"]
        for k, v in E.info_fields(info).items():
            assert v == start[k], (k, v, start[k], opt)
        assert len(got) == len(want)
        for c, (g, w) in enumerate(zip(got, want)):
            assert g.shape == w.shape
            if g.tobytes() != w.tobytes():
                bad = np.flatnonzero(g != w)
                raise AssertionError(f"option {opt} call {c}: {bad.size} bytes differ, first at {bad[0]}")
    return info


@pytest.mark.parametrize("name", sorted(E.FORMS))
def test_every_form(lib, name):
    for w, h, mips, cube, seed in ((1, 1, 1, False, 1), (5, 3, 1, False, 2), (5, 3, 3, False, 3), (7, 9, 1, False, 4),
                                   (7, 9, 4, False, 5), (257, 129, 1, False, 6), (257, 129, 9, False, 7), (3, 3, 2, True, 8)):
        check_open(lib, E.file_of(name, w, h, mips, cube, seed=seed))


@pytest.mark.parametrize("name", sorted(E.FORMS))
def test_cube_with_alpha_forces_the_last_plane(lib, name):
    info = check_open(lib, E.file_of(name, 6, 6, 3, True, seed=21))      # random alphas: has_alpha holds, the last plane is forced
    assert info.desc.array_size == 6 and info.has_alpha


# an opaque texel of each form and a transparent one (P8 / A8P8 through the palette below: entry 1 opaque, entry 2 transparent)
OPAQUE = {"P8": b"\x01", "A8P8": b"\x01\x00", "A8R3G3B2": b"\x5a\xff", "A4L4": b"\xf7"}
CLEAR = {"P8": b"\x02", "A8P8": b"\x02\x00", "A8R3G3B2": b"\x5a\xfc", "A4L4": b"\xe7"}


@pytest.mark.parametrize("name", sorted(E.FORMS))
def test_one_transparent_texel_in_the_deepest_mip_of_the_last_face(lib, name):
    pal = E.random_palette(5, 0x00)
    pal[1] |= np.uint32(0xFF000000)
    w, h, mips = 37, 20, 6
    n = U.payload_bytes(w, h, mips, 6, E.FORMS[name][3]) // E.FORMS[name][3]
    pay = bytearray(OPAQUE[name] * n)
    for has in (False, True):
        if has:
            at = len(pay) - E.FORMS[name][3]                               # the one texel of the last face's 1x1 level
            pay[at:at + E.FORMS[name][3]] = CLEAR[name]
        info = check_open(lib, E.file_of(name, w, h, mips, True, payload=bytes(pay), palette=pal), options=(0,))
        assert info.has_alpha == has, (name, has)


@pytest.mark.parametrize("name", ["P8", "A8P8"])
def test_4096_with_full_chain(lib, name):
    check_open(lib, E.file_of(name, 4096, 4096, 13, seed=11), options=(0, B.OPEN_MIPS))


def test_palette_alpha_all_zero_opens_transparent(lib):
    """A P8 palette whose fourth bytes are all 0 (peFlags, not alpha, in many D3D9 writers): the layers are transparent."""
    file = E.file_of("P8", 33, 17, 3, palette=E.random_palette(9, 0x00), seed=9)
    info = check_open(lib, file)
    assert info.has_alpha
    _, loaded = E.ref_load(file)
    assert (loaded.reshape(-1, 4)[:, 3] == 0).all()               # every loaded texel's alpha is 0


def test_a8p8_palette_alpha_all_ff_is_opaque(lib):
    """A8P8 alpha is the palette alpha OR'd with the texel's: an all-0xFF palette alpha makes every texel opaque."""
    info = check_open(lib, E.file_of("A8P8", 29, 31, 5, palette=E.random_palette(10, 0xFF), seed=10))
    assert not info.has_alpha


def test_unreferenced_transparent_entries_do_not_count(lib):
    pal = E.random_palette(12, 0x00)
    used = np.arange(0, 256, 5, dtype=np.uint8)
    pal[used] |= np.uint32(0xFF000000)
    for w, h, mips in ((1, 1, 1), (13, 7, 4), (300, 2, 3)):
        n = U.payload_bytes(w, h, mips, 1, 1)
        info = check_open(lib, E.file_of("P8", w, h, mips, payload=np.resize(used, n).tobytes(), palette=pal), options=(0,))
        assert not info.has_alpha, (w, h, mips)


def test_host_and_device_operands(lib):
    """Host and device files, host and device layers, and wider rows whose bytes outside the layer stay untouched."""
    import torch
    for file in (E.file_of("P8", 45, 19, 3, seed=6), E.file_of("A8P8", 31, 9, 2, True, seed=7), E.file_of("A8R3G3B2", 13, 7, 2, seed=8),
                 E.file_of("A4L4", 45, 19, 3, seed=9)):
        for opt in (0, B.OPEN_MIPS):
            info = lib.dds_expanded_layout(lib.dds_open_expanded(file.ctypes.data, file.size), opt)
            _, _, want = E.oracle_open(file, opt)
            d_file = torch.from_numpy(file.copy()).cuda()
            dinfo = lib.dds_expanded_layout(lib.dds_open_expanded(d_file.data_ptr(), file.size), opt)
            assert bytes(dinfo) == bytes(info)
            tight = info.width * info.planes
            for call in range(info.calls):
                w8 = np.ascontiguousarray(want[call]).reshape(info.height, tight)
                for row in (0, tight + 3, (tight + 15) // 16 * 16 + 32):
                    pitch = row or tight
                    host = np.full((info.height, pitch), 0xAB, np.uint8)
                    assert lib.dds_read_expanded_layer_raw(file.ctypes.data, file.size, info, call, host.ctypes.data, row) == 0
                    assert np.array_equal(host[:, :tight], w8) and (host[:, tight:] == 0xAB).all(), (opt, call, row)
                    dev = torch.full((info.height * pitch + 16,), 0xAB, dtype=torch.uint8, device="cuda")
                    for off, src in ((0, d_file.data_ptr()), (4, file.ctypes.data)):
                        dev.fill_(0xAB)
                        assert lib.dds_read_expanded_layer_raw(src, file.size, info, call, dev.data_ptr() + off, row) == 0
                        got = dev.cpu().numpy()
                        assert (got[:off] == 0xAB).all() and (got[off + info.height * pitch:] == 0xAB).all()
                        got = got[off:off + info.height * pitch].reshape(info.height, pitch)
                        assert np.array_equal(got[:, :tight], w8) and (got[:, tight:] == 0xAB).all(), (opt, call, row, off)


def test_refusals_launch_nothing_and_older_calls_still_refuse(lib):
    import torch
    file = E.file_of("P8", 8, 8, 1, seed=1)
    info = lib.dds_expanded_layout(lib.dds_open_expanded(file.ctypes.data, file.size), 0)
    r332 = np.frombuffer(U.header(8, 8, 1, E.R3G3B2) + bytes(64), np.uint8).copy()
    d_bad = torch.from_numpy(r332).cuda()
    d_short = torch.from_numpy(file[:1151].copy()).cuda()
    dev = torch.full((8 * 8 * 4,), 0x3C, dtype=torch.uint8, device="cuda")
    before = lib.launch_count()
    out = B.DdsExpandedInfo()
    assert lib.dds_open_expanded_raw(d_bad.data_ptr(), r332.size, out) != 0 and "WIC" in lib.last_error()
    assert lib.dds_open_expanded_raw(d_short.data_ptr(), 1151, out) != 0 and "palette" in lib.last_error()
    assert bytes(out) == bytes(B.DdsExpandedInfo())
    assert lib.dds_read_expanded_layer_raw(d_bad.data_ptr(), r332.size, info, 0, dev.data_ptr()) != 0
    assert lib.dds_read_expanded_layer_raw(file.ctypes.data, file.size - 1, info, 0, dev.data_ptr()) != 0
    assert lib.launch_count() == before and (dev.cpu().numpy() == 0x3C).all()
    for name in E.FORMS:                         # the calls of sections 9, 13, 14 and 15 keep refusing these files
        f = E.file_of(name, 4, 4, 1, seed=2)
        assert lib.dds_open_uncompressed_raw(f.ctypes.data, f.size, B.DdsUncompressedInfo()) != 0, name
        assert lib.dds_open_converted_raw(f.ctypes.data, f.size, B.DdsConvertedInfo()) != 0, name
        assert lib.dds_open_other_bc_raw(f.ctypes.data, f.size, B.DdsOtherBcInfo()) != 0, name
        with pytest.raises(RuntimeError):
            lib.dds_open(f.ctypes.data, f.size)


def test_kernel_time_is_reported(lib):
    for name in E.FORMS:
        file = E.file_of(name, 256, 256, 1, seed=2)
        info = lib.dds_expanded_layout(lib.dds_open_expanded(file.ctypes.data, file.size), 0)
        assert lib.last_kernel_ms() > 0
        out = np.empty((info.height, info.width, info.planes), np.uint8)
        assert lib.dds_read_expanded_layer_raw(file.ctypes.data, file.size, info, 0, out.ctypes.data) == 0
        assert lib.last_kernel_ms() > 0
