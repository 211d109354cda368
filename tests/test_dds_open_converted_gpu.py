"""The converted open path (include/itw_bcn.h section 14) on the GPU: every decision and every layer byte for byte against the
reference pipeline of tests/open_converted_lib.py (the cut _DecodeDDSHeader, _LoadScanline, _ConvertScanline, _StoreScanline and
IsAlphaAllOpaque branch, with DoReadStart / DoReadContinue restated), for every load-dialog answer.  Every header form at 1x1, ragged
sizes and 257x129, four forms at 4096² with full chains, cubes with alpha, the alpha thresholds, host and device operands with wide rows,
an HDR file of values above 1 and below 0, and the refusals of the section 9 and 13 calls."""
import numpy as np
import pytest

import itw_testlib as T
import open_converted_lib as C
import open_uncompressed_lib as U

B = T.binding

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if C.ref() is None or U.ref() is None:
        pytest.skip("oracle/_ref/libitw_ref_open_converted.so not built")
    return T.product()


def check_open(lib, file, options=C.OPTIONS):
    """Every option: info and every layer equal the oracle's."""
    file = np.ascontiguousarray(file)
    for opt in options:
        m, start, want = C.oracle_open(file, opt)
        info, got = lib.dds_open_converted_layers(file, opt)
        d = info.desc
        assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
            (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
        assert info.payload_offset == m["offset"]
        for k, v in C.info_fields(info).items():
            assert v == start[k], (k, v, start[k], opt)
        assert len(got) == len(want)
        for c, (g, w) in enumerate(zip(got, want)):
            assert g.dtype == w.dtype and g.shape == w.shape
            if g.tobytes() != w.tobytes():
                bad = np.flatnonzero(g.view(np.uint8) != w.view(np.uint8))
                raise AssertionError(f"option {opt} call {c}: {bad.size} bytes differ, first at {bad[0]}")
    return info


@pytest.mark.parametrize("label,writer", C.FORMS, ids=[f[0] for f in C.FORMS])
def test_every_header_form(lib, label, writer):
    for w, h, mips, cube, seed in ((1, 1, 1, False, 1), (5, 3, 3, False, 2), (7, 9, 4, False, 3), (3, 3, 1, True, 4),
                                   (257, 129, 9, False, 5)):
        check_open(lib, writer(w, h, mips, cube, seed=seed))


@pytest.mark.parametrize("label", ["FourCC113", "DX10-26", "A4R4G4B4", "G16R16"])
def test_4096_with_full_chain(lib, label):
    writer = dict(C.FORMS)[label]
    check_open(lib, writer(4096, 4096, 13, False, seed=11), options=(0, B.OPEN_MIPS))


@pytest.mark.parametrize("label", ["A4R4G4B4", "FourCC113", "FourCC110", "A8", "DX10-31"])
def test_cube_with_alpha_forces_the_last_plane(lib, label):
    file = dict(C.FORMS)[label](6, 6, 1, True, seed=21)               # random alphas: has_alpha holds, the last plane is forced
    info = check_open(lib, file)
    assert info.desc.array_size == 6 and info.has_alpha


# (label, texel bytes, offset of the alpha in the texel, alpha bytes, an alpha just below 0.99, one at or above it)
THRESHOLDS = [("FourCC113", 8, 6, 2, 0x3BEB, 0x3BEC), ("FourCC110", 8, 6, 2, 32439, 32440), ("DX10-31", 4, 3, 1, 125, 126),
              ("A8", 1, 0, 1, 252, 253), ("A4R4G4B4", 2, 0, 2, 0xEFFF, 0xF000)]


@pytest.mark.parametrize("label,tb,at,ab,below,above", THRESHOLDS)
def test_alpha_either_side_of_099(lib, label, tb, at, ab, below, above):
    writer = dict(C.FORMS)[label]
    for w, h, mips in ((1, 1, 1), (9, 5, 3), (64, 33, 2)):
        n = U.payload_bytes(w, h, mips, 1, tb)
        base = np.frombuffer(writer(w, h, mips, False, seed=3)[-n:].tobytes(), np.uint8).copy().reshape(-1, tb)
        for i in range(base.shape[0]):               # every texel opaque first
            base[i, at:at + ab] = np.frombuffer(int(above if label != "A4R4G4B4" else 0xFFFF).to_bytes(ab, "little"), np.uint8)
        for pos in (0, base.shape[0] // 2, base.shape[0] - 1):
            for a, has in ((above, False), (below, True)):
                pay = base.copy()
                pay[pos, at:at + ab] = np.frombuffer(int(a).to_bytes(ab, "little"), np.uint8)
                info = check_open(lib, writer(w, h, mips, False, payload=pay.tobytes()), options=(0,))
                assert info.has_alpha == has, (label, w, h, mips, pos, a)


def test_hdr_values_in_fourcc_113(lib):
    """A FourCC 113 file of the HDR corpus's values (above 1, negative, zero, tiny) saturates into the 16-bit layer as the reference
    converts it."""
    import hdr_corpus
    halves = np.asarray(hdr_corpus.log_uniform(48, 64, seed=5), np.uint16)
    file = C.legacy_file("FourCC113", 64, 48, 1, False, payload=halves.tobytes())
    check_open(lib, file)


def test_host_and_device_operands(lib):
    """Host and device files, host and device layers, and wider rows whose bytes outside the layer stay untouched."""
    import torch
    forms = dict(C.FORMS)
    for file in (forms["FourCC113"](45, 19, 3, False, seed=6), forms["A8"](45, 19, 3, False, seed=7),
                 forms["A4R4G4B4"](31, 9, 2, True, seed=8), forms["FourCC115"](13, 7, 2, False, seed=9)):
        for opt in (0, B.OPEN_MIPS):
            info = lib.dds_converted_layout(lib.dds_open_converted(file.ctypes.data, file.size), opt)
            _, _, want = C.oracle_open(file, opt)
            d_file = torch.from_numpy(file.copy()).cuda()
            dinfo = lib.dds_converted_layout(lib.dds_open_converted(d_file.data_ptr(), file.size), opt)
            assert bytes(dinfo) == bytes(info)
            tight = info.width * info.planes * info.depth // 8
            for call in range(info.calls):
                w8 = np.ascontiguousarray(want[call]).view(np.uint8).reshape(info.height, tight)
                for row in (0, tight + 3, (tight + 15) // 16 * 16 + 32):
                    pitch = row or tight
                    host = np.full((info.height, pitch), 0xAB, np.uint8)
                    assert lib.dds_read_converted_layer_raw(file.ctypes.data, file.size, info, call, host.ctypes.data, row) == 0
                    assert np.array_equal(host[:, :tight], w8) and (host[:, tight:] == 0xAB).all(), (opt, call, row)
                    dev = torch.full((info.height * pitch + 16,), 0xAB, dtype=torch.uint8, device="cuda")
                    for off, src in ((0, d_file.data_ptr()), (4, file.ctypes.data)):
                        dev.fill_(0xAB)
                        assert lib.dds_read_converted_layer_raw(src, file.size, info, call, dev.data_ptr() + off, row) == 0
                        got = dev.cpu().numpy()
                        assert (got[:off] == 0xAB).all() and (got[off + info.height * pitch:] == 0xAB).all()
                        got = got[off:off + info.height * pitch].reshape(info.height, pitch)
                        assert np.array_equal(got[:, :tight], w8) and (got[:, tight:] == 0xAB).all(), (opt, call, row, off)


def test_refusals_launch_nothing_and_older_calls_still_refuse(lib):
    import torch
    file = C.legacy_file("FourCC113", 8, 8, 1, False, seed=1)
    info = lib.dds_converted_layout(lib.dds_open_converted(file.ctypes.data, file.size), 0)
    bad = np.frombuffer(U.header(8, 8, 1, (0x41, 0, 32, 0xff0000, 0xff00, 0xff, 0xff000000)) + bytes(256), np.uint8).copy()
    d_bad = torch.from_numpy(bad).cuda()
    dev = torch.full((8 * 8 * 8,), 0x3C, dtype=torch.uint8, device="cuda")
    before = lib.launch_count()
    out = B.DdsConvertedInfo()
    assert lib.dds_open_converted_raw(d_bad.data_ptr(), bad.size, out) != 0 and "WIC" in lib.last_error()
    assert lib.dds_read_converted_layer_raw(d_bad.data_ptr(), bad.size, info, 0, dev.data_ptr()) != 0
    assert lib.dds_read_converted_layer_raw(file.ctypes.data, file.size - 1, info, 0, dev.data_ptr()) != 0
    assert lib.launch_count() == before and (dev.cpu().numpy() == 0x3C).all()
    for label, writer in C.FORMS:                   # sections 9 and 13 keep refusing every converted file
        f = writer(4, 4, 1, False, seed=2)
        assert lib.dds_open_uncompressed_raw(f.ctypes.data, f.size, B.DdsUncompressedInfo()) != 0, label
        with pytest.raises(RuntimeError):
            lib.dds_open(f.ctypes.data, f.size)


def test_kernel_time_is_reported(lib):
    file = C.legacy_file("FourCC113", 256, 256, 1, False, seed=2)
    lib.dds_open_converted(file.ctypes.data, file.size)
    assert lib.last_kernel_ms() > 0
    g = C.legacy_file("G16R16", 256, 256, 1, False, seed=2)
    lib.dds_open_converted(g.ctypes.data, g.size)
    assert lib.last_kernel_ms() < 0                                # no scan for a format without alpha
