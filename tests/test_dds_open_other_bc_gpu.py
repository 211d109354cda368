"""The open path for the block-compressed files itw_dds_open does not serve (include/itw_bcn.h section 15) on the GPU: every decision and
every layer byte for byte against the reference pipeline of tests/open_other_bc_lib.py (the cut _DecodeDDSHeader, _IsAlphaAllOpaqueBC and
_DecompressBC with the reference's BC2 / BC4S / BC5S decoders), for every load-dialog answer.  Every header form at 1x1 and ragged sizes,
with and without chains, opaque and not; cubes with alpha; 4096² files with full chains; a non-opaque texel only in the deepest mip of a
cube; host and device operands with wide rows; refusals launch nothing."""
import numpy as np
import pytest

import itw_testlib as T
import open_other_bc_lib as L
import open_uncompressed_lib as U

B = T.binding

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if L.ref() is None or U.ref() is None:
        pytest.skip("oracle/_ref/libitw_ref_open_other_bc.so not built")
    return T.product()


def check_open(lib, file, options=L.OPTIONS):
    """Every option: info and every layer equal the oracle's."""
    file = np.ascontiguousarray(file)
    for opt in options:
        m, start, want = L.oracle_open(file, opt)
        info, got = lib.dds_open_other_bc_layers(file, opt)
        d = info.desc
        assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
            (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
        assert info.payload_offset == m["offset"]
        for k, v in L.info_fields(info).items():
            assert v == start[k], (k, v, start[k], opt)
        assert len(got) == len(want)
        for c, (g, w) in enumerate(zip(got, want)):
            assert g.dtype == w.dtype and g.shape == w.shape
            if g.tobytes() != w.tobytes():
                bad = np.flatnonzero(g.view(np.uint8) != w.view(np.uint8))
                raise AssertionError(f"option {opt} call {c}: {bad.size} bytes differ, first at {bad[0]}")
    return info


@pytest.mark.parametrize("label,fmt,writer", L.FORMS, ids=[f[0] for f in L.FORMS])
def test_every_header_form(lib, label, fmt, writer):
    for w, h, mips, cube, seed in ((1, 1, 1, False, 1), (5, 3, 3, False, 2), (7, 9, 4, False, 3), (3, 3, 1, True, 4),
                                   (257, 129, 9, False, 5), (6, 6, 3, True, 6)):
        info = check_open(lib, writer(w, h, mips, cube, seed=seed))
        if L.LOADED[fmt][4]:                      # and the same shapes with every texel opaque
            assert not check_open(lib, writer(w, h, mips, cube, opaque=True)).has_alpha
        else:
            assert not info.has_alpha


@pytest.mark.parametrize("label", ["DX10-74", "DXT3", "DX10-70"])
def test_cube_with_alpha_forces_the_last_plane(lib, label):
    writer = next(f[2] for f in L.FORMS if f[0] == label)
    info = check_open(lib, writer(6, 6, 1, True, seed=21))             # random alphas: has_alpha holds, the last plane is forced
    assert info.desc.array_size == 6 and info.has_alpha


@pytest.mark.parametrize("label", ["DX10-74", "DX10-70", "DXT4", "DX10-97"])
def test_non_opaque_texel_only_in_the_deepest_mip_of_a_cube(lib, label):
    _, fmt, writer = next(f for f in L.FORMS if f[0] == label)
    w, h, mips = 8, 8, 4
    bpb = L.LOADED[fmt][1]
    pay = bytearray(L.opaque_blocks(fmt, L.payload_bytes(w, h, mips, 6, bpb) // bpb).tobytes())
    at = 6 * L.payload_bytes(w, h, mips, 1, bpb) - bpb               # the 1x1 level of the last face: its texel 0 is transparent
    if fmt == 97:
        pay[at:at + 16] = bytes([0x40] + [0] * 15)                    # mode 6, every endpoint 0: alpha 0
    elif L.LOADED[fmt][0] == 74:
        pay[at] = 0xF0
    elif L.LOADED[fmt][0] == 77:
        pay[at:at + 8] = bytes([255, 255, 6, 0, 0, 0, 0, 0])          # index 6 of the six-value mode: 0
    else:
        pay[at:at + 8] = bytes([0x34, 0x12, 0x78, 0x56, 3, 0, 0, 0])  # three-colour mode, index 3: punch-through
    info = check_open(lib, writer(w, h, mips, True, payload_=bytes(pay)))
    assert info.has_alpha
    pay[at:at + bpb] = L.opaque_blocks(fmt, 1).tobytes()
    assert not check_open(lib, writer(w, h, mips, True, payload_=bytes(pay))).has_alpha


@pytest.mark.parametrize("label", ["DX10-74", "DX10-84", "DX10-94"])
def test_4096_with_full_chain(lib, label):
    writer = next(f[2] for f in L.FORMS if f[0] == label)
    check_open(lib, writer(4096, 4096, 13, False, seed=11), options=(0, B.OPEN_MIPS))


def test_host_and_device_operands(lib):
    """Host and device files, host and device layers, and wider rows whose bytes outside the layer stay untouched."""
    import torch
    forms = {f[0]: f[2] for f in L.FORMS}
    for file in (forms["DXT3"](45, 19, 3, False, seed=6), forms["BC5S"](45, 19, 3, False, seed=7),
                 forms["DX10-70"](31, 9, 2, True, seed=8), forms["DX10-94"](13, 7, 2, False, seed=9)):
        for opt in (0, B.OPEN_MIPS):
            info = lib.dds_other_bc_layout(lib.dds_open_other_bc(file.ctypes.data, file.size), opt)
            _, _, want = L.oracle_open(file, opt)
            d_file = torch.from_numpy(file.copy()).cuda()
            dinfo = lib.dds_other_bc_layout(lib.dds_open_other_bc(d_file.data_ptr(), file.size), opt)
            assert bytes(dinfo) == bytes(info)
            tight = info.width * info.planes * info.depth // 8
            for call in range(info.calls):
                w8 = np.ascontiguousarray(want[call]).view(np.uint8).reshape(info.height, tight)
                for row in (0, tight + 3, (tight + 15) // 16 * 16 + 32):
                    pitch = row or tight
                    host = np.full((info.height, pitch), 0xAB, np.uint8)
                    assert lib.dds_read_other_bc_layer_raw(file.ctypes.data, file.size, info, call, host.ctypes.data, row) == 0
                    assert np.array_equal(host[:, :tight], w8) and (host[:, tight:] == 0xAB).all(), (opt, call, row)
                    dev = torch.full((info.height * pitch + 16,), 0xAB, dtype=torch.uint8, device="cuda")
                    for off, src in ((0, d_file.data_ptr()), (4, file.ctypes.data)):
                        dev.fill_(0xAB)
                        assert lib.dds_read_other_bc_layer_raw(src, file.size, info, call, dev.data_ptr() + off, row) == 0
                        got = dev.cpu().numpy()
                        assert (got[:off] == 0xAB).all() and (got[off + info.height * pitch:] == 0xAB).all()
                        got = got[off:off + info.height * pitch].reshape(info.height, pitch)
                        assert np.array_equal(got[:, :tight], w8) and (got[:, tight:] == 0xAB).all(), (opt, call, row, off)


def test_refusals_launch_nothing_and_older_calls_still_refuse(lib):
    import torch
    file = L.legacy_file("DXT3", 8, 8, 1, False, seed=1)
    info = lib.dds_other_bc_layout(lib.dds_open_other_bc(file.ctypes.data, file.size), 0)
    bad = np.frombuffer(U.header(8, 8, 1, (U.FOURCC, U.fourcc("DXT5"), 0, 0, 0, 0, 0)) + bytes(64), np.uint8).copy()
    d_bad = torch.from_numpy(bad).cuda()
    dev = torch.full((8 * 8 * 4,), 0x3C, dtype=torch.uint8, device="cuda")
    before = lib.launch_count()
    out = B.DdsOtherBcInfo()
    assert lib.dds_open_other_bc_raw(d_bad.data_ptr(), bad.size, out) != 0 and "itw_dds_open" in lib.last_error()
    assert bytes(out) == bytes(B.DdsOtherBcInfo())
    assert lib.dds_read_other_bc_layer_raw(d_bad.data_ptr(), bad.size, info, 0, dev.data_ptr()) != 0
    assert lib.dds_read_other_bc_layer_raw(file.ctypes.data, file.size - 1, info, 0, dev.data_ptr()) != 0
    assert lib.launch_count() == before and (dev.cpu().numpy() == 0x3C).all()
    for label, _, writer in L.FORMS:                # section 9 keeps refusing every one of these files
        f = writer(4, 4, 1, False, seed=2)
        with pytest.raises(RuntimeError):
            lib.dds_open(f.ctypes.data, f.size)


def test_kernel_time_is_reported(lib):
    file = L.legacy_file("DXT3", 256, 256, 1, False, seed=2)
    lib.dds_open_other_bc(file.ctypes.data, file.size)
    assert lib.last_kernel_ms() > 0
    g = L.legacy_file("BC5S", 256, 256, 1, False, seed=2)
    lib.dds_open_other_bc(g.ctypes.data, g.size)
    assert lib.last_kernel_ms() < 0                                # no scan for a format without alpha
