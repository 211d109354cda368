"""The uncompressed open path (include/itw_bcn.h section 13) on the GPU: every decision and every layer byte for byte against the
reference pipeline of tests/open_uncompressed_lib.py (the cut _DecodeDDSHeader, _CopyImage row paths and IsAlphaAllOpaque branch,
with DoReadStart / DoReadContinue restated), for every load-dialog answer.  Files of itw_dds_save_none, synthetic files of every header
form, cubes with alpha at depths 8, 16 and 32, the alpha thresholds, host and device operands, and a round trip through the save."""
import numpy as np
import pytest

import itw_testlib as T
import open_uncompressed_lib as U
import preview_uncompressed_lib as P

B = T.binding
NO = B.NoneOptions
D2, CR, LY = B.PANE_2D, B.PANE_CUBE_CROSS, B.PANE_CUBE_LAYERS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if U.ref() is None:
        pytest.skip("oracle/_ref/libitw_ref_open_uncompressed.so not built")
    return T.product()


def check_open(lib, file, options=U.OPTIONS):
    """Every option: info and every layer equal the oracle's."""
    file = np.ascontiguousarray(file)
    for opt in options:
        m, start, want = U.oracle_open(file, opt)
        info, got = lib.dds_open_uncompressed_layers(file, opt)
        d = info.desc
        assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
            (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
        assert info.payload_offset == m["offset"]
        fields = U.info_fields(info)
        for k, v in fields.items():
            assert v == start[k], (k, v, start[k], opt)
        assert len(got) == len(want)
        for c, (g, w) in enumerate(zip(got, want)):
            assert g.dtype == w.dtype and g.shape == w.shape
            if g.tobytes() != w.tobytes():
                bad = np.flatnonzero(g.view(np.uint8) != w.view(np.uint8))
                raise AssertionError(f"option {opt} call {c}: {bad.size} bytes differ, first at {bad[0]}")
    return info


@pytest.mark.parametrize("texture,mips,level,flags", [(D2, 0, -1, 0), (D2, 1, -1, B.FRONT_HAS_ALPHA), (D2, 1, -1, B.FRONT_FLIP_X |
                                                      B.FRONT_NORMALIZE), (CR, 1, -1, 0), (CR, 0, -1, B.FRONT_HAS_ALPHA), (CR, 1, 2, 0),
                                                      (LY, 1, -1, B.FRONT_HAS_ALPHA), (LY, 1, 1, B.FRONT_HAS_ALPHA)])
def test_files_of_the_none_save(lib, texture, mips, level, flags):
    for depth in (8, 16, 32):
        w, h = (64, 48) if texture == CR else (37, 19)
        doc = P.document(w, h, 4, depth, seed=depth + mips + texture)
        if flags & B.FRONT_HAS_ALPHA:
            doc[..., 3] = doc[..., 3] // 2 if depth != 32 else doc[..., 3] * 0.5
        layers = P.cube_layers(w, h, depth, seed=5) if texture == LY else None
        file = lib.dds_save_none(NO(texture, mips, level), doc, layers, flags)
        check_open(lib, file)


def test_mips_from_layers_file(lib):
    doc = P.document(40, 24, 4, 8, seed=2)
    layers = [P.layer(40, 24, 8, 3, True, seed=3 + i) for i in range(3)]
    file = lib.dds_save_none(NO(D2, 1, -1), doc, layers, B.FRONT_HAS_ALPHA)
    check_open(lib, file)


FORMS = [(n, None) for n in U.PF] + [("DX10", f) for f in (2, 11, 28, 29)]


def synthetic(name, fmt, w, h, mips, cube, seed, alpha=None):
    """A file of every header form; `alpha` (when given) overwrites every loaded alpha of an RGBA form."""
    src = U.SRC_BYTES[name] if fmt is None else U.TEXEL[fmt]
    n = U.payload_bytes(w, h, mips, 6 if cube else 1, src)
    rng = np.random.default_rng(seed)
    if (fmt or {"A16B16G16R16": 11, "A32B32G32R32F": 2}.get(name)) == 2:
        payload = rng.uniform(-0.5, 1.5, n // 4).astype(np.float32)
        if alpha is not None:
            payload.reshape(-1, 4)[:, 3] = alpha
    else:
        payload = rng.integers(0, 256, n, dtype=np.uint8)
        if alpha is not None and src in (4, 8):
            payload.view(np.uint8 if src == 4 else np.uint16).reshape(-1, 4)[:, 3] = alpha
    payload = payload.tobytes()
    return U.legacy_file(name, w, h, mips, cube, payload) if fmt is None else U.dx10_file(fmt, w, h, mips, cube, payload)


@pytest.mark.parametrize("name,fmt", FORMS)
def test_every_header_form(lib, name, fmt):
    for w, h, mips, cube in [(1, 1, 1, False), (37, 19, 6, False), (130, 3, 3, False), (17, 17, 5, True), (5, 7, 1, True)]:
        check_open(lib, synthetic(name, fmt, w, h, mips, cube, seed=w + h))
        if name not in ("X8B8G8R8", "R8G8B8"):        # the same with every alpha opaque: no alpha, other layers
            opaque = {None: 255, 28: 255, 29: 255, 11: 65535, 2: 1.0}[fmt if name == "DX10" else
                                                                     {"A16B16G16R16": 11, "A32B32G32R32F": 2}.get(name)]
            check_open(lib, synthetic(name, fmt, w, h, mips, cube, seed=w, alpha=opaque))


@pytest.mark.parametrize("name,fmt", [("A8B8G8R8", None), ("A32B32G32R32F", None), ("R8G8B8", None), ("DX10", 11)])
def test_4096_with_full_chain(lib, name, fmt):
    options = (0, B.OPEN_MIPS) if name == "A8B8G8R8" else (0,)    # mips as layers: thirteen full-size layers per side
    check_open(lib, synthetic(name, fmt, 4096, 4096, 13, False, seed=1), options=options)


@pytest.mark.parametrize("name,fmt,alpha", [("A8B8G8R8", None, 100), ("A16B16G16R16", None, 1000), ("A32B32G32R32F", None, 0.25),
                                            ("DX10", 29, 3)])
def test_cube_with_alpha_forces_the_last_plane(lib, name, fmt, alpha):
    """Depth 8: 255; depth 16: ConvertTo16Bit((unsigned8)255) = 0x3C00; depth 32: 1.0f."""
    file = synthetic(name, fmt, 9, 9, 2, True, seed=3, alpha=alpha)
    info = check_open(lib, file)
    assert info.has_alpha == 1 and info.layers == 6 and info.planes == 4
    _, layers = lib.dds_open_uncompressed_layers(file, 0)
    want = {8: 255, 16: 0x3C00, 32: 1.0}[info.depth]
    assert (layers[0][..., 3] == want).all()


@pytest.mark.parametrize("name,fmt,below,above", [("A8B8G8R8", None, 252, 253), ("A16B16G16R16", None, 64879, 64880),
                                                  ("A32B32G32R32F", None, np.nextafter(np.float32(0.99), np.float32(0)), np.float32(0.99)),
                                                  ("A32B32G32R32F", None, np.float32(0.0), np.float32(np.nan)), ("DX10", 11, 64879, 64880)])
def test_alpha_either_side_of_099(lib, name, fmt, below, above):
    opaque = {"A8B8G8R8": 255, "A16B16G16R16": 65535, "A32B32G32R32F": 1.0, "DX10": 65535}[name]
    for w, h, mips in [(1, 1, 1), (33, 17, 6), (300, 200, 9)]:
        for at in (0, -1):                                         # the first texel of level 0, the last texel of the last level
            for a, has in ((below, 1), (above, 0)):
                file = synthetic(name, fmt, w, h, mips, False, seed=4, alpha=opaque)
                m = U.ref_header(file)
                tex = U.SRC_BYTES.get(name, 8)
                dt = {4: np.uint8, 8: np.uint16, 16: np.float32}[tex]
                pay = file[m["offset"]:].view(dt).reshape(-1, 4)
                pay[at, 3] = a
                info = check_open(lib, file, options=(0,))
                assert info.has_alpha == has, (w, h, mips, at, a)


def test_host_and_device_operands(lib):
    """Host and device files (payload at 128 and at 148, the latter scanned in place from a 4-byte aligned address), host and device
    layers, and wider rows whose bytes outside the layer stay untouched."""
    import torch
    for file in (synthetic("A8B8G8R8", None, 45, 19, 3, False, seed=6), synthetic("DX10", 2, 45, 19, 3, False, seed=7),
                 synthetic("R8G8B8", None, 45, 19, 3, False, seed=8), synthetic("A16B16G16R16", None, 31, 9, 2, True, seed=9, alpha=7)):
        for opt in (0, B.OPEN_MIPS):
            info = lib.dds_uncompressed_layout(lib.dds_open_uncompressed(file.ctypes.data, file.size), opt)
            _, _, want = U.oracle_open(file, opt)
            d_file = torch.from_numpy(file.copy()).cuda()
            dinfo = lib.dds_uncompressed_layout(lib.dds_open_uncompressed(d_file.data_ptr(), file.size), opt)
            assert bytes(dinfo) == bytes(info)
            tight = info.width * info.planes * info.depth // 8
            for call in range(info.calls):
                w8 = np.ascontiguousarray(want[call]).view(np.uint8).reshape(info.height, tight)
                for row in (0, tight + 3, (tight + 15) // 16 * 16 + 32):
                    pitch = row or tight
                    host = np.full((info.height, pitch), 0xAB, np.uint8)
                    assert lib.dds_read_uncompressed_layer_raw(file.ctypes.data, file.size, info, call, host.ctypes.data, row) == 0
                    assert np.array_equal(host[:, :tight], w8) and (host[:, tight:] == 0xAB).all(), (opt, call, row)
                    dev = torch.full((info.height * pitch + 16,), 0xAB, dtype=torch.uint8, device="cuda")
                    for off, src in ((0, d_file.data_ptr()), (4, file.ctypes.data), (0, file.ctypes.data)):
                        dev.fill_(0xAB)
                        assert lib.dds_read_uncompressed_layer_raw(src, file.size, info, call, dev.data_ptr() + off, row) == 0
                        got = dev.cpu().numpy()
                        assert (got[:off] == 0xAB).all() and (got[off + info.height * pitch:] == 0xAB).all()
                        got = got[off:off + info.height * pitch].reshape(info.height, pitch)
                        assert np.array_equal(got[:, :tight], w8) and (got[:, tight:] == 0xAB).all(), (opt, call, row, off)


def test_refusals_against_device_operands_launch_nothing(lib):
    import torch
    file = synthetic("A8B8G8R8", None, 8, 8, 1, False, seed=1)
    info = lib.dds_uncompressed_layout(lib.dds_open_uncompressed(file.ctypes.data, file.size), 0)
    bad = np.frombuffer(U.header(8, 8, 1, (0x41, 0, 32, 0xff0000, 0xff00, 0xff, 0xff000000)) + bytes(256), np.uint8).copy()
    d_bad = torch.from_numpy(bad).cuda()
    dev = torch.full((8 * 8 * 4,), 0x3C, dtype=torch.uint8, device="cuda")
    before = lib.launch_count()
    out = B.DdsUncompressedInfo()
    assert lib.dds_open_uncompressed_raw(d_bad.data_ptr(), bad.size, out) != 0 and "Convert" in lib.last_error()
    assert lib.dds_read_uncompressed_layer_raw(d_bad.data_ptr(), bad.size, info, 0, dev.data_ptr()) != 0
    assert lib.dds_read_uncompressed_layer_raw(file.ctypes.data, file.size - 1, info, 0, dev.data_ptr()) != 0
    assert lib.launch_count() == before and (dev.cpu().numpy() == 0x3C).all()


def test_kernel_time_is_reported(lib):
    file = synthetic("A8B8G8R8", None, 256, 256, 1, False, seed=2)
    lib.dds_open_uncompressed(file.ctypes.data, file.size)
    assert lib.last_kernel_ms() > 0
    x8 = synthetic("X8B8G8R8", None, 256, 256, 1, False, seed=2)
    lib.dds_open_uncompressed(x8.ctypes.data, x8.size)
    assert lib.last_kernel_ms() < 0                                # no scan for a form that loads opaque


def test_round_trip_of_the_none_save(lib):
    """A depth-8, 4-plane document saved with the "none" encoding (no flips, normalise or gamma) and reopened with mips as layers
    gives back its own texels in layer 0."""
    for w, h in ((1, 1), (37, 19), (256, 128)):
        doc = P.document(w, h, 4, 8, seed=w)
        doc[0, 0, 3] = 17                                          # not opaque: the layers keep four planes
        file = lib.dds_save_none(NO(D2, 1, -1), doc, None, B.FRONT_HAS_ALPHA)
        info, layers = lib.dds_open_uncompressed_layers(file, B.OPEN_MIPS)
        assert info.source == B.RAW_A8B8G8R8 and info.depth == 8 and info.planes == 4
        assert np.array_equal(layers[0], doc)
