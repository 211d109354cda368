"""The open path on the GPU (itw_dds_open + itw_dds_open_layout + itw_dds_read_layer) against the open oracle of tests/open_lib.py: the
reference's own IsAlphaAllOpaque and DirectX::Decompress, and the plug-in's DoReadStart / DoReadContinue rules.  Every layer of every
call is compared byte for byte, for every answer of the load dialog."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import open_lib as O
import preview_lib as P

B = T.binding
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(O.ref() is None or P.ref() is None, reason="oracle/_ref/libitw_ref_open.so / _preview.so unavailable")]
PROFILES = {98: "alpha_basic", 99: "alpha_basic", 95: "bc6h_basic", 96: "bc6h_basic"}


@pytest.fixture(scope="module")
def lib():
    lib = T.product()
    lib.set_device(0)
    return lib


def _desc_tuple(d):
    return (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap)


def check_open(lib, file, d, options=O.OPTIONS):
    """Open `file` as the plug-in does for each dialog answer; every decision and every layer equals the oracle's."""
    for opt in options:
        start, want = O.oracle_open(file, d, opt)
        info, got = lib.dds_open_layers(file, opt)
        assert _desc_tuple(info.desc) == _desc_tuple(d)
        assert O.info_fields(info) == {k: start[k] for k in O.info_fields(info)}, opt
        assert len(got) == len(want)
        for c, (g, w) in enumerate(zip(got, want)):
            assert g.dtype == w.dtype and g.shape == w.shape, (opt, c)
            if g.tobytes() != w.tobytes():
                bad = np.argwhere((g.view(np.uint8).reshape(g.shape[0], g.shape[1], -1) != w.view(np.uint8).reshape(w.shape[0], w.shape[1], -1)).any(-1))
                raise AssertionError(f"options {opt} layer {c}: {len(bad)} texels differ, first {bad[:4].tolist()}")
    return start


def saved_file(lib, fmt, w, h, mips, cube=False, seed=0):
    """A file written by the library's own save path (itw_dds_encode_pixels)."""
    d = O.desc(w, h, fmt, mips, cube)
    depth = 16 if fmt in (95, 96) else 8
    faces = [P.document(w, h, 4, depth, seed=seed + i) for i in range(d.array_size)]
    if depth == 8:
        for f in faces:                                                  # some transparency in the top level
            f[: max(1, h // 3), :, 3] //= 2
    prof = PROFILES.get(fmt)
    return lib.dds_encode_pixels(d, faces, B.FRONT_HAS_ALPHA, lib.profile(prof) if prof else None), d


@pytest.mark.parametrize("fmt", O.FORMATS)
def test_saved_files_open_like_the_plugin(lib, fmt):
    for w, h in ((1, 1), (5, 3), (130, 67)):
        file, d = saved_file(lib, fmt, w, h, O.full_chain(w, h), seed=w)
        check_open(lib, file, d)
        file, d = saved_file(lib, fmt, w, h, 1, seed=h)
        check_open(lib, file, d, (0, B.OPEN_SEPARATE_ALPHA))


@pytest.mark.parametrize("fmt", [71, 99, 95])
def test_saved_cube_maps_with_mips(lib, fmt):
    file, d = saved_file(lib, fmt, 20, 20, 5, cube=True, seed=fmt)
    start = check_open(lib, file, d, (0, B.OPEN_SEPARATE_ALPHA | B.OPEN_MIPS))
    assert start["layers"] == 6


@pytest.mark.parametrize("fmt", [98, 71])
def test_4096_with_full_chain(lib, fmt):
    file, d = saved_file(lib, fmt, 4096, 4096, 13, seed=1)
    check_open(lib, file, d, (0, B.OPEN_MIPS))


@pytest.mark.parametrize("fourcc,fmt", [("DXT1", 71), ("DXT5", 77), ("ATI1", 80), ("ATI2", 83), ("BC4U", 80), ("BC5U", 83)])
def test_legacy_headers(lib, fourcc, fmt):
    for w, h, mips, cube in ((130, 67, 8, False), (5, 3, 1, False), (8, 8, 4, True)):
        d = O.desc(w, h, fmt, mips, cube)
        file = O.legacy_file(fourcc, w, h, mips, P.random_blocks(fmt, O.payload_bytes(d) // O.bpb(fmt), seed=w + mips), cube)
        check_open(lib, file, d)


@pytest.mark.parametrize("fmt", [71, 77, 80, 83, 72, 99])
def test_dx10_headers(lib, fmt):
    """Files with the 'DX10' extension header for formats this library writes with a legacy one (and for the _SRGB / BC7 formats
    it always writes that way): the payload starts at byte 148, 20 bytes later than the legacy header of the same description."""
    for w, h, mips, cube in ((130, 67, 8, False), (5, 3, 1, False), (12, 12, 4, True)):
        d = O.desc(w, h, fmt, mips, cube)
        file = O.dx10_file(d, P.random_blocks(fmt, O.payload_bytes(d) // O.bpb(fmt), seed=w + mips + fmt))
        check_open(lib, file, d)
    if fmt in (77, 99):                                                             # the alpha scan reads from the right place too
        d = O.desc(37, 21, fmt, 6)
        payload = O.padding_only_payload(d)
        assert not check_open(lib, O.dx10_file(d, payload), d)["has_alpha"]
        payload[-16:] = O.padding_only_block(fmt, 1, 1, inside_bad=True)
        assert check_open(lib, O.dx10_file(d, payload), d)["has_alpha"]


@pytest.mark.parametrize("fmt", [77, 78, 98, 99])
def test_alpha_only_in_the_padding_of_ragged_blocks(lib, fmt):
    """Every image transparent only outside itself (ragged edge blocks of every level, width and height different): opaque.  One
    transparent texel inside the last image, or in the first texel of the top level's last ragged block: not opaque."""
    for w, h, mips, cube in ((37, 21, 6, False), (21, 37, 6, False), (13, 6, 3, True)):
        d = O.desc(w, h, fmt, mips, cube)
        payload = O.padding_only_payload(d)
        start = check_open(lib, O.make_file(d, payload), d)
        assert not start["has_alpha"], (w, h, cube)
        bad = payload.copy()
        bad[-16:] = O.padding_only_block(fmt, 1, 1, inside_bad=True)
        assert check_open(lib, O.make_file(d, bad), d, (0,))["has_alpha"], (w, h, cube)
        bw, bh = (w + 3) // 4, (h + 3) // 4
        bad = payload.copy()
        at = 16 * (bw * bh - 1)                                                     # top level, last block (ragged in both directions)
        bad[at:at + 16] = O.padding_only_block(fmt, w - 4 * (bw - 1), h - 4 * (bh - 1), inside_bad=True)
        assert check_open(lib, O.make_file(d, bad), d, (0,))["has_alpha"], (w, h, cube)


def test_last_kernel_ms_is_not_stale(lib):
    file, d = saved_file(lib, 98, 64, 64, 3, seed=5)
    lib.dds_open(file.ctypes.data, file.size)
    assert lib.last_kernel_ms() >= 0.0
    other, _ = saved_file(lib, 71, 64, 64, 3, seed=5)
    lib.dds_open(other.ctypes.data, other.size)                                     # BC1: no scan, no kernel
    assert lib.last_kernel_ms() == -1.0


def _constant_alpha_file(fmt, w, h, mips, alpha, deep_alpha=None, cube=False):
    """Every block has alpha `alpha`; with deep_alpha, the last (1x1) level of the last item has that alpha instead."""
    d = O.desc(w, h, fmt, mips, cube)
    mk = (lambda a: O.bc3_block(a, a, [0] * 16)) if fmt in (77, 78) else (lambda a: O.bc7_mode6(a, a, [0] * 16))
    n = O.payload_bytes(d) // 16
    payload = np.tile(mk(alpha), n)
    if deep_alpha is not None:
        payload[-16:] = mk(deep_alpha)
    return O.make_file(d, payload), d


@pytest.mark.parametrize("fmt", [77, 78, 98, 99])
def test_alpha_either_side_of_099(lib, fmt):
    for alpha in (252, 253):
        file, d = _constant_alpha_file(fmt, 37, 21, 6, alpha)
        start = check_open(lib, file, d)
        assert start["has_alpha"] == (alpha == 252)
    file, d = _constant_alpha_file(fmt, 37, 21, 6, 255, deep_alpha=252)          # only the 1x1 level is not opaque
    assert check_open(lib, file, d)["has_alpha"]
    file, d = _constant_alpha_file(fmt, 37, 21, 6, 255, deep_alpha=253)
    assert not check_open(lib, file, d)["has_alpha"]


def test_cube_with_alpha_is_forced_white(lib):
    file, d = _constant_alpha_file(98, 12, 12, 4, 255, deep_alpha=10, cube=True)  # alpha only in face 5's deepest mip
    info, layers = lib.dds_open_layers(file, 0)
    assert info.has_alpha and info.layers == 6 and not info.ask_user
    assert all((layer[..., 3] == 255).all() for layer in layers)
    check_open(lib, file, d)
    file, d = _constant_alpha_file(98, 12, 12, 1, 100, cube=True)
    info, layers = lib.dds_open_layers(file, 0)
    assert info.has_alpha and all((layer[..., 3] == 255).all() for layer in layers)
    check_open(lib, file, d)


def test_bc1_punch_through_with_mips(lib):
    d = O.desc(40, 24, 71, 6)
    blocks = P.random_blocks(71, O.payload_bytes(d) // 8, seed=7).reshape(-1, 8)
    blocks[:, 4:] = 0xFF                                                          # every texel index 3
    blocks[::2, 0:4] = (0x00, 0x10, 0xFF, 0xFF)                                  # c0 <= c1: three-colour mode, index 3 transparent
    file = O.make_file(d, blocks.reshape(-1))
    start = check_open(lib, file, d)
    assert not start["has_alpha"]
    info, layers = lib.dds_open_layers(file, B.OPEN_MIPS)
    assert info.planes == 4 and (layers[0][..., 3] == 0).any() and (layers[0][..., 3] == 255).any()


def _expected_layer(file, d, options, call=0):
    start, want = O.oracle_open(file, d, options)
    return want[call]


@pytest.mark.parametrize("fmt", [77, 95])
def test_strides_and_device_operands(lib, fmt):
    """row_bytes 0 / padded / odd, host and device dst, host and device file; padding bytes are never written."""
    import torch
    file, d = saved_file(lib, fmt, 45, 19, 3, seed=4)
    for opt in (0, B.OPEN_MIPS):
        info = lib.dds_open_layout(lib.dds_open(file.ctypes.data, file.size), opt)
        d_file = torch.from_numpy(file.copy()).cuda()
        dinfo = lib.dds_open_layout(lib.dds_open(d_file.data_ptr(), file.size), opt)
        assert bytes(dinfo) == bytes(info)
        tight = info.width * info.planes * info.depth // 8
        for call in range(info.calls):
            want = _expected_layer(file, d, opt, call).view(np.uint8).reshape(info.height, tight)
            for row in (0, tight + 16, tight + 3, (tight + 15) // 16 * 16 + 32):          # the last one 16-byte aligned
                pitch = row or tight
                host = np.full((info.height, pitch), 0xAB, np.uint8)
                lib.dds_read_layer_raw(file.ctypes.data, file.size, info, call, host.ctypes.data, row)
                assert np.array_equal(host[:, :tight], want) and (host[:, tight:] == 0xAB).all(), (opt, call, row)
                dev = torch.full((info.height * pitch + 16,), 0xAB, dtype=torch.uint8, device="cuda")
                for off, src in ((0, file.ctypes.data), (4, d_file.data_ptr())):
                    dev.fill_(0xAB)
                    lib.dds_read_layer_raw(src, file.size, info, call, dev.data_ptr() + off, row)
                    got = dev.cpu().numpy()
                    assert (got[:off] == 0xAB).all() and (got[off + info.height * pitch:] == 0xAB).all()
                    got = got[off:off + info.height * pitch].reshape(info.height, pitch)
                    assert np.array_equal(got[:, :tight], want) and (got[:, tight:] == 0xAB).all(), (opt, call, row, off)


def test_rejected_calls_change_nothing(lib):
    import torch
    file, d = saved_file(lib, 98, 16, 8, 3, seed=2)
    info = lib.dds_open_layout(lib.dds_open(file.ctypes.data, file.size), B.OPEN_MIPS)
    tight = info.width * info.planes
    host = np.full((info.height, tight), 0x3C, np.uint8)
    dev = torch.full((info.height * tight,), 0x3C, dtype=torch.uint8, device="cuda")
    d_file = torch.from_numpy(file.copy()).cuda()

    def rejects(f_ptr, size, inf, call, row_bytes=0):
        for dst in (host.ctypes.data, dev.data_ptr()):
            before = lib.launch_count()
            with pytest.raises(RuntimeError):
                lib.dds_read_layer_raw(f_ptr, size, inf, call, dst, row_bytes)
            assert lib.launch_count() == before
        assert (host == 0x3C).all() and (dev == 0x3C).all().item()

    for f_ptr in (file.ctypes.data, d_file.data_ptr()):
        rejects(f_ptr, file.size - 1, info, 0)                                      # truncated
        rejects(f_ptr, file.size, info, info.calls)                                 # call out of range
        rejects(f_ptr, file.size, info, 0, tight - 1)                               # stride too small
        rejects(f_ptr, file.size, B.DdsOpenInfo(), 0)                               # not laid out
    other = lib.dds_open_layout(lib.dds_open(*_as_ptr(_constant_alpha_file(98, 16, 4, 3, 255)[0])), B.OPEN_MIPS)
    rejects(file.ctypes.data, file.size, other, 0)                                  # info of another file
    f = lib.lib.itw_dds_open
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    before = lib.launch_count()
    scratch = B.DdsOpenInfo()
    assert f(d_file.data_ptr(), file.size - 1, ctypes.addressof(scratch)) != 0 and "truncated" in lib.last_error()
    assert lib.launch_count() == before and bytes(scratch) == bytes(B.DdsOpenInfo())
    lib.dds_open_layout(info, B.OPEN_MIPS)                                           # a call that succeeds clears the last error
    assert lib.last_error() == ""


_keep = []


def _as_ptr(arr):
    _keep.append(arr)
    return arr.ctypes.data, arr.size


def test_kernel_counts(lib):
    """One alpha-scan launch for BC3 / BC7 files (none for the other formats), one layer-kernel launch per layer."""
    for fmt, scans in ((99, 1), (77, 1), (71, 0), (83, 0), (96, 0)):
        file, d = saved_file(lib, fmt, 33, 17, 4, seed=3)
        before = lib.launch_count()
        info = lib.dds_open(file.ctypes.data, file.size)
        assert lib.launch_count() - before == scans, fmt
        lib.dds_open_layout(info, B.OPEN_MIPS)
        before = lib.launch_count()
        out = np.empty((info.height, info.width, info.planes), np.float32 if info.depth == 32 else np.uint8)
        for c in range(info.calls):
            lib.dds_read_layer_raw(file.ctypes.data, file.size, info, c, out.ctypes.data)
        assert lib.launch_count() - before == info.calls
