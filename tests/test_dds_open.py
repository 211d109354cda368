"""The open path without a GPU: itw_dds_open_layout against the plug-in's DoReadStart decisions (restated in tests/open_lib.py), the
alpha scan's per-block predicate (csrc/open.cuh, run on the CPU) against the reference's own _IsAlphaAllOpaqueBC for every BC3 alpha
block shape and every BC7 alpha byte, and the argument checks that run before any CUDA call."""
import ctypes
import itertools

import numpy as np
import pytest

import itw_testlib as T
import open_lib as O

B = T.binding
needs_ref = pytest.mark.skipif(O.ref() is None, reason="oracle/_ref/libitw_ref_open.so unavailable")


@pytest.fixture(scope="module")
def lib():
    return T.product()


def _layout(lib, d, has_alpha, options):
    info = B.DdsOpenInfo()
    info.desc = d
    info.has_alpha = has_alpha
    info.has_mips = d.mip_levels > 1
    return lib.dds_open_layout(info, options)


@pytest.mark.parametrize("fmt", O.FORMATS)
def test_layout_equals_plugin_decisions(lib, fmt):
    for opaque, mips, cube, options in itertools.product((True, False), (1, 7), (False, True), O.OPTIONS):
        d = O.desc(70, 70, fmt, mips, cube)
        want = O.read_start(d, opaque, options)
        info = _layout(lib, d, want["has_alpha"], options)
        got = O.info_fields(info)
        for k in ("layers", "calls", "planes", "depth", "width", "height", "target_dxgi"):
            assert got[k] == want[k], (fmt, opaque, mips, cube, options, k, got[k], want[k])


def test_layout_cases_by_hand(lib):
    """A few rows of the table read straight off IntelPlugin.cpp:2507-2602."""
    bc7 = O.desc(64, 32, 98, 7)
    assert O.info_fields(_layout(lib, bc7, 1, 0))["layers"] == 1                       # alpha -> one transparent layer, 4 planes
    assert O.info_fields(_layout(lib, bc7, 1, B.OPEN_SEPARATE_ALPHA))["layers"] == 0   # background + alpha channel
    assert O.info_fields(_layout(lib, bc7, 1, B.OPEN_SEPARATE_ALPHA))["planes"] == 4
    assert O.info_fields(_layout(lib, bc7, 0, B.OPEN_MIPS))["layers"] == 7             # mips as layers
    assert O.info_fields(_layout(lib, bc7, 0, 0))["planes"] == 3                        # opaque background
    cube = _layout(lib, O.desc(16, 16, 99, 5, True), 1, B.OPEN_SEPARATE_ALPHA | B.OPEN_MIPS)
    assert (cube.layers, cube.calls, cube.planes, cube.depth, cube.target_dxgi) == (6, 6, 4, 8, 29)
    hdr = _layout(lib, O.desc(5, 3, 96), 0, 0)
    assert (hdr.layers, hdr.calls, hdr.planes, hdr.depth, hdr.target_dxgi) == (0, 1, 3, 32, 2)


def _bc3_all_palette_entries():
    """Every (a0, a1, index): sixteen texels of the same index."""
    a0, a1, q = [a.ravel() for a in np.meshgrid(np.arange(256), np.arange(256), np.arange(8), indexing="ij")]
    idx = np.zeros(len(q), np.uint64)
    for k in range(16):
        idx |= q.astype(np.uint64) << np.uint64(3 * k)
    b = np.zeros((len(q), 16), np.uint8)
    b[:, 0], b[:, 1] = a0, a1
    for k in range(6):
        b[:, 2 + k] = ((idx >> np.uint64(8 * k)) & np.uint64(255)).astype(np.uint8)
    b[:, 8:10] = (0x00, 0xF8)
    return b


@needs_ref
def test_bc3_alpha_predicate_exhaustive():
    """All 524 288 (a0, a1, index) triples: the integer palette byte test equals the float < 0.99 test of _IsAlphaAllOpaqueBC."""
    blocks = _bc3_all_palette_entries()
    want = O.blocks_opaque(O.ref(), 77, blocks)
    assert np.array_equal(O.blocks_opaque(O.emu(), 77, blocks), want)
    assert np.array_equal(O.blocks_opaque(O.emu(), 78, blocks), O.blocks_opaque(O.ref(), 78, blocks))
    assert 0 < want.sum() < len(want)
    # the boundary the predicate rests on: endpoint 253 reads opaque, 252 does not
    pick = lambda a0, a1, q: want[(a0 * 256 + a1) * 8 + q]
    assert pick(253, 253, 0) == 1 and pick(252, 252, 0) == 0 and pick(0, 0, 7) == 1 and pick(255, 255, 6) == 0


def _bc7_alpha_blocks(seed):
    rng = np.random.default_rng(seed)
    out = []
    for a0 in range(256):                                          # mode 6: every 8-bit endpoint pair, random 4-bit indices
        for a1 in range(256):
            out.append(O.bc7_mode6(a0, a1, rng.integers(0, 16, 16)))
    for a0 in range(256):                                          # mode 5: every 8-bit alpha endpoint pair, every rotation
        for a1 in range(0, 256, 3):
            out.append(O.bc7_mode5(a0, a1, rng.integers(0, 4, 16), rot=int(rng.integers(0, 4)),
                                   rgb=tuple(int(v) for v in rng.integers(0, 256, 3))))
    for a in range(32):                                            # mode 7: every 5-bit alpha endpoint of subset 0 with both p-bits
        for b in range(32):
            for p in range(4):
                ep = [a, b, int(rng.integers(28, 32)), int(rng.integers(28, 32))]
                out.append(O.bc7_mode7(ep, [p & 1, p >> 1, 1, 1], rng.integers(0, 4, 16)))
    out.append(np.zeros(16, np.uint8))                             # the reserved mode: transparent black
    return np.stack(out)


@needs_ref
def test_bc7_alpha_predicate_every_alpha_byte():
    blocks = _bc7_alpha_blocks(seed=3)
    for fmt in (98, 99):
        want = O.blocks_opaque(O.ref(), fmt, blocks)
        assert np.array_equal(O.blocks_opaque(O.emu(), fmt, blocks), want), fmt
    # constant-alpha mode 6 blocks cross over exactly between 252 and 253
    const = np.stack([O.bc7_mode6(a, a, np.zeros(16, int)) for a in range(256)])
    assert O.blocks_opaque(O.ref(), 98, const).tolist() == [0] * 253 + [1] * 3
    assert O.blocks_opaque(O.emu(), 98, const).tolist() == [0] * 253 + [1] * 3
    rnd = np.random.default_rng(5).integers(0, 256, (20000, 16), dtype=np.uint8)
    assert np.array_equal(O.blocks_opaque(O.emu(), 98, rnd), O.blocks_opaque(O.ref(), 98, rnd))


@needs_ref
@pytest.mark.parametrize("fmt", [77, 98])
def test_ragged_blocks_ignore_padding(fmt):
    for cols in range(1, 5):
        for rows in range(1, 5):
            for bad in (False, True):
                blk = O.padding_only_block(fmt, cols, rows, bad)
                want = O.blocks_opaque(O.ref(), fmt, blk, cols, rows)
                assert want[0] == (0 if bad else 1), (cols, rows, bad)
                assert np.array_equal(O.blocks_opaque(O.emu(), fmt, blk, cols, rows), want), (cols, rows, bad)


@needs_ref
@pytest.mark.parametrize("fmt", [78, 99])
def test_whole_file_check_equals_blocks(fmt):
    """ScratchImage::IsAlphaAllOpaque over every image of a ragged 2-D chain and a cube map with mips, against the per-block predicate
    applied image by image: non-opaque texels in the padding of every image, and one in the deepest mip only."""
    for w, h, mips, cube in ((13, 6, 4, False), (5, 5, 3, True)):
        d = O.desc(w, h, fmt, mips, cube)
        payload = O.padding_only_payload(d)
        assert O.ref_all_opaque(O.make_file(d, payload), d)
        last = len(payload) - 16                                   # the 1x1 level of the last item: its texel 0
        bad = payload.copy()
        bad[last:] = O.padding_only_block(fmt, 1, 1, inside_bad=True)
        assert not O.ref_all_opaque(O.make_file(d, bad), d)
        assert O.blocks_opaque(O.emu(), fmt, bad[last:], 1, 1)[0] == 0


def test_layout_rejects(lib):
    f = lib.lib.itw_dds_open_layout
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
    assert f(None, 0) != 0 and "null" in lib.last_error()
    info = B.DdsOpenInfo()
    info.desc = O.desc(8, 8, 74)                                   # BC2
    assert f(ctypes.addressof(info), 0) != 0 and "desc" in lib.last_error()
    info.desc = O.desc(8, 8, 98)
    assert f(ctypes.addressof(info), 4) != 0 and "option" in lib.last_error()
    assert f(ctypes.addressof(info), 3) == 0 and lib.last_error() == ""


def test_read_layer_rejects_before_any_cuda_call(lib):
    """Checks that need no device: every one fails with its own message and leaves dst untouched."""
    d = O.desc(8, 8, 98)
    file = O.make_file(d, np.zeros(4 * 16, np.uint8))
    info = B.DdsOpenInfo()
    info.desc = d
    dst = np.full(8 * 8 * 4, 0x5A, np.uint8)

    def rejects(what, inf, call=0, row_bytes=0, f=file, size=None):
        with pytest.raises(RuntimeError, match=what):
            lib.dds_read_layer_raw(f.ctypes.data, f.size if size is None else size, inf, call, dst.ctypes.data, row_bytes)
        assert (dst == 0x5A).all()

    rejects("not laid out", info)                                  # itw_dds_open_layout not called
    lib.dds_open_layout(info, 0)
    rejects("call out of range", info, call=1)
    rejects("call out of range", info, call=-1)
    rejects("row_bytes", info, row_bytes=8 * 3 - 1)
    rejects("row_bytes", info, row_bytes=-4)
    rejects("truncated", info, size=file.size - 1)
    other = B.DdsOpenInfo()
    other.desc = O.desc(8, 4, 98)
    lib.dds_open_layout(other, 0)
    rejects("does not match", other)
    forged = B.DdsOpenInfo()
    ctypes.memmove(ctypes.addressof(forged), ctypes.addressof(info), ctypes.sizeof(info))
    forged.layers, forged.calls = 6, 6                             # a 2-D texture without mips has no six layers
    rejects("not laid out", forged, call=5)
    bc2 = file.copy()
    bc2[128 + 0] = 74                                              # DX10 header naming BC2
    rejects("not a DDS file", info, f=bc2)
    lib.dds_open_layout(info, 0)
    assert lib.last_error() == ""


def test_open_rejects_before_any_cuda_call(lib):
    f = lib.lib.itw_dds_open
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    info = B.DdsOpenInfo()
    d = O.desc(8, 8, 77, 4)
    file = O.make_file(d, np.zeros(O.payload_bytes(d), np.uint8))
    assert f(file.ctypes.data, file.size - 1, ctypes.addressof(info)) != 0 and "truncated" in lib.last_error()
    dxt3 = O.legacy_file("DXT3", 8, 8, 1, np.zeros(4 * 16, np.uint8))
    assert f(dxt3.ctypes.data, dxt3.size, ctypes.addressof(info)) != 0 and "not a DDS file" in lib.last_error()
    assert f(None, 0, ctypes.addressof(info)) != 0 and "null" in lib.last_error()
    assert bytes(info) == bytes(B.DdsOpenInfo())                   # info untouched
    info.desc = d
    lib.dds_open_layout(info, 0)                                   # a call that succeeds clears the thread's last error
    assert lib.last_error() == ""


def test_dx10_headers_give_the_payload_offset_of_the_file(lib):
    """A 'DX10' extension header on a format the library writes with a legacy header: the payload starts at 148, not at the 128 the
    library would write, and a file cut short of that payload is rejected before any CUDA call."""
    f = lib.lib.itw_dds_open
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    info = B.DdsOpenInfo()
    for fmt, cube in ((71, False), (77, False), (80, True), (83, False)):
        d = O.desc(8, 8, fmt, 2, cube)
        file = O.dx10_file(d, np.zeros(O.payload_bytes(d), np.uint8))
        got = B.DdsDesc()
        assert lib.lib.itw_dds_read_header(file.ctypes.data, file.size, ctypes.byref(got)) == 148
        assert lib.lib.itw_dds_file_bytes(ctypes.byref(d)) == file.size - 20            # the size the library would write
        for cut in (1, 19, 20):
            assert f(file.ctypes.data, file.size - cut, ctypes.addressof(info)) != 0 and "truncated" in lib.last_error(), (fmt, cut)
            dst = np.full(8 * 8 * 4, 0x5A, np.uint8)
            with pytest.raises(RuntimeError, match="truncated"):
                lib.dds_read_layer_raw(file.ctypes.data, file.size - cut, lib.dds_open_layout(info_for(d), 0), 0, dst.ctypes.data)
            assert (dst == 0x5A).all()
    lib.dds_open_layout(info_for(d), 0)
    assert lib.last_error() == ""


def info_for(d):
    info = B.DdsOpenInfo()
    info.desc = d
    return info
