"""itw_decompress and itw_preview_pixels on the GPU against the reference's own DirectX::Decompress (oracle/_ref) and the preview
oracle (tests/preview_lib.py); argument checks before the first enqueue."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import preview_lib as P

B = T.binding
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(P.ref() is None, reason="oracle/_ref/libitw_ref_preview.so unavailable")]


@pytest.fixture(scope="module")
def lib():
    return T.product()


def _streams(src):
    profiles = {"BC7": ("basic", "alpha_basic"), "BC6H": ("bc6h_basic",)}.get(P.NAME[src], (None,))
    yield from P.encoded_streams(src, profiles)
    yield "random", P.random_blocks(src, 64 * 72, seed=src), 256, 288


@pytest.mark.parametrize("pair", sorted(P.PAIRS), ids=lambda p: f"{p[0]}-to-{p[1]}")
def test_decompress_equals_directxtex(lib, pair):
    src, target = pair
    for tag, blocks, w, h in _streams(src):
        got = lib.decompress(src, blocks, w, h, target)
        assert got.tobytes() == P.ref_decompress(src, blocks, w, h, target).tobytes(), f"{pair} {tag}"
    for w, h in ((1, 1), (3, 7), (5, 9), (9, 2), (13, 6), (130, 67)):
        blocks = P.random_blocks(src, P.nblocks(w, h), seed=w * 131 + h)
        got = lib.decompress(src, blocks, w, h, target)
        assert got.tobytes() == P.ref_decompress(src, blocks, w, h, target).tobytes(), f"{pair} {w}x{h}"


@pytest.mark.parametrize("pair", [(71, 29), (78, 28), (83, 28), (96, 2), (99, 29)], ids=lambda p: f"{p[0]}-to-{p[1]}")
def test_decompress_device_operands(lib, pair):
    """Device blocks / device destination (aligned and 4-byte offset rows), and the mixed cases."""
    import torch
    src, target = pair
    w, h = 70, 45
    blocks = P.random_blocks(src, P.nblocks(w, h), seed=5)
    want = P.ref_decompress(src, blocks, w, h, target).view(np.uint8).reshape(h, -1)
    row = w * P.texel(target)
    d_blocks = torch.from_numpy(blocks.copy()).cuda()
    for stride in (row, row + 4, row + 16):
        d_out = torch.full((h * stride,), 0xAB, dtype=torch.uint8, device="cuda")
        lib.decompress_raw(src, d_blocks.data_ptr(), w, h, target, d_out.data_ptr(), stride)
        got = d_out.cpu().numpy().reshape(h, stride)
        assert np.array_equal(got[:, :row], want) and (got[:, row:] == 0xAB).all(), stride
    host = np.zeros((h, row), np.uint8)
    lib.decompress_raw(src, d_blocks.data_ptr(), w, h, target, host.ctypes.data, row)
    assert np.array_equal(host, want)
    d_out = torch.zeros(h * row, dtype=torch.uint8, device="cuda")
    lib.decompress_raw(src, blocks.ctypes.data, w, h, target, d_out.data_ptr(), row)
    assert np.array_equal(d_out.cpu().numpy().reshape(h, row), want)


@pytest.mark.parametrize("fmt", ["BC1", "BC3", "BC5", "BC7"])
def test_decompress_equals_decode_where_they_overlap(lib, fmt):
    """UNORM -> R8G8B8A8_UNORM at multiple-of-4 sizes.  Not BC4: DirectX::Decompress shows it grey, itw_decode red-only."""
    src = B.FORMATS[fmt][0]
    blocks = P.random_blocks(src, 32 * 20, seed=9)
    assert np.array_equal(lib.decompress(src, blocks, 128, 80, 28), lib.decode(fmt, blocks, 128, 80))


@pytest.mark.parametrize("target", [28, 29])
def test_decompress_bc4_grey(lib, target):
    blocks = np.tile(np.array([200, 200, 0, 0, 0, 0, 0, 0], np.uint8), 6)          # constant red 200, 3 x 2 blocks
    got = lib.decompress(80, blocks, 11, 7, target)
    assert got[..., 0].min() > 0 and (got[..., 1] == got[..., 0]).all() and (got[..., 2] == got[..., 0]).all()
    assert got.tobytes() == P.ref_decompress(80, blocks, 11, 7, target).tobytes()
    red = lib.decode("BC4", blocks[:16], 8, 4)                                     # itw_decode: (r, 0, 0, 255)
    assert (red[..., 1] == 0).all() and (red[..., 2] == 0).all()
    if target == 28:                                                                # 29 stores the sRGB encoding of r
        assert np.array_equal(got[:4, :8, 0], red[..., 0])


CASES = [(71, None), (77, None), (80, None), (83, None), (98, "basic"), (98, "alpha_basic"), (95, "bc6h_basic"), (96, "bc6h_basic"),
         (72, None), (78, None), (99, "basic")]


@pytest.mark.parametrize("fmt,prof", CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("depth", [8, 16, 32])
@pytest.mark.parametrize("planes", [3, 4])
def test_preview_equals_oracle(lib, fmt, prof, depth, planes):
    flags = B.FRONT_HAS_ALPHA if planes == 4 else 0
    doc = P.document(37, 22, planes, depth, seed=depth + fmt)
    want, nbytes = P.oracle_preview(fmt, [doc], flags, prof)
    got, n = lib.preview_pixels(fmt, [doc], flags, lib.profile(prof) if prof else None)
    assert n == nbytes and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("fmt,prof", [(71, None), (83, None), (98, "basic"), (95, "bc6h_basic"), (99, "alpha_basic")], ids=lambda v: str(v))
@pytest.mark.parametrize("flags", [0, B.FRONT_FLIP_X | B.FRONT_FLIP_Y, B.FRONT_NORMALIZE | B.FRONT_FLIP_Y, B.FRONT_HAS_ALPHA])
def test_preview_cube_cross_equals_oracle(lib, fmt, prof, flags):
    faces = [P.document(9, 7, 4, 8 if fmt != 95 else 16, seed=i) for i in range(6)]
    want, nbytes = P.oracle_preview(fmt, faces, flags, prof)
    got, n = lib.preview_pixels(fmt, faces, flags, lib.profile(prof) if prof else None)
    assert got.shape == (21, 36, 4) and n == nbytes and got.tobytes() == want.tobytes()


def test_preview_normal_map_flags_and_gamma(lib):
    doc = P.document(30, 19, 3, 32, seed=3)
    for flags in (B.FRONT_FLIP_X, B.FRONT_NORMALIZE, B.FRONT_GAMMA | B.FRONT_FLIP_Y):
        want, _ = P.oracle_preview(71, [doc], flags, None)
        got, _ = lib.preview_pixels(71, [doc], flags)
        assert got.tobytes() == want.tobytes(), flags


def test_preview_device_operands(lib):
    import torch
    doc = P.document(33, 17, 4, 8, seed=2)
    want, _ = P.oracle_preview(98, [doc], B.FRONT_HAS_ALPHA, "basic")
    d_doc = torch.from_numpy(doc.copy()).cuda()
    d_out = torch.zeros(17 * 33 * 4, dtype=torch.uint8, device="cuda")
    src = (B.PixelSource * 1)(B.PixelSource(d_doc.data_ptr(), 33, 17, 4, 8, 0))
    lib.preview_pixels_raw(98, src, 1, B.FRONT_HAS_ALPHA, lib.profile("basic"), d_out.data_ptr(), 33, 17, 33 * 4)
    assert d_out.cpu().numpy().tobytes() == want.tobytes()


def _rejects(lib, call, out):
    before, snapshot = lib.launch_count(), out.copy()
    with pytest.raises(RuntimeError):
        call()
    assert lib.launch_count() == before and np.array_equal(out, snapshot)


def test_rejections_before_enqueue(lib):
    blocks = P.random_blocks(98, 4, seed=1)
    out = np.full((8, 8, 4), 7, np.uint8)
    raw = lambda src, w, h, t, stride=32: lambda: lib.decompress_raw(src, blocks.ctypes.data, w, h, t, out.ctypes.data, stride)
    _rejects(lib, raw(98, 8, 8, 2), out)            # unsupported pair
    _rejects(lib, raw(95, 8, 8, 29), out)
    _rejects(lib, raw(80, 8, 8, 2), out)
    _rejects(lib, raw(97, 8, 8, 28), out)           # typeless source
    _rejects(lib, raw(98, 0, 8, 28), out)           # empty image
    _rejects(lib, raw(98, 8, 8, 28, stride=28), out)
    doc = P.document(8, 8, 4, 8, seed=1)
    faces = [doc] * 5 + [P.document(8, 4, 4, 8, seed=1)]
    keep = [np.ascontiguousarray(a) for a in faces]
    srcs = (B.PixelSource * 6)(*[B.PixelSource(a.ctypes.data, a.shape[1], a.shape[0], 4, 8, 0) for a in keep])
    prev = lambda fmt, n, w, h, stride: lambda: lib.preview_pixels_raw(fmt, srcs, n, 0, None, out.ctypes.data, w, h, stride)
    _rejects(lib, prev(71, 6, 32, 24, 128), out)    # faces of unequal size
    _rejects(lib, prev(71, 2, 8, 8, 32), out)       # count neither 1 nor 6
    _rejects(lib, prev(71, 1, 8, 4, 32), out)       # display of the wrong size
    _rejects(lib, prev(71, 1, 8, 8, 16), out)       # display rows too short for the texels
    _rejects(lib, prev(97, 1, 8, 8, 32), out)       # unsupported format
    _rejects(lib, prev(98, 1, 8, 8, 32), out)       # BC7 without settings
