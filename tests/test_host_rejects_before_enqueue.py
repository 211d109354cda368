"""Every entry point checks its arguments before it enqueues anything: a rejected call reports the error, launches no kernel
and leaves its output untouched, and the next valid call on the same thread gives the bytes of a fresh encode."""
import ctypes
import importlib

import numpy as np
import pytest

import itw_testlib as T

B = T.binding
sharding = importlib.import_module("intel-texture-works-plugin_b200.sharding")
pytestmark = pytest.mark.gpu


def _pinned(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).reshape(-1).copy()).pin_memory()


def _out(nbytes, device="cpu"):
    import torch
    t = torch.empty(nbytes, dtype=torch.uint8, device=device)
    return t.pin_memory() if device == "cpu" else t


def _sp(settings):
    return ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None


def _bad_bc7(lib):
    s = lib.profile("slow")
    s.fastSkipTreshold_mode1 = 65
    return s


def _rejected_then_valid(lib, run, bad, good, match, out):
    """run(arg) writes `out` and raises RuntimeError on a failure.  run(good) before and after the rejected run(bad) give the
    same bytes; run(bad) fails with `match`, launches nothing and leaves `out` as it was."""
    import torch
    out.fill_(0xAB)
    run(good)
    torch.cuda.synchronize()
    want = out.cpu().clone()
    out.fill_(0xAB)
    torch.cuda.synchronize()
    launches = lib.launch_count()
    with pytest.raises(RuntimeError, match=match):
        run(bad)
    assert lib.launch_count() == launches
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())
    run(good)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), want)


def _raise_unless(lib, ok):
    if not ok:
        raise RuntimeError(lib.last_error())


def test_encode_pixels_rejects_bad_settings():
    lib = T.product()
    pixels = _pinned(T.synth.random_rgba8(64, 64))
    src = B.PixelSource(pixels.data_ptr(), 64, 64, 4, 8, 0)
    out = _out(16 * 16 * 16)
    _rejected_then_valid(lib, lambda s: lib.encode_pixels_raw("BC7", src, 0, out.data_ptr(), s), _bad_bc7(lib), lib.profile("veryfast"),
                         "fastSkipTreshold", out)


def _dds_texture(lib, desc, tops, settings, out):
    surf = (B.RgbaSurface * len(tops))(*[B.RgbaSurface(t.data_ptr(), w, h, w * 4) for t, w, h in tops])
    got = lib.lib.itw_dds_encode_texture(ctypes.byref(desc), surf, _sp(settings), ctypes.c_void_p(out.data_ptr()), out.numel())
    _raise_unless(lib, got == out.numel())


def test_dds_encode_texture_rejects_bad_settings():
    lib = T.product()
    desc = B.DdsDesc(64, 64, 3, 1, 98, 0)
    tops = [(_pinned(T.synth.random_rgba8(64, 64)), 64, 64)]
    out = _out(lib.lib.itw_dds_file_bytes(ctypes.byref(desc)))
    _rejected_then_valid(lib, lambda s: _dds_texture(lib, desc, tops, s, out), _bad_bc7(lib), lib.profile("veryfast"), "fastSkipTreshold", out)


def test_dds_encode_texture_checks_every_item_first():
    lib = T.product()
    desc = B.DdsDesc(64, 64, 3, 2, 71, 0)
    first = (_pinned(T.synth.random_rgba8(64, 64, seed=1)), 64, 64)
    good = [first, (_pinned(T.synth.random_rgba8(64, 64, seed=2)), 64, 64)]
    bad = [first, (_pinned(T.synth.random_rgba8(32, 64, seed=2)), 64, 32)]
    out = _out(lib.lib.itw_dds_file_bytes(ctypes.byref(desc)))
    _rejected_then_valid(lib, lambda tops: _dds_texture(lib, desc, tops, None, out), bad, good, "must match the description", out)


def test_dds_encode_pixels_rejects_bad_settings():
    lib = T.product()
    desc = B.DdsDesc(64, 64, 3, 1, 98, 0)
    pixels = _pinned(T.synth.random_rgba8(64, 64))
    srcs = (B.PixelSource * 1)(B.PixelSource(pixels.data_ptr(), 64, 64, 4, 8, 0))
    out = _out(lib.lib.itw_dds_file_bytes(ctypes.byref(desc)))
    f = lib.lib.itw_dds_encode_pixels
    f.restype = ctypes.c_size_t
    f.argtypes = [ctypes.POINTER(B.DdsDesc), ctypes.POINTER(B.PixelSource), ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    _rejected_then_valid(lib, lambda s: _raise_unless(lib, f(ctypes.byref(desc), srcs, 0, _sp(s), out.data_ptr(), out.numel()) == out.numel()),
                         _bad_bc7(lib), lib.profile("veryfast"), "fastSkipTreshold", out)


def test_sharded_mip_chain_rejects_bad_settings_before_filtering():
    """Single rank, no communicator: 256 x 256 with 3 band-local levels."""
    lib = T.product()
    band = _pinned(T.synth.random_rgba8(256, 256)).cuda()
    plan = sharding.make_plan(lib, "BC7", 256, 256, 3, 1, 0)
    assert plan.band_levels == 3
    chain = _out(plan.chain_bytes, "cuda")
    _rejected_then_valid(lib, lambda s: sharding.encode_mip_chain_sharded(lib, "BC7", band, 256, 256, 3, s, chain=chain), _bad_bc7(lib),
                         lib.profile("veryfast"), "fastSkipTreshold", chain)


@pytest.mark.parametrize("device", ["cpu", "cuda"])
def test_encode_rejects_bad_settings(device):
    """512 host rows take the banded pipeline; device operands the single launch on the legacy stream."""
    lib = T.product()
    img = _pinned(T.synth.random_rgba8(512, 64))
    src = img if device == "cpu" else img.cuda()
    out = _out(128 * 16 * 16, device)
    _rejected_then_valid(lib, lambda s: lib.encode_raw("BC7", src.data_ptr(), 64, 512, 256, out.data_ptr(), s), _bad_bc7(lib),
                         lib.profile("veryfast"), "fastSkipTreshold", out)


def test_encode_batch_rejects_bad_settings():
    lib = T.product()
    tiles = [_pinned(T.synth.random_rgba8(64, 64, seed=i)) for i in range(2)]
    out = _out(2 * 16 * 16 * 16)
    dsts = [out.data_ptr(), out.data_ptr() + 16 * 16 * 16]
    _rejected_then_valid(lib, lambda s: lib.encode_batch("BC7", [(t.data_ptr(), 64, 64, 256) for t in tiles], dsts, s), _bad_bc7(lib),
                         lib.profile("veryfast"), "fastSkipTreshold", out)


def test_compress_blocks_bc7_rejects_null_settings():
    lib = T.product()
    img = _pinned(T.synth.random_rgba8(64, 64))
    out = _out(16 * 16 * 16)
    surf = B.RgbaSurface(img.data_ptr(), 64, 64, 256)
    f = lib.lib.CompressBlocksBC7
    f.restype = None

    def run(s):
        f(ctypes.byref(surf), ctypes.c_void_p(out.data_ptr()), ctypes.byref(s) if s is not None else None)
        lib.check()
    _rejected_then_valid(lib, run, None, lib.profile("veryfast"), "null settings", out)
