"""The "none" save (itw_dds_save_none, include/itw_bcn.h section 12) on the GPU: whole files byte for byte against the oracle of
tests/none_lib.py (the plug-in's DoWriteDDS for encoding 28 over the reference's own bodies), agreement with the merged uncompressed
pane, device-resident operands, a file above 256 MiB, and refusals that launch nothing."""
import ctypes
import itertools

import numpy as np
import pytest

import itw_testlib as T
import none_lib as N
import preview_uncompressed_lib as U

B = T.binding
O = B.NoneOptions
D2, CR, LY = B.PANE_2D, B.PANE_CUBE_CROSS, B.PANE_CUBE_LAYERS
ALPHA, GAMMA, NORMALIZE = B.FRONT_HAS_ALPHA, B.FRONT_GAMMA, B.FRONT_NORMALIZE
FX, FY = B.FRONT_FLIP_X, B.FRONT_FLIP_Y

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    if not N.available():
        pytest.skip("reference cuts not built (no reference tree and no prebuilt oracle/_ref)")


def check(o, doc, layers=None, flags=0):
    p = T.product()
    got = p.dds_save_none(o, doc, layers, flags)
    want = N.oracle_save(o, doc, layers, flags)
    assert got.size == want.size
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got != want)
        raise AssertionError(f"{bad.size} bytes differ, first at {bad[0]} (header 128)")
    return got


SIZES = ((1, 1), (3, 5), (37, 19), (257, 129), (1024, 512))


@pytest.mark.parametrize("depth,planes,flags", [(d, p, f) for d, p in itertools.product((8, 16, 32), (3, 4))
                                                for f in (0, ALPHA, GAMMA, ALPHA | GAMMA) if p == 4 or not f & ALPHA])
def test_2d_matches_oracle(ref, depth, planes, flags):
    for (w, h), mips in itertools.product(SIZES, (0, 1)):
        doc = U.document(w, h, planes, depth, seed=w * 7 + h + depth + planes + flags)
        check(O(D2, mips, -1), doc, None, flags)


@pytest.mark.parametrize("flags", [FX, FY, FX | FY, NORMALIZE, FX | NORMALIZE, FX | FY | NORMALIZE | ALPHA, GAMMA | FY | NORMALIZE])
def test_normal_map_matches_oracle(ref, flags):
    for (w, h), depth, mips in itertools.product(((1, 1), (37, 19), (64, 64), (257, 129)), (8, 32), (0, 1)):
        doc = U.document(w, h, 4, depth, seed=w + depth + flags)
        check(O(D2, mips, -1), doc, None, flags)


@pytest.mark.parametrize("depth,channels,alpha,flags", [(d, c, a, f) for d in (8, 16, 32) for c in (1, 2, 3) for a in (False, True)
                                                        for f in (ALPHA, 0) if not (a and not f)] + [(8, 3, True, ALPHA | FX | NORMALIZE),
                                                                                                    (32, 2, True, ALPHA | GAMMA | FY)])
def test_mips_from_layers_match_oracle(ref, depth, channels, alpha, flags):
    for (w, h), count in (((64, 32), 1), ((64, 32), 3), ((37, 19), 6), ((37, 19), 9), ((16, 16), 5)):
        doc = U.document(w, h, 4, depth, seed=w + count + depth)
        layers = [U.layer(w, h, depth, channels, alpha, seed=100 + i + depth) for i in range(count)]
        check(O(D2, 1, -1), doc, layers, flags)
    doc = U.document(37, 19, 4, depth, seed=3)                 # without mip maps only layer 0 is read
    check(O(D2, 0, -1), doc, [U.layer(37, 19, depth, channels, alpha, seed=9)] * 2, flags)


@pytest.mark.parametrize("texture,w,h", [(CR, 64, 48), (CR, 48, 64), (CR, 150, 100), (CR, 40, 53), (LY, 37, 19), (LY, 32, 32)])
def test_cube_matches_oracle(ref, texture, w, h):
    fw, fh = (w, h) if texture == LY else ((w // 3, h // 4) if w < h else (w // 4, h // 3))
    for depth, flags in ((8, 0), (16, ALPHA), (32, ALPHA | GAMMA)):
        doc = U.document(w, h, 4, depth, seed=w + depth)
        layers = U.cube_layers(w, h, depth, seed=depth, missing=(1, 4)) if texture == LY else None
        for mips in (0, 1):
            check(O(texture, mips, -1), doc, layers, flags)
        for L in range(N.full_levels(fw, fh)):
            check(O(texture, L % 2, L), doc, layers, flags)


def test_level0_is_the_uncompressed_pane():
    p = T.product()
    for depth, (w, h), flags in itertools.product((8, 16, 32), ((37, 19), (64, 32)), (0, ALPHA, FX | FY)):
        doc = U.document(w, h, 4, depth, seed=depth + w)
        blob = p.dds_save_none(O(D2, 1, -1), doc, None, flags)
        pane, size = p.preview_uncompressed(B.PaneOptions(28, B.PANE_2D, -1), doc, None, flags)
        assert np.array_equal(blob[128:128 + w * h * 4].reshape(h, w, 4), pane), (depth, flags)
        assert size == w * h * 4


def test_cube_level_faces_are_the_pane_cells():
    p = T.product()
    for texture, (w, h) in ((CR, (64, 48)), (LY, (24, 20))):
        doc = U.document(w, h, 4, 8, seed=w)
        layers = U.cube_layers(w, h, 8, seed=4, missing=(2,)) if texture == LY else None
        fw, fh = (w, h) if texture == LY else (w // 4, h // 3)
        for L in range(N.full_levels(fw, fh)):
            blob = p.dds_save_none(O(texture, 0, L), doc, layers, ALPHA)
            pane, _ = p.preview_uncompressed(B.PaneOptions(28, texture, L), doc, layers, ALPHA)
            wl, hl = N.lvl(fw, L), N.lvl(fh, L)
            faces = blob[128:].reshape(6, hl, wl, 4)
            for f, (cx, cy) in enumerate(((2, 1), (0, 1), (1, 0), (1, 2), (1, 1), (3, 1))):
                assert np.array_equal(faces[f], pane[cy * hl:(cy + 1) * hl, cx * wl:(cx + 1) * wl]), (texture, L, f)


def _device_call(o, doc, layers, count, flags):
    """itw_dds_save_none with the document, the layer planes and the file in device memory."""
    import torch
    p = T.product()
    keep = []

    def dev(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        keep.append(t)
        return t.data_ptr()
    src = B.PixelSource(dev(doc), doc.shape[1], doc.shape[0], doc.shape[2], doc.itemsize * 8, 0)
    arr = None
    if layers is not None:
        arr = (B.LayerSource * max(count, 1))()
        for i, entry in enumerate(layers):
            if entry is None:
                continue
            channels, alpha = entry
            arr[i].channel_count = len(channels)
            for c, pl in enumerate(channels):
                arr[i].channels[c] = dev(pl)
            arr[i].alpha = dev(alpha) if alpha is not None else None
    n = p.none_layout(o, doc.shape[1], doc.shape[0])[0]
    file = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    got = p.dds_save_none_raw(o, src, arr, count, flags, file.data_ptr(), n)
    assert got == n, p.last_error()
    return file.cpu().numpy()


def test_device_operands_give_the_host_bytes(ref):
    p = T.product()
    doc = U.document(37, 19, 4, 16, seed=8)
    layers = [U.layer(37, 19, 16, 2, True, seed=20 + i) for i in range(3)]
    for o, ls, count, flags in ((O(D2, 1, -1), None, 0, ALPHA | FX | NORMALIZE), (O(D2, 1, -1), layers, 3, ALPHA | FY)):
        assert np.array_equal(_device_call(o, doc, ls, count, flags), p.dds_save_none(o, doc, ls, flags))
    cross = U.document(64, 48, 4, 32, seed=9)
    assert np.array_equal(_device_call(O(CR, 1, -1), cross, None, 0, ALPHA | GAMMA), N.oracle_save(O(CR, 1, -1), cross, None, ALPHA | GAMMA))
    faces = U.cube_layers(24, 20, 8, seed=5, missing=(0,))
    assert np.array_equal(_device_call(O(LY, 0, 2), U.document(24, 20, 4, 8, seed=1), faces, 6, ALPHA),
                          N.oracle_save(O(LY, 0, 2), U.document(24, 20, 4, 8, seed=1), faces, ALPHA))


def test_file_above_256_mib(ref):
    """8192 x 8192 with its full chain: 358 MB, payload offsets beyond 32 bits of texels * 4 within one launch."""
    doc = U.document(8192, 8192, 4, 8, seed=12)
    got = check(O(D2, 1, -1), doc, None, ALPHA)
    assert got.size > 256 << 20


def test_refusals_launch_nothing_and_the_kernel_time():
    import test_dds_none as C
    p = T.product()
    cases, keep = C.refusal_cases()
    for name, o, doc, layers, count, flags, file_ptr, capacity, text in cases:
        before = p.launch_count()
        assert p.dds_save_none_raw(o, doc, layers, count, flags, file_ptr, capacity) == 0, name
        assert p.launch_count() == before, name
    assert (keep[1] == 0xAB).all()
    before = p.launch_count()
    p.dds_save_none(O(D2, 1, -1), U.document(256, 256, 4, 8, seed=1), None, NORMALIZE)
    assert p.last_kernel_ms() > 0
    assert p.launch_count() - before >= 2                 # the front end, the chain and ONE store launch
    p.dds_save_none(O(CR, 1, -1), U.document(64, 48, 4, 8, seed=1))
    assert p.last_kernel_ms() > 0
