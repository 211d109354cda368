"""The "none" save (include/itw_bcn.h section 12, itw_dds_none_layout / itw_dds_save_none) on the CPU: the layout of every option
class, every refusal before any CUDA call (nothing launched, the file untouched, the call named in the error text), the shared
header routine against the reference's _EncodeDDSHeader, the store's per-texel routine under emulation, and the oracle of
tests/none_lib.py against the merged uncompressed pane.  tests/test_dds_none_gpu.py holds the library to the oracle on the GPU."""
import ctypes
import itertools
import os

import numpy as np
import pytest

import itw_testlib as T
import none_lib as N

B = T.binding
O = B.NoneOptions
D2, CR, LY = B.PANE_2D, B.PANE_CUBE_CROSS, B.PANE_CUBE_LAYERS
ALPHA = B.FRONT_HAS_ALPHA


def want_layout(o, dw, dh):
    """(desc fields, level-0 width, height) of a "none" save, from the plug-in's rules."""
    if o.texture == D2:
        return (dw, dh, N.full_levels(dw, dh) if o.mip_maps else 1, 1, 28, 0), dw, dh
    fw, fh = (dw, dh) if o.texture == LY else ((dw // 3, dh // 4) if dw < dh else (dw // 4, dh // 3))
    L = o.mip_level
    if L >= 0:
        return (N.lvl(fw, L), N.lvl(fh, L), 1, 6, 28, 1), fw, fh
    return (fw, fh, N.full_levels(fw, fh) if o.mip_maps else 1, 6, 28, 1), fw, fh


LAYOUTS = ([(O(D2, m, -1), w, h) for m in (0, 1) for w, h in ((1, 1), (3, 5), (37, 19), (257, 129), (1024, 512), (4096, 4096), (1, 300))]
           + [(O(CR, m, -1), w, h) for m in (0, 1) for w, h in ((4, 3), (3, 4), (64, 48), (48, 64), (150, 100), (1026, 771))]
           + [(O(LY, m, -1), w, h) for m in (0, 1) for w, h in ((1, 1), (37, 19), (2048, 2048))]
           + [(O(t, m, L), w, h) for t, w, h in ((CR, 64, 48), (CR, 60, 80), (LY, 37, 19)) for m in (0, 1)
              for L in range(N.full_levels(*want_layout(O(t, 0, -1), w, h)[1:]))])


@pytest.mark.parametrize("o,w,h", LAYOUTS)
def test_layout(o, w, h):
    p = T.product()
    n, d, fw, fh = p.none_layout(o, w, h)
    fields, ww, wh = want_layout(o, w, h)
    assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == fields
    assert (fw, fh) == (ww, wh)
    assert n == N.file_bytes(d)
    assert p.last_error() == ""


def test_layout_refusals_name_the_call():
    p = T.product()
    for o, w, h in ((None, 4, 4), (O(3, 0, -1), 4, 4), (O(D2, 2, -1), 4, 4), (O(D2, 0, 0), 4, 4), (O(D2, 0, -1), 0, 4),
                    (O(D2, 0, -1), 4, 65533), (O(CR, 0, -1), 3, 3), (O(CR, 0, 3), 16, 12), (O(LY, 0, -2), 4, 4), (O(LY, 5, -1), 4, 4)):
        n, _, _, _ = p.none_layout(o, w, h)
        assert n == 0 and p.last_error().startswith("itw_dds_none_layout:"), (o and (o.texture, o.mip_maps, o.mip_level), w, h)


def test_format_28_stays_unknown_elsewhere():
    p = T.product()
    d = B.DdsDesc(16, 16, 1, 1, 28, 0)
    assert p.lib.itw_dds_header_bytes(ctypes.byref(d)) == 0
    assert p.lib.itw_dds_file_bytes(ctypes.byref(d)) == 0
    assert p.lib.itw_bytes_per_block(28) == 0


def refusal_cases():
    """(description, options, document, layers, layer_count, flags, file, capacity, expected text)."""
    keep = []
    doc = np.full((12, 16, 4), 0xAB, np.uint8)
    keep.append(doc)
    big = np.full(1 << 16, 0xAB, np.uint8)                # larger than any file below
    keep.append(big)

    def src(**kw):
        s = B.PixelSource(doc.ctypes.data, 16, 12, 4, 8, 0)
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    def layer(n=1, bad=None, **kw):
        arr = (B.LayerSource * max(n, 1))()
        plane = np.zeros((12, 16), np.uint8)
        keep.append(plane)
        for i in range(n):
            arr[i].channel_count = 1
            arr[i].channels[0] = plane.ctypes.data
            if i == bad:
                for k, v in kw.items():
                    if k == "null":
                        arr[i].channels[v] = None
                    else:
                        setattr(arr[i], k, v)
        return arr

    def faces(bad=None, **kw):
        arr = layer(6, bad, **kw)
        arr[5].channels[0] = None                          # a face without a layer of that name
        return arr

    F, cap = big.ctypes.data, big.size
    n2d = N.file_bytes(B.DdsDesc(16, 12, 1, 1, 28, 0))
    ncube = N.file_bytes(B.DdsDesc(4, 4, 3, 6, 28, 1))
    cases = [
        ("null options", None, src(), None, 0, 0, F, cap, "null options"),
        ("null document", O(D2, 0, -1), None, None, 0, 0, F, cap, "null document"),
        ("null cross document", O(CR, 0, -1), None, None, 0, 0, F, cap, "null document"),
        ("texture 3", O(3, 0, -1), src(), None, 0, 0, F, cap, "texture"),
        ("texture -1", O(-1, 0, -1), src(), None, 0, 0, F, cap, "texture"),
        ("mip_maps 2", O(D2, 2, -1), src(), None, 0, 0, F, cap, "mip_maps"),
        ("cross mip_maps -1", O(CR, -1, -1), src(), None, 0, 0, F, cap, "mip_maps"),
        ("level on 2-D", O(D2, 1, 0), src(), None, 0, 0, F, cap, "mip_level"),
        ("level -2 on 2-D", O(D2, 0, -2), src(), None, 0, 0, F, cap, "mip_level"),
        ("level -2 on a cross", O(CR, 0, -2), src(), None, 0, 0, F, cap, "mip_level"),
        ("level past the chain", O(CR, 0, 3), src(), None, 0, 0, F, cap, "mip_level"),       # 4 x 4 faces: levels 0..2
        ("level past the chain of layers", O(LY, 0, 5), src(), faces(), 6, 0, F, cap, "mip_level"),
        ("flip on a cross", O(CR, 1, -1), src(), None, 0, B.FRONT_FLIP_X, F, cap, "flags"),
        ("normalise on layers", O(LY, 0, -1), src(), faces(), 6, B.FRONT_NORMALIZE, F, cap, "flags"),
        ("unknown flag", O(D2, 0, -1), src(), None, 0, 32, F, cap, "flag"),
        ("high flag", O(D2, 0, -1), src(), None, 0, 1 << 31, F, cap, "flag"),
        ("layer_count -1", O(D2, 1, -1), src(), layer(), -1, 0, F, cap, "layer"),
        ("null layer list", O(D2, 1, -1), src(), None, 2, 0, F, cap, "layer"),
        ("layer 0 channel_count 0", O(D2, 1, -1), src(), layer(1, 0, channel_count=0), 1, 0, F, cap, "channel_count"),
        ("layer 1 channel_count 4", O(D2, 1, -1), src(), layer(2, 1, channel_count=4), 2, 0, F, cap, "channel_count"),
        ("layer 0 null channel", O(D2, 1, -1), src(), layer(1, 0, channel_count=2, null=1), 1, 0, F, cap, "null channel"),
        ("layer 0 short rows", O(D2, 1, -1), src(), layer(1, 0, row_bytes=15), 1, 0, F, cap, "row_bytes"),
        ("layers of depth 24", O(D2, 1, -1), src(depth=24), layer(), 1, 0, F, cap, "depth"),
        ("cube layers: layer_count 5", O(LY, 0, -1), src(), faces(), 5, 0, F, cap, "layer_count"),
        ("null face list", O(LY, 0, -1), src(), None, 6, 0, F, cap, "face"),
        ("face channel_count 4", O(LY, 0, -1), src(), faces(2, channel_count=4), 6, 0, F, cap, "channel_count"),
        ("face short rows", O(LY, 0, -1), src(), faces(0, row_bytes=8), 6, 0, F, cap, "row_bytes"),
        ("faces of depth 24", O(LY, 0, -1), src(depth=24), faces(), 6, 0, F, cap, "depth"),
        ("depth 24", O(D2, 0, -1), src(depth=24), None, 0, 0, F, cap, "depth"),
        ("planes 0", O(D2, 0, -1), src(planes=0), None, 0, 0, F, cap, "planes"),
        ("planes 5", O(D2, 0, -1), src(planes=5), None, 0, 0, F, cap, "planes"),
        ("width 0", O(D2, 0, -1), src(width=0), None, 0, 0, F, cap, "width"),
        ("height -1", O(D2, 0, -1), src(height=-1), None, 0, 0, F, cap, "height"),
        ("height 65533", O(D2, 0, -1), src(height=65533), None, 0, 0, F, cap, "65532"),
        ("null data", O(D2, 0, -1), src(data=None), None, 0, 0, F, cap, "null pixel source"),
        ("cross of null data", O(CR, 1, -1), src(data=None), None, 0, 0, F, cap, "null pixel source"),
        ("alpha without a fourth plane", O(D2, 0, -1), src(planes=3, row_bytes=48), None, 0, ALPHA, F, cap, "alpha"),
        ("short row_bytes", O(D2, 0, -1), src(row_bytes=63), None, 0, 0, F, cap, "row_bytes"),
        ("cross smaller than a texel per face", O(CR, 0, -1), src(width=3, height=3), None, 0, 0, F, cap, "smaller than one texel"),
        ("null file", O(D2, 0, -1), src(), None, 0, 0, 0, cap, "file"),
        ("capacity one short", O(D2, 0, -1), src(), None, 0, 0, F, n2d - 1, "capacity"),
        ("cube null file", O(CR, 1, -1), src(), None, 0, 0, 0, cap, "file"),
        ("cube capacity one short", O(CR, 1, -1), src(), None, 0, 0, F, ncube - 1, "capacity"),
    ]
    return cases, keep


def test_refusals_before_any_cuda_call():
    p = T.product()
    cases, keep = refusal_cases()
    for name, o, doc, layers, count, flags, file_ptr, capacity, text in cases:
        before = p.launch_count()
        n = p.dds_save_none_raw(o, doc, layers, count, flags, file_ptr, capacity)
        err = p.last_error()
        assert n == 0, name
        assert err.startswith("itw_dds_save_none: "), (name, err)
        assert text in err, (name, err)
        assert p.launch_count() == before, name
    assert (keep[1] == 0xAB).all()                        # the file of every case is untouched


# ---- the header: one routine for the block-compressed files and the "none" files ----
@pytest.fixture(scope="module")
def ref():
    if not N.available():
        pytest.skip("reference cuts not built (no reference tree and no prebuilt oracle/_ref)")


def test_shared_header_routine_keeps_the_block_compressed_headers(ref):
    """itw_dds_write_header (now the shared routine with the table's facts) equals _EncodeDDSHeader for every format and shape class,
    and the recipe that knows R8G8B8A8_UNORM gives the block-compressed headers of the original recipe."""
    import cube_lib as C
    p = T.product()
    for fmt, (w, h, levels, items, cube) in itertools.product((71, 72, 77, 78, 80, 83, 95, 96, 98, 99),
                                                            ((1, 1, 1, 1, 0), (37, 19, 6, 1, 0), (64, 64, 7, 1, 0), (16, 16, 5, 6, 1),
                                                             (8, 4, 1, 3, 0), (5, 5, 3, 12, 1))):
        d = B.DdsDesc(w, h, levels, items, fmt, cube)
        got = np.zeros(256, np.uint8)
        n = p.lib.itw_dds_write_header(ctypes.byref(d), got.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), 256)
        want = C.dds_header(d)
        assert n == want.size and np.array_equal(got[:n], want), (fmt, w, h, levels, items, cube)
        assert np.array_equal(N.dds_header(d), want), (fmt, w, h, levels, items, cube)


@pytest.mark.parametrize("w,h,levels,items,cube", [(16, 16, 1, 1, 0), (16, 16, 5, 1, 0), (37, 19, 1, 1, 0), (37, 19, 6, 1, 0),
                                                   (1, 1, 1, 1, 0), (8, 8, 1, 6, 1), (8, 8, 4, 6, 1), (3, 2, 1, 6, 1)])
def test_rgba8_header_of_the_cut(ref, w, h, levels, items, cube):
    """What the library's "none" files carry (checked byte for byte on the GPU): the legacy header of the cut, with the pitch 4 * w."""
    hd = N.dds_header(B.DdsDesc(w, h, levels, items, 28, cube))
    words = hd.view(np.uint32)
    assert hd.size == 128
    assert words[5] == 4 * w                              # dwPitchOrLinearSize
    assert words[2] & 0x8 and not words[2] & 0x80000      # DDS_HEADER_FLAGS_PITCH, not LINEARSIZE


# ---- the store's per-texel routine ----
@pytest.fixture(scope="module")
def emu():
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_none_emu.so")
    if not os.path.exists(path):
        T.build_emu().compile_cpu(os.path.join(T.ROOT, "tests", "emu", "none_emu.cpp"), path)
    lib = ctypes.CDLL(path)
    lib.emu_none_texels.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]
    return lib


def test_emulated_store_texel(ref, emu):
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (64, 256, 4), dtype=np.uint8)
    img[0, :128, :3] = 128                                # the zero vector (128, 128, 128)
    img[1, :27, :3] = np.array(list(itertools.product((0, 128, 255), repeat=3)), np.uint8)
    flat = np.ascontiguousarray(img).view(np.uint32)
    for normalize in (0, 1):
        out = np.zeros_like(flat)
        emu.emu_none_texels(flat.ctypes.data, flat.size, normalize, out.ctypes.data)
        want = N.normalize(img) if normalize else img
        assert np.array_equal(out.view(np.uint8).reshape(img.shape), want), normalize


# ---- the oracle against merged code ----
@pytest.mark.parametrize("depth,planes", [(8, 3), (16, 4), (32, 4)])
def test_oracle_level0_is_the_uncompressed_pane(ref, depth, planes):
    import preview_uncompressed_lib as U
    doc = U.document(37, 19, planes, depth, seed=depth)
    for flags in (0, ALPHA if planes == 4 else 0, B.FRONT_FLIP_X | B.FRONT_FLIP_Y):
        desc, levels = N.oracle_2d(doc, [], flags, 1)
        pane, _ = U.oracle_pane(28, D2, -1, doc, None, flags)
        assert np.array_equal(levels[0], pane), flags
        assert desc.mip_levels == 6 and len(levels) == 6


def test_oracle_file_size_is_the_layout(ref):
    import preview_uncompressed_lib as U
    p = T.product()
    doc = U.document(48, 36, 4, 8, seed=1)
    for o in (O(D2, 0, -1), O(D2, 1, -1), O(CR, 1, -1), O(CR, 0, 2), O(LY, 1, -1)):
        layers = U.cube_layers(48, 36, 8, seed=2) if o.texture == LY else None
        blob = N.oracle_save(o, doc, layers, ALPHA)
        assert blob.size == p.none_layout(o, 48, 36)[0], (o.texture, o.mip_maps, o.mip_level)
