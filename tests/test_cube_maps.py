"""Cube maps from the document (include/itw_bcn.h section 10): the save dialog's CUBEMAP_CROSSED and CUBEMAP_LAYERS types, with and
without a set mip level, saved (itw_dds_encode_cube) and previewed (itw_preview_cube).

CPU: itw_cube_layout for every option class and every refusal; the cross-to-faces kernel's per-texel routine (cube_texel in
csrc/frontend.cuh, through tests/emu/cube_emu.cpp) against the oracle's front end and sRGB conversion, both cross orientations, ragged
faces, depths 8 / 16 / 32; the linearising byte map for all 256 bytes.
GPU: every byte of the file and of the preview against the oracle pipeline of tests/cube_lib.py; agreement with itw_dds_encode_pixels;
a round trip through the open path; device operands; refusals that leave the output untouched and enqueue nothing."""
import ctypes
import itertools

import numpy as np
import pytest

import cube_lib as C
import itw_testlib as T
import preview_lib as PL

B = T.binding
FORMATS = {71: None, 72: None, 77: None, 78: None, 95: "bc6h_veryfast", 98: "veryfast", 99: "alpha_veryfast"}


def opts(fmt, source=B.CUBE_CROSS, mips=0, level=-1):
    return B.CubeOptions(fmt, source, mips, level)


# ---- layout (no CUDA call) ----
@pytest.mark.parametrize("source,dw,dh,w,h", [(0, 64, 48, 16, 16), (0, 48, 64, 16, 16), (0, 50, 31, 12, 10), (0, 31, 50, 10, 12),
                                              (0, 4, 3, 1, 1), (0, 3, 4, 1, 1), (0, 4096, 3072, 1024, 1024), (1, 13, 7, 13, 7),
                                              (1, 1, 1, 1, 1)])
def test_layout_every_option_class(source, dw, dh, w, h):
    p = T.product()
    full = max(w, h).bit_length()
    for fmt in FORMATS:
        for mips, level in [(0, -1), (1, -1)] + [(m, l) for m in (0, 1) for l in sorted({0, full // 2, full - 1})]:
            n, d, fw, fh = p.cube_layout(opts(fmt, source, mips, level), dw, dh)
            assert (fw, fh) == (w, h) and n, p.last_error()
            want = (C.lvl(w, level), C.lvl(h, level), 1) if level >= 0 else (w, h, full if mips else 1)
            assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == want + (6, fmt, 1)
            assert n == p.lib.itw_dds_file_bytes(ctypes.byref(d))
            assert p.last_error() == ""


def test_layout_refusals():
    p = T.product()
    for o, dw, dh in [(opts(80), 64, 48), (opts(83), 64, 48), (opts(96), 64, 48), (opts(0), 64, 48), (opts(28), 64, 48),
                      (opts(98, source=2), 64, 48), (opts(98, mips=2), 64, 48), (opts(98, level=-2), 64, 48),
                      (opts(98, level=5), 64, 48),                  # 16 x 16 faces: five levels, 0..4
                      (opts(98, B.CUBE_LAYERS, level=4), 13, 7),   # 13 x 7: four levels
                      (opts(98), 3, 3), (opts(98), 3, 2), (opts(98), 2, 3), (opts(98), 0, 48), (opts(98, B.CUBE_LAYERS), 0, 5)]:
        n, _, _, _ = p.cube_layout(o, dw, dh)
        assert n == 0 and p.last_error() != "", (o.dxgi_format, o.source, o.mip_maps, o.mip_level, dw, dh)
    assert p.cube_layout(opts(98), 64, 48)[0] and p.last_error() == ""       # the next call clears the error text


# ---- the kernel's per-texel routine on the CPU ----
@pytest.fixture(scope="module")
def emu_cube():
    import os
    path = os.path.join(T.ROOT, "tests", "emu", "libitw_cube_emu.so")
    src = os.path.join(T.ROOT, "tests", "emu", "cube_emu.cpp")
    deps = [src, os.path.join(T.ROOT, "intel-texture-works-plugin_b200", "csrc", "frontend.cuh")]
    if not os.path.exists(path) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(path):
        T.build_emu().compile_cpu(src, path)              # __graft_entry__.build() made it; rebuilt only when stale
    lib = ctypes.CDLL(path)
    lib.emu_cube_faces.restype = ctypes.c_int
    return lib


def emu_faces(lib, fmt, doc, flags, linear):
    dh, dw = doc.shape[:2]
    w, h = C.face_size(B.CUBE_CROSS, dw, dh)
    hdr = fmt == 95
    out = np.zeros((6, h, w, 4), np.uint16 if hdr else np.uint8)
    doc = np.ascontiguousarray(doc)
    assert lib.emu_cube_faces(2 if hdr else 0, doc.ctypes.data_as(ctypes.c_void_p), dw, dh, doc.shape[2], doc.itemsize * 8, flags, int(linear),
                              out.ctypes.data_as(ctypes.c_void_p)) == 0
    return list(out)


@pytest.mark.parametrize("fmt,depth", list(itertools.product((71, 99, 95), (8, 16, 32))))
def test_emulated_cube_texel_matches_oracle(emu_cube, fmt, depth):
    for (dw, dh), planes, flags in itertools.product(((64, 48), (48, 64), (50, 31), (31, 50), (4, 3), (3, 4)), (3, 4), (0, 1, 2, 3)):
        if (flags & 1) and planes < 4:
            continue
        doc = PL.document(dw, dh, planes, depth, seed=dw * 7 + depth + planes + flags)
        for linear in ((False, True) if fmt != 95 else (False,)):
            want = C.oracle_cross_faces(fmt, doc, flags, linear)
            got = emu_faces(emu_cube, fmt, doc, flags, linear)
            for f in range(6):
                assert np.array_equal(got[f], want[f]), (dw, dh, planes, flags, linear, f)


def test_linearising_copy_of_all_256_bytes(emu_cube):
    """Every byte through the sRGB -> UNORM conversion of CopyRectangle, in r, g and b, alpha untouched."""
    v = np.arange(256, dtype=np.uint8)
    doc = np.zeros((3, 4 * 256, 4), np.uint8)                      # one row of faces, 256 x 1 texels each
    doc[1, :, 0] = np.tile(v, 4)
    doc[1, :, 1] = np.tile(v[::-1], 4)
    doc[1, :, 2] = np.tile(np.roll(v, 77), 4)
    doc[1, :, 3] = np.tile(np.roll(v, 5), 4)
    got = emu_faces(emu_cube, 99, doc, B.FRONT_HAS_ALPHA, True)
    lin = C.srgb_in_bytes()
    assert lin[0] == 0 and lin[255] == 255 and (np.diff(lin.astype(int)) >= 0).all()
    for f in (0, 1, 4, 5):                                        # +X, -X, +Z, -Z lie in the middle row
        px = got[f][0]
        assert np.array_equal(px[:, 0], lin[v]) and np.array_equal(px[:, 1], lin[v[::-1]]) and np.array_equal(px[:, 2], lin[np.roll(v, 77)])
        assert np.array_equal(px[:, 3], np.roll(v, 5))


# ---- GPU ----
def cross_doc(fmt, dw, dh, depth, planes, seed):
    doc = PL.document(dw, dh, planes, depth, seed)
    if fmt == 95 and depth == 32:
        doc = np.clip(doc, 0, 4).astype(np.float32)
    return doc


def face_layers(fmt, w, h, depth, seed, missing=(4,)):
    """Six face layers: one missing, one grey (one channel), two with an alpha plane, the rest RGB."""
    import test_mips_from_layers as ML
    rng = np.random.default_rng(seed)
    out = []
    for i in range(6):
        if i in missing:
            out.append(None)
            continue
        channels = [ML.plane(depth, w, h, rng, specials=(fmt != 95)) for _ in range(1 if i == 2 else 3)]
        alpha = ML.plane(depth, w, h, rng, specials=(fmt != 95)) if i in (0, 3) else None
        if fmt == 95 and depth == 32:
            channels = [np.clip(c, 0, 4) for c in channels]
            alpha = None if alpha is None else np.clip(alpha, 0, 4)
        out.append((channels, alpha))
    return out


def case_levels(w, h):
    full = max(w, h).bit_length()
    return [(0, -1), (1, -1), (1, 0), (0, full // 2), (1, full - 1)]


SAVE_CASES = []
for _fmt in FORMATS:
    for _src in (B.CUBE_CROSS, B.CUBE_LAYERS):
        SAVE_CASES.append((_fmt, _src))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,source", SAVE_CASES)
def test_gpu_save_matches_oracle_pipeline(fmt, source):
    p = T.product()
    prof = FORMATS[fmt]
    s = p.profile(prof) if prof else None
    depth = {71: 8, 72: 16, 77: 32, 78: 8, 95: 32, 98: 16, 99: 8}[fmt]
    for k, (mips, level) in enumerate(case_levels(12, 10) if source == B.CUBE_CROSS else case_levels(13, 7)):
        flags = (B.FRONT_HAS_ALPHA if k % 2 == 0 else 0) | (B.FRONT_GAMMA if depth == 32 else 0)
        if source == B.CUBE_CROSS:
            dw, dh = (48, 30) if k % 2 == 0 else (36, 40)            # horizontal and vertical, 12 x 10 faces
            doc = cross_doc(fmt, dw, dh, depth, 4 if flags & 1 else 3, seed=fmt + k)
            faces = None
        else:
            doc = cross_doc(fmt, 13, 7, depth, 4, seed=fmt + k)
            faces = face_layers(fmt, 13, 7, depth, seed=fmt * 3 + k, missing=(4,) if k % 2 else (1, 5))
        o = opts(fmt, source, mips, level)
        got = p.dds_encode_cube(o, doc, faces, flags, s)
        want = C.oracle_save(o, doc, faces, flags, prof)
        assert got.size == want.size and np.array_equal(got, want), (mips, level, flags, int((got != want).sum()) if got.size == want.size else -1)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,source", SAVE_CASES)
def test_gpu_preview_matches_oracle(fmt, source):
    p = T.product()
    prof = FORMATS[fmt]
    s = p.profile(prof) if prof else None
    depth = {71: 16, 72: 8, 77: 8, 78: 32, 95: 32, 98: 8, 99: 16}[fmt]
    for k, (mips, level) in enumerate(case_levels(12, 10) if source == B.CUBE_CROSS else case_levels(13, 7)):
        flags = B.FRONT_HAS_ALPHA if k % 2 == 0 else 0
        if source == B.CUBE_CROSS:
            dw, dh = (48, 30) if k % 2 == 0 else (36, 40)
            doc = cross_doc(fmt, dw, dh, depth, 4 if flags & 1 else 3, seed=fmt + 5 * k)
            faces = None
        else:
            doc = cross_doc(fmt, 13, 7, depth, 4, seed=fmt + k)
            faces = face_layers(fmt, 13, 7, depth, seed=fmt * 5 + k)
        o = opts(fmt, source, mips, level)
        img, n = p.preview_cube(o, doc, faces, flags, s)
        want, wn = C.oracle_preview(o, doc, faces, flags, prof)
        assert n == wn and img.shape == want.shape, (mips, level)
        assert np.array_equal(img.view(np.uint8), want.view(np.uint8)), (mips, level, flags)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,mips", [(71, 1), (77, 0), (98, 1), (95, 1)])
def test_gpu_cross_equals_encode_pixels_with_six_row_offset_sources(fmt, mips):
    """A cross of a non-sRGB format: the file equals itw_dds_encode_pixels of six sources pointing into the document."""
    p = T.product()
    prof = FORMATS[fmt]
    s = p.profile(prof) if prof else None
    dw, dh, depth = 64, 48, (32 if fmt == 95 else 8)
    doc = np.ascontiguousarray(cross_doc(fmt, dw, dh, depth, 4, seed=3))
    w, h = 16, 16
    got = p.dds_encode_cube(opts(fmt, B.CUBE_CROSS, mips), doc, None, B.FRONT_HAS_ALPHA, s)
    esize = doc.itemsize * 4
    srcs = (B.PixelSource * 6)(*[B.PixelSource(doc.ctypes.data + (cy * h * dw + cx * w) * esize, w, h, 4, doc.itemsize * 8, dw * esize)
                                 for cx, cy in C.CELLS[0]])
    d = B.DdsDesc(w, h, 5 if mips else 1, 6, fmt, 1)
    n = p.lib.itw_dds_file_bytes(ctypes.byref(d))
    out = np.zeros(n, np.uint8)
    f = p.lib.itw_dds_encode_pixels
    f.restype = ctypes.c_size_t
    f.argtypes = [ctypes.POINTER(B.DdsDesc), ctypes.POINTER(B.PixelSource), ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
    sp = ctypes.cast(ctypes.byref(s), ctypes.c_void_p) if s is not None else None
    assert f(ctypes.byref(d), srcs, B.FRONT_HAS_ALPHA, sp, out.ctypes.data, n) == n, p.last_error()
    assert np.array_equal(got, out)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,source,mips,level", [(71, 0, 0, -1), (77, 0, 1, -1), (99, 0, 1, -1), (98, 1, 1, 2), (78, 1, 0, -1),
                                                   (95, 0, 0, 1), (95, 1, 1, -1)])
def test_gpu_round_trip_through_the_open_path(fmt, source, mips, level):
    """The file opens as a cube map: six four-plane layers of the file's top level, each the decoded face (DirectX::Decompress to the
    open path's target); the alpha plane is the decoded alpha, or 255 / 1.0 for a cube map with alpha, as the plug-in's read path does."""
    p = T.product()
    prof = FORMATS[fmt]
    s = p.profile(prof) if prof else None
    depth = 32 if fmt == 95 else 8
    o = opts(fmt, source, mips, level)
    if source == B.CUBE_CROSS:
        doc, faces = cross_doc(fmt, 52, 30, depth, 4, seed=11), None
    else:
        doc, faces = cross_doc(fmt, 13, 10, depth, 4, seed=12), face_layers(fmt, 13, 10, depth, seed=13)
    blob = p.dds_encode_cube(o, doc, faces, B.FRONT_HAS_ALPHA, s)
    info, layers = p.dds_open_layers(blob)
    L = max(level, 0)
    want_faces = C.oracle_faces(o, doc, faces, B.FRONT_HAS_ALPHA)
    hl, wl = C.oracle_chain(fmt, want_faces[0], L + 1)[L].shape[:2]
    assert info.desc.is_cubemap == 1 and info.layers == 6 and len(layers) == 6 and (info.width, info.height) == (wl, hl)
    assert info.planes == 4                                             # layers carry a transparency plane (IntelPlugin.cpp:2599-2602)
    for i, (layer, face) in enumerate(zip(layers, want_faces)):
        blocks = C.encode_level(fmt, C.oracle_chain(fmt, face, L + 1)[L], prof)
        decoded = PL.ref_decompress(fmt, blocks, wl, hl, info.target_dxgi)
        assert np.array_equal(layer[..., :3], decoded[..., :3]), i
        if info.has_alpha:                                                  # a cube map with alpha: the last plane forced opaque
            assert (layer[..., 3] == (1.0 if layer.dtype == np.float32 else 255)).all(), i
        else:
            assert np.array_equal(layer[..., 3], decoded[..., 3]), i


def _device_doc(doc, keep):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(doc).view(np.uint8).reshape(-1)).cuda()
    keep.append(t)
    return B.PixelSource(t.data_ptr(), doc.shape[1], doc.shape[0], doc.shape[2], doc.itemsize * 8, 0)


def _device_faces(faces, w, h, pitch, keep):
    import torch
    arr = (B.LayerSource * 6)()

    def dev(a):
        buf = np.zeros((h, pitch), a.dtype)
        buf[:, :w] = a
        t = torch.from_numpy(buf.view(np.uint8).reshape(-1)).cuda()
        keep.append(t)
        return t.data_ptr()
    for i, face in enumerate(faces):
        if face is None:
            continue
        arr[i].channel_count = len(face[0])
        for c, pl in enumerate(face[0]):
            arr[i].channels[c] = dev(pl)
        arr[i].alpha = dev(face[1]) if face[1] is not None else None
        arr[i].row_bytes = pitch * face[0][0].itemsize
    return arr


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,source", SAVE_CASES)
def test_gpu_device_operands_give_the_host_file(fmt, source):
    """Device documents and device face layers (rows wider than the document) give the host-operand file, for every format, source
    and level class."""
    p = T.product()
    prof = FORMATS[fmt]
    s = p.profile(prof) if prof else None
    sp = ctypes.cast(ctypes.byref(s), ctypes.c_void_p) if s is not None else None
    depth = {71: 16, 72: 8, 77: 8, 78: 32, 95: 32, 98: 8, 99: 16}[fmt]
    for mips, level in ((1, -1), (0, 1)):
        o = opts(fmt, source, mips, level)
        keep = []
        if source == B.CUBE_CROSS:
            doc = cross_doc(fmt, 48, 30, depth, 4, seed=fmt + mips)
            want = p.dds_encode_cube(o, doc, None, B.FRONT_HAS_ALPHA, s)
            src, arr = _device_doc(doc, keep), None
        else:
            doc = cross_doc(fmt, 13, 7, depth, 4, seed=fmt + mips)
            faces = face_layers(fmt, 13, 7, depth, seed=fmt * 7 + mips)
            want = p.dds_encode_cube(o, doc, faces, B.FRONT_HAS_ALPHA, s)
            src, arr = B.PixelSource(None, 13, 7, 4, depth, 0), _device_faces(faces, 13, 7, 16, keep)
        out = np.zeros(want.size, np.uint8)
        assert p.dds_encode_cube_raw(o, src, arr, B.FRONT_HAS_ALPHA, sp, out.ctypes.data, out.size) == want.size, p.last_error()
        assert np.array_equal(out, want), (mips, level)


@pytest.mark.gpu
def test_gpu_device_operands():
    import torch
    p = T.product()
    fmt, w, h, depth = 77, 13, 7, 16
    doc = cross_doc(fmt, 48, 30, depth, 4, seed=2)
    want = p.dds_encode_cube(opts(fmt, B.CUBE_CROSS, 1, 1), doc, None, B.FRONT_HAS_ALPHA)
    d_doc = torch.from_numpy(doc.view(np.int16)).cuda()
    src = B.PixelSource(d_doc.data_ptr(), 48, 30, 4, depth, 0)
    n = p.cube_layout(opts(fmt, B.CUBE_CROSS, 1, 1), 48, 30)[0]
    out = np.zeros(n, np.uint8)
    assert p.dds_encode_cube_raw(opts(fmt, B.CUBE_CROSS, 1, 1), src, None, B.FRONT_HAS_ALPHA, None, out.ctypes.data, n) == n, p.last_error()
    assert np.array_equal(out, want)
    # face layers in device memory, rows wider than the document
    comp = cross_doc(fmt, w, h, depth, 4, seed=4)
    faces = face_layers(fmt, w, h, depth, seed=5)
    want = p.dds_encode_cube(opts(fmt, B.CUBE_LAYERS, 1), comp, faces, B.FRONT_HAS_ALPHA)
    keep = []

    def dev(a):
        buf = np.zeros((h, 16), a.dtype)
        buf[:, :w] = a
        t = torch.from_numpy(buf.view(np.int16)).cuda()
        keep.append(t)
        return t.data_ptr()
    arr = (B.LayerSource * 6)()
    for i, face in enumerate(faces):
        if face is None:
            continue
        arr[i].channel_count = len(face[0])
        for c, pl in enumerate(face[0]):
            arr[i].channels[c] = dev(pl)
        arr[i].alpha = dev(face[1]) if face[1] is not None else None
        arr[i].row_bytes = 32
    src = B.PixelSource(None, w, h, 4, depth, 0)                     # a layer cube reads only the size and depth of the document
    n = p.cube_layout(opts(fmt, B.CUBE_LAYERS, 1), w, h)[0]
    out = np.zeros(n, np.uint8)
    assert p.dds_encode_cube_raw(opts(fmt, B.CUBE_LAYERS, 1), src, arr, B.FRONT_HAS_ALPHA, None, out.ctypes.data, n) == n, p.last_error()
    assert np.array_equal(out, want)
    # a device display
    img, size = p.preview_cube(opts(fmt, B.CUBE_LAYERS, 0, 1), comp, faces, B.FRONT_HAS_ALPHA)
    d_img = torch.zeros(img.shape, dtype=torch.uint8, device="cuda")
    keep_faces = []
    arr = p.cube_faces(faces, comp.dtype, keep_faces)
    src = B.PixelSource(comp.ctypes.data, w, h, 4, depth, 0)
    got_size = ctypes.c_size_t(0)
    disp = B.RgbaSurface(d_img.data_ptr(), img.shape[1], img.shape[0], img.shape[1] * 4)
    assert p.preview_cube_raw(opts(fmt, B.CUBE_LAYERS, 0, 1), src, arr, B.FRONT_HAS_ALPHA, None, disp, ctypes.byref(got_size)) == 0, p.last_error()
    assert got_size.value == size and np.array_equal(d_img.cpu().numpy(), img)


@pytest.mark.gpu
def test_gpu_refusals_enqueue_nothing():
    p = T.product()
    doc = cross_doc(98, 64, 48, 8, 4, seed=1)
    s = p.profile("veryfast")
    sp = ctypes.cast(ctypes.byref(s), ctypes.c_void_p)
    p.dds_encode_cube(opts(98, B.CUBE_CROSS, 1), doc, None, 1, s)            # warm: the context exists
    faces = face_layers(98, 16, 12, 8, seed=3)
    keep = []
    good_faces = p.cube_faces(faces, np.uint8, keep)
    comp = np.zeros((12, 16, 4), np.uint8)

    def call(o, document=doc, arr=None, flags=1, settings=sp):
        src = B.PixelSource(document.ctypes.data, document.shape[1], document.shape[0], document.shape[2], 8, 0)
        out = np.full(1 << 16, 0xAB, np.uint8)
        disp = np.full((48, 64, 4), 0xCD, np.uint8)
        before = p.launch_count()
        assert p.dds_encode_cube_raw(o, src, arr, flags, settings, out.ctypes.data, out.size) == 0 and p.last_error() != ""
        assert p.preview_cube_raw(o, src, arr, flags, settings, B.RgbaSurface(disp.ctypes.data, 64, 48, 256), None) != 0
        assert p.last_error() != ""
        assert (out == 0xAB).all() and (disp == 0xCD).all() and p.launch_count() == before
    call(opts(80))                                                             # BC4: no cube map in the plug-in
    call(opts(83))
    call(opts(96))                                                             # BC6H_SF16
    call(opts(98, level=5))                                                    # 16 x 16 faces: five levels
    call(opts(98, level=-2))
    call(opts(98, source=7))
    call(opts(98), document=np.zeros((2, 3, 4), np.uint8))                     # smaller than one texel per face
    call(opts(98), flags=1 | 4)                                                # flip: normal maps only
    call(opts(98), flags=1 | 16)                                               # normalise: normal maps only
    call(opts(98), settings=None)                                              # BC7 needs settings
    for disp in (B.RgbaSurface(None, 64, 12, 256), B.RgbaSurface(0, 64, 12, 256)):  # preview only: null display
        assert p.preview_cube_raw(opts(98, level=1), B.PixelSource(doc.ctypes.data, 64, 48, 4, 8, 0), None, 1, sp, disp, None) != 0
    for w, h, stride in ((64, 48, 256), (32, 24, 64), (32, 24, 96)):           # cross of level 1 is 32 x 24: size, then stride
        disp = np.full((h, w, 4), 0xCD, np.uint8)
        before = p.launch_count()
        assert p.preview_cube_raw(opts(98, level=1), B.PixelSource(doc.ctypes.data, 64, 48, 4, 8, 0), None, 1, sp,
                                  B.RgbaSurface(disp.ctypes.data, w, h, stride), None) != 0 and p.last_error() != ""
        assert (disp == 0xCD).all() and p.launch_count() == before, (w, h, stride)
    call(opts(98, B.CUBE_LAYERS), document=comp, arr=None)                     # no face list
    bad = p.cube_faces(faces, np.uint8, keep)
    bad[1].channel_count = 4
    call(opts(98, B.CUBE_LAYERS), document=comp, arr=bad)
    bad = p.cube_faces(faces, np.uint8, keep)
    bad[0].channels[1] = None
    call(opts(98, B.CUBE_LAYERS), document=comp, arr=bad)
    bad = p.cube_faces(faces, np.uint8, keep)
    bad[3].row_bytes = 15
    call(opts(98, B.CUBE_LAYERS), document=comp, arr=bad)
    assert good_faces is not None
