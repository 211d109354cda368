"""The DXGI format facts as the pure-host entry points show them, for every id 0..255: bytes per block, the DDS header a format gets
(legacy FourCC or 'DX10' extension) and reads back, and the open path's target format and depth.  The expected values are written
out here from the formats' definitions (DirectXTex DDS.h / DirectXTexDDS.cpp, the plug-in's DoReadStart), not taken from the library."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T

B = T.binding

IDS = range(256)
ITW_FORMATS = {71: 8, 77: 16, 80: 8, 83: 16, 95: 16, 96: 16, 98: 16}       # ITW_FORMAT_* -> bytes per block
DDS_BPB = {71: 8, 72: 8, 77: 16, 78: 16, 80: 8, 83: 16, 95: 16, 96: 16, 98: 16, 99: 16}
LEGACY_FOURCC = {71: b"DXT1", 77: b"DXT5", 80: b"BC4U", 83: b"BC5U"}       # every other format needs the DX10 extension
SRGB = {72, 78, 99}
HDR = {95, 96}


@pytest.fixture(scope="module")
def L():
    lib = T.product().lib
    lib.GetBytesPerBlock.restype = ctypes.c_int
    lib.itw_dds_open_layout.restype = ctypes.c_int
    lib.itw_dds_open_layout.argtypes = [ctypes.POINTER(B.DdsOpenInfo), ctypes.c_uint32]
    return lib


def test_bytes_per_block(L):
    for f in IDS:
        assert L.itw_bytes_per_block(f) == ITW_FORMATS.get(f, 0), f


def test_get_bytes_per_block_keeps_the_reference_default(L):
    # win32Threads.cpp:192-209: BC3, BC6H and BC7 (UNORM and SRGB / UF16 and SF16) are 16, everything else 8
    for f in IDS:
        assert L.GetBytesPerBlock(f) == (16 if f in (77, 78, 95, 96, 98, 99) else 8), f


def _descs(f):
    return {"2d": B.DdsDesc(64, 32, 3, 1, f, 0), "cube": B.DdsDesc(16, 16, 5, 6, f, 1)}


@pytest.mark.parametrize("kind", ["2d", "cube"])
def test_dds_header_round_trip(L, kind):
    for f in IDS:
        d = _descs(f)[kind]
        want = 0 if f not in DDS_BPB else (128 if f in LEGACY_FOURCC else 148)
        assert L.itw_dds_header_bytes(ctypes.byref(d)) == want, f
        buf = np.zeros(256, np.uint8)
        assert L.itw_dds_write_header(ctypes.byref(d), buf.ctypes.data, buf.size) == want, f
        if not want:
            continue
        assert L.itw_dds_image_bytes(ctypes.byref(d), 0) == ((d.width + 3) // 4) * ((d.height + 3) // 4) * DDS_BPB[f], f
        assert bytes(buf[84:88]) == LEGACY_FOURCC.get(f, b"DX10"), f
        if want == 148:
            assert int.from_bytes(bytes(buf[128:132]), "little") == f, f
        back = B.DdsDesc()
        assert L.itw_dds_read_header(buf.ctypes.data, want, ctypes.byref(back)) == want, f
        assert bytes(back) == bytes(d), f


def test_open_layout_target_and_depth(L):
    for f in IDS:
        info = B.DdsOpenInfo()
        info.desc = B.DdsDesc(40, 24, 1, 1, f, 0)
        rc = L.itw_dds_open_layout(ctypes.byref(info), 0)
        if f not in DDS_BPB:
            assert rc == -1, f
            continue
        assert rc == 0, f
        want_target = 2 if f in HDR else (29 if f in SRGB else 28)       # R32G32B32A32_FLOAT / R8G8B8A8_UNORM_SRGB / R8G8B8A8_UNORM
        assert (info.target_dxgi, info.depth) == (want_target, 32 if f in HDR else 8), f
