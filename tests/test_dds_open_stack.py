"""The stack open path on the CPU (include/itw_bcn.h section 17): header verdicts and payload sizes of volumes, 1-D textures and arrays
in one or more forms of every family against the compiled LoadFromDDSMemory (_DecodeDDSHeader, ScratchImage::Initialize, _CopyImage's
size check), the edge headers, the image each call reads against the compiled GetImage, refusals (all before any CUDA call), the
older calls' refusals of the new shapes, and the layout."""
import ctypes

import numpy as np
import pytest

import itw_testlib as T
import open_lib
import open_stack_lib as S
import open_uncompressed_lib as U

B = T.binding

pytestmark = pytest.mark.skipif(not S.refs_ready(), reason="oracle/_ref/libitw_ref_open_stack.so not built")

SIZES = [(1, 1, 1, None), (5, 3, 7, None), (4, 4, 64, 7)]


def verdict(file):
    """Open the file with its payload one byte short (every accepted header then fails at its size check, before any CUDA call)."""
    lib = T.product()
    f = np.ascontiguousarray(file[:-1])
    info = B.DdsStackInfo()
    before = bytes(info)
    launches = lib.launch_count()
    assert lib.dds_open_stack_raw(f.ctypes.data, f.size, info) != 0
    assert bytes(info) == before and lib.launch_count() == launches
    msg = lib.last_error()
    assert msg.startswith("itw_dds_open_stack: "), msg
    if "truncated file" in msg:
        return True, int(msg.split("needs ")[1].rstrip(")")), msg
    return False, None, msg


def mips_of(shape, w, h, d, mips):
    dim = S.SHAPES[shape][0]
    if mips is not None and dim == 3:
        return mips
    return S.count_mips(w, 1 if dim == 1 else h, d if dim == 3 else 1)


@pytest.mark.parametrize("label", sorted(S.FORMS))
@pytest.mark.parametrize("shape", sorted(S.SHAPES))
@pytest.mark.parametrize("w,h,d,mips", SIZES)
def test_header_verdicts_and_sizes_against_load_from_dds_memory(label, shape, w, h, d, mips):
    """The file loads, LoadFromDDSMemory's description is the expected one, the product needs exactly the file's bytes, and one byte
    less fails in both."""
    if not S.shape_ok(label, shape):
        pytest.skip("the form cannot express the shape")
    n = mips_of(shape, w, h, d, mips)
    file = S.make_file(label, shape, w, h, d, n, seed=w + d)
    m = S.ref_load(file)
    dim, _, items, cube = S.SHAPES[shape]
    assert m is not None
    assert (m["width"], m["height"], m["depth"], m["mip_levels"]) == (w, 1 if dim == 1 else h, d if dim == 3 else 1, n)
    assert (m["array_size"], m["cube"], m["dimension"], m["format"]) == (items * (6 if cube else 1), int(cube), dim + 1, S.FORMS[label][3])
    assert S.ref_load(file[:-1]) is None
    ok, need, msg = verdict(file)
    assert ok and need == file.size, msg


def with_caps2(head, caps2):
    return head[:112] + caps2.to_bytes(4, "little") + head[116:]


def test_edge_headers_are_refused_where_the_reference_refuses_them():
    cases = [
        # a volume flag on a cube map: read as a volume by both
        (with_caps2(S.header("A8B8G8R8", "legacy-volume", 4, 4, 2, 1), 0xFE00), 4 * 4 * 4 * 2, True),
        (S.header("BC7", "dx10-volume", 4, 4, 2, 1, hflags=0x1007), 16 * 2, False),       # dimension 4 without the volume flag
        (S.header("DX10-11", "1d", 4, 4, 1, 1, height=2), 4 * 8, False),               # DDS_HEIGHT with height 2
        (S.header("DX10-11", "1d", 4, 4, 1, 1, height=2, hflags=0x1005), 4 * 8, True),  # height 2 without DDS_HEIGHT: height 1
        (S.header("A8R3G3B2", "legacy-volume", 4, 4, 0, 1), 4 * 4 * 2, False),         # depth 0
        (S.header("DX10-2", "dx10-volume", 4, 4, 64, 8), 1 << 16, False),               # one level above _CountMips3D
        (S.header("DX10-2", "dx10-volume", 4, 4, 64, 1, count=2), 1 << 16, False),      # a volume array
        (S.header("DX10-10", "cube-array-2", 1, 1, 1, 1, count=0x80000001), 6 * 64, False),
        (S.header("DX10-10", "2d-array-2", 1, 1, 1, 1, count=0), 64, False),
        (S.header("DX10-10", "2d-array-2", 1, 1, 1, 1, dim=5), 64, False),
    ]
    for head, payload, loads in cases:            # the 0x80000001 cube array walks _DetermineImageArray's 12.9e9 images: slow
        m = S.ref_load(head + bytes(payload))
        assert (m is not None) == loads, head
        if loads:
            file = np.frombuffer(head + bytes(m["payload"]), np.uint8).copy()
            ok, need, msg = verdict(file)
            assert ok and need == file.size, msg
        else:
            ok, _, msg = verdict(np.frombuffer(head + bytes(payload + 1), np.uint8).copy())
            assert not ok, msg
    bc1_array = S.header("BC1", "2d-array-2", 4, 4, 1, 1, dim=3)                  # loads, but is itw_dds_open's
    assert S.ref_load(bc1_array + bytes(16)) is not None
    assert "open it with itw_dds_open" in verdict(np.frombuffer(bc1_array + bytes(17), np.uint8).copy())[2]
    assert "32 bits" in verdict(np.frombuffer(cases[7][0] + bytes(6 * 64 + 1), np.uint8).copy())[2]


@pytest.mark.parametrize("shape", ["legacy-volume", "dx10-volume", "1d-array-3", "1d-array-6", "2d-array-2", "2d-array-6", "cube-array-2"])
@pytest.mark.parametrize("options", S.OPTIONS)
def test_each_call_reads_the_image_get_image_names(shape, options):
    """DoReadContinue's GetImage(mip, item, slice) for every call and every layout option is the image the layer call reads: item
    `call` of a six-item texture, else slice 0 of level `call` (mips as layers) or the first image."""
    label = "A8B8G8R8" if shape == "legacy-volume" else "DX10-11"
    w, h, d = 8, 4, 16
    n = mips_of(shape, w, h, d, None)
    file = S.make_file(label, shape, w, h, d, n)
    lib = T.product()
    m = S.ref_load(file)
    info = B.DdsStackInfo()
    dim = S.SHAPES[shape][0]
    info.desc = B.DdsDesc(m["width"], m["height"], n, m["array_size"], m["format"], m["cube"])
    info.dimension, info.slices, info.section = dim, m["depth"], S.FORMS[label][0]
    info.form = B.RAW_A8B8G8R8 if label == "A8B8G8R8" else B.RAW_DX10
    info.payload_offset, info.has_alpha = m["offset"], 1
    lib.dds_stack_layout(info, options)
    start = open_lib.read_start(B.DdsDesc(m["width"], m["height"], n, m["array_size"], 77, m["cube"]), False, options)
    assert info.calls == start["calls"]
    images = S.ref_images(file)
    for call in range(info.calls):
        mip, item, slice_ = S.call_image(start, call)
        index = S.ref_get_image(file, mip, item, slice_)
        off = images[index][0] - m["offset"]
        unit = S.FORMS[label][4]
        per_item = sum(S.level(d if dim == 3 else 1, l) * S.level(w, l) * S.level(m["height"], l) * unit for l in range(n))
        before = sum(S.level(d if dim == 3 else 1, l) * S.level(w, l) * S.level(m["height"], l) * unit for l in range(mip))
        assert off == item * per_item + before, (call, index)
        if m["array_size"] == 6:
            assert (mip, item) == (0, call)


def refused(file, text):
    lib = T.product()
    info = B.DdsStackInfo()
    launches = lib.launch_count()
    assert lib.dds_open_stack_raw(file.ctypes.data, file.size, info) != 0
    msg = lib.last_error()
    assert text in msg and msg.startswith("itw_dds_open_stack: "), msg
    assert bytes(info) == bytes(B.DdsStackInfo()) and lib.launch_count() == launches
    return msg


def test_refusals_name_the_serving_call_and_launch_nothing():
    refused(U.legacy_file("A8B8G8R8", 4, 4), "a 2-D texture: open it with itw_dds_open_uncompressed")
    refused(U.legacy_file("A8B8G8R8", 4, 4, cube=True), "one cube map: open it with itw_dds_open_uncompressed")
    refused(U.dx10_file(11, 4, 4), "itw_dds_open_uncompressed")
    refused(np.frombuffer(U.header(4, 4, 1, S.FORMS["DXT5"][1]) + bytes(16), np.uint8).copy(), "a 2-D texture: open it with itw_dds_open")
    refused(np.frombuffer(U.header(4, 4, dx10=(10, 3, 0, 1)) + bytes(128), np.uint8).copy(), "itw_dds_open_converted")
    refused(np.frombuffer(U.header(4, 4, dx10=(84, 3, 4, 1)) + bytes(96), np.uint8).copy(), "one cube map: open it with itw_dds_open_other_bc")
    refused(np.frombuffer(U.header(4, 4, 1, S.FORMS["P8"][1]) + bytes(1024 + 16), np.uint8).copy(), "itw_dds_open_expanded")
    refused(np.frombuffer(U.header(4, 4, dx10=(98, 3, 0, 2)) + bytes(32), np.uint8).copy(), "open it with itw_dds_open")
    # every family's format reasons stay the same
    vol = lambda pf: S.header("A8B8G8R8", "legacy-volume", 4, 4, 2, 1)[:76] + U.header(4, 4, 1, pf)[76:]
    refused(np.frombuffer(vol((U.RGB, 0, 8, 0xe0, 0x1c, 0x03, 0)) + bytes(64), np.uint8).copy(), "R3G3B2")
    refused(np.frombuffer(vol((U.RGBA, 0, 32, 0xff0000, 0xff00, 0xff, 0xff000000)) + bytes(128), np.uint8).copy(), "WIC")
    refused(np.frombuffer(U.header(4, 4, dx10=(6, 2, 0, 2)) + bytes(96), np.uint8).copy(), "R32G32B32_FLOAT")
    refused(np.frombuffer(U.header(4, 4, dx10=(30, 2, 0, 2)) + bytes(96), np.uint8).copy(), "UINT")
    refused(np.frombuffer(U.header(4, 4, dx10=(87, 2, 0, 2)) + bytes(96), np.uint8).copy(), "WIC")
    refused(np.frombuffer(S.header("DX10-2", "dx10-volume", (1 << 24) + 1, 1, 1, 1) + bytes(64), np.uint8).copy(), "above 16777216")
    refused(np.frombuffer(S.header("DX10-2", "dx10-volume", 1, 1, (1 << 24) + 1, 1) + bytes(64), np.uint8).copy(), "depth above")


def dds_open_raw(lib, file, info):
    """itw_dds_open's status on a host file."""
    f = lib.lib.itw_dds_open
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(B.DdsOpenInfo)]
    return f(file.ctypes.data, file.size, ctypes.byref(info))


def test_older_calls_keep_refusing_the_new_shapes():
    """The calls of sections 13-16 refuse every new shape with their current texts; itw_dds_open refuses 'DX10' volumes and 1-D
    textures.  A legacy-header DXT1 volume is the known exception: itw_dds_open never tests DDS_HEADER_FLAGS_VOLUME and reads it as
    a 2-D texture (its size check asks for level 0's slice 0 chain only), which this test pins as today's behaviour."""
    lib = T.product()
    calls = {B.STACK_RAW: (lib.dds_open_uncompressed_raw, B.DdsUncompressedInfo, "itw_dds_open_uncompressed"),
             B.STACK_CONVERTED: (lib.dds_open_converted_raw, B.DdsConvertedInfo, "itw_dds_open_converted"),
             B.STACK_OTHER_BC: (lib.dds_open_other_bc_raw, B.DdsOtherBcInfo, "itw_dds_open_other_bc"),
             B.STACK_EXPANDED: (lib.dds_open_expanded_raw, B.DdsExpandedInfo, "itw_dds_open_expanded")}
    for label, form in S.FORMS.items():
        for shape in S.SHAPES:
            if not S.shape_ok(label, shape) and not (form[0] == B.STACK_BC and S.SHAPES[shape][0] == 2 and form[2]):
                continue
            file = S.make_file(label, shape, 8, 4, 4, 1)
            launches = lib.launch_count()
            if form[0] == B.STACK_BC:
                info = B.DdsOpenInfo()
                if S.SHAPES[shape][0] == 2 or S.SHAPES[shape][1] == "legacy":
                    continue                                        # its own 2-D arrays; the legacy volume is the exception below
                assert dds_open_raw(lib, file, info) != 0
                assert "not a DDS file of a supported block-compressed format" in lib.last_error(), (label, shape)
            else:
                fn, cls, who = calls[form[0]]
                info = cls()
                assert fn(file.ctypes.data, file.size, info) != 0
                msg = lib.last_error()
                assert msg.startswith(who + ": ") and ("volume" in msg or "dimension" in msg or "an array of" in msg), (label, shape, msg)
            assert lib.launch_count() == launches
    # the legacy DXT1 volume: accepted by itw_dds_open as an 8 x 4 2-D texture, whose size check is all this CPU test reaches
    head = S.header("DXT5", "legacy-volume", 8, 4, 4, 1)
    head = head[:84] + U.fourcc("DXT1").to_bytes(4, "little") + head[88:]
    short = np.frombuffer(head + bytes(2 * 8 - 1), np.uint8).copy()
    info = B.DdsOpenInfo()
    assert dds_open_raw(lib, short, info) != 0
    assert "truncated file (143 bytes, the header needs 144)" in lib.last_error(), lib.last_error()


def test_layout_and_layer_reads_refuse_before_any_cuda_call():
    lib = T.product()
    file = S.make_file("DX10-11", "2d-array-2", 4, 4, 1, 1)
    info = B.DdsStackInfo()
    info.desc = B.DdsDesc(4, 4, 1, 2, 11, 0)
    info.dimension, info.slices, info.section, info.form, info.payload_offset = 2, 1, B.STACK_RAW, B.RAW_DX10, 148
    lib.dds_stack_layout(info, 0)
    assert (info.calls, info.planes, info.depth, info.target_dxgi) == (1, 3, 16, 11)
    bad = B.DdsStackInfo.from_buffer_copy(bytes(info))
    bad.desc.array_size = 1                                         # a plain 2-D texture is not a description of this call
    assert lib.dds_stack_layout_raw(bad, 0) != 0 and "not a description" in lib.last_error()
    bad = B.DdsStackInfo.from_buffer_copy(bytes(info))
    bad.section = B.STACK_BC
    assert lib.dds_stack_layout_raw(bad, 0) != 0 and "not a description" in lib.last_error()
    out = np.full((4, 4, 3), 0x5A, np.uint16)
    launches = lib.launch_count()
    for size, call, text in [(file.size - 1, 0, "truncated"), (file.size, 1, "call out of range")]:
        assert lib.dds_read_stack_layer_raw(file.ctypes.data, size, info, call, out.ctypes.data) != 0
        assert text in lib.last_error(), lib.last_error()
    other = S.make_file("DX10-11", "1d-array-3", 4, 4, 1, 1)
    assert lib.dds_read_stack_layer_raw(other.ctypes.data, other.size, info, 0, out.ctypes.data) != 0
    assert "does not match" in lib.last_error() or "truncated" in lib.last_error()
    assert lib.launch_count() == launches and (out == 0x5A).all()
