"""The stack open path (include/itw_bcn.h section 17) on the GPU: every decision and every layer byte for byte against the reference
pipeline of tests/open_stack_lib.py (the cut loader, image table and GetImage, each family's own reference decode / convert / expand
and alpha check, DoReadStart / DoReadContinue restated), for every load-dialog answer.  Forms of every family in volumes, 1-D arrays
and 2-D / cube arrays, host and device operands with wide rows, one translucent texel only in a volume's last slice of its deepest
level or in the last item's smallest mip, and six-item non-cube arrays whose layers get their alpha forced."""
import numpy as np
import pytest

import itw_testlib as T
import open_stack_lib as S

B = T.binding

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    if not S.refs_ready():
        pytest.skip("oracle/_ref/libitw_ref_open_stack.so not built")
    return T.product()


def check_open(lib, label, file, options=S.OPTIONS):
    """Every option: info and every layer equal the oracle's; returns the last info."""
    file = np.ascontiguousarray(file)
    for opt in options:
        m, start, want = S.oracle_open(label, file, opt)
        info, got = lib.dds_open_stack_layers(file, opt)
        d = info.desc
        assert (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap) == \
            (m["width"], m["height"], m["mip_levels"], m["array_size"], m["format"], m["cube"])
        assert (info.dimension, info.slices, info.section, info.payload_offset) == \
            (m["dimension"] - 1, m["depth"], S.FORMS[label][0], m["offset"])
        for k, v in S.info_fields(info).items():
            assert v == start[k], (label, k, v, start[k], opt)
        assert len(got) == len(want)
        for c, (g, w) in enumerate(zip(got, want)):
            assert g.shape == w.shape and g.dtype == w.dtype, (label, c)
            assert g.tobytes() == w.tobytes(), (label, opt, c, int((g != w).sum()))
    return info


CASES = [(label, shape) for label in S.FORMS for shape in ("legacy-volume", "dx10-volume", "1d-array-6", "2d-array-2", "cube-array-2")
         if S.shape_ok(label, shape)]


@pytest.mark.parametrize("label,shape", CASES)
def test_layers_against_the_reference(lib, label, shape):
    for w, h, d in ((1, 1, 1), (5, 3, 7), (9, 6, 4)):
        n = S.count_mips(w, 1 if S.SHAPES[shape][0] == 1 else h, d if S.SHAPES[shape][0] == 3 else 1)
        for mips in sorted({1, n}):
            check_open(lib, label, S.make_file(label, shape, w, h, d, mips, seed=w * 7 + mips))


@pytest.mark.parametrize("label,shape", [("DX10-2", "2d-array-2"), ("DX10-10", "2d-array-2"), ("BC7", "dx10-volume"),
                                         ("A8P8", "legacy-volume")])
def test_device_operands_and_wide_rows(lib, label, shape):
    import torch
    file = S.make_file(label, shape, 13, 7, 5, 3, seed=5)
    for opt in S.OPTIONS:
        _, _, want = S.oracle_open(label, file, opt)
        d_file = torch.from_numpy(file.copy()).cuda()
        for fptr in (file.ctypes.data, d_file.data_ptr()):
            info = B.DdsStackInfo()
            assert lib.dds_open_stack_raw(fptr, file.size, info) == 0, lib.last_error()
            lib.dds_stack_layout(info, opt)
            item = want[0].dtype.itemsize
            pitch = info.width * info.planes * item + 48
            for call in range(info.calls):
                host = np.full(info.height * pitch, 0xAB, np.uint8)
                dev = torch.full((info.height * pitch,), 0xAB, dtype=torch.uint8, device="cuda")
                for dst, out in ((host.ctypes.data, host), (dev.data_ptr(), None)):
                    assert lib.dds_read_stack_layer_raw(fptr, file.size, info, call, dst, pitch) == 0, lib.last_error()
                    got = out if out is not None else dev.cpu().numpy()
                    rows = got.reshape(info.height, pitch)
                    assert rows[:, info.width * info.planes * item:].tobytes() == b"\xab" * (info.height * 48)
                    assert rows[:, :info.width * info.planes * item].tobytes() == want[call].tobytes(), (label, opt, call)


def test_alpha_in_slices_and_items_no_layer_shows(lib):
    """One translucent texel only in the last slice of a volume's deepest level, or only in the last item's smallest mip: has_alpha
    is 1 (IsAlphaAllOpaque looks at every image).  The same files all opaque: 0."""
    w, h, d, mips = 8, 4, 16, 3                                       # level 2 holds 4 slices of 2 x 1: slices 1-3 show in no layer
    vol = S.make_file("A8B8G8R8", "legacy-volume", w, h, d, mips, payload=b"\xff" * S.payload_bytes("A8B8G8R8", w, h, d, mips, 1))
    check_open(lib, "A8B8G8R8", vol)
    assert lib.dds_open_stack_layers(vol, 0)[0].has_alpha == 0
    vol[-1] = 0x10                                                    # alpha of the last texel: the last slice of the deepest level
    info = check_open(lib, "A8B8G8R8", vol)
    assert info.has_alpha == 1 and info.slices == 16
    arr = S.make_file("DX10-10", "2d-array-2", w, h, 1, 4, payload=(np.full(S.payload_bytes("DX10-10", w, h, 1, 4, 2) // 2, 0x3C00, "<u2")).tobytes())
    assert check_open(lib, "DX10-10", arr).has_alpha == 0
    arr[-2:] = np.frombuffer(np.array([0x3800], "<u2").tobytes(), np.uint8)     # half 0.5: the last item's smallest mip
    assert check_open(lib, "DX10-10", arr).has_alpha == 1
    bc7 = S.make_file("BC7", "dx10-volume", w, h, d, mips, seed=3)
    check_open(lib, "BC7", bc7)


def test_six_item_arrays_open_as_forced_cube_layers(lib):
    for label in ("A8B8G8R8", "DX10-10", "DXT3", "A8P8", "BC7"):
        shape = "1d-array-6" if S.FORMS[label][1] is None else None
        if shape is None:
            continue
        file = S.make_file(label, shape, 7, 1, 1, 1, seed=11)
        info = check_open(lib, label, file)
        assert info.layers == 6 and info.calls == 6
    file = S.make_file("DX10-10", "2d-array-6", 6, 5, 1, 2, seed=12)
    info = check_open(lib, "DX10-10", file)
    assert info.layers == 6 and info.has_alpha == 1


def test_refusals_launch_nothing(lib):
    import torch
    file = S.make_file("DX10-2", "dx10-volume", 4, 4, 4, 1)
    d_short = torch.from_numpy(file[:-1].copy()).cuda()
    info = B.DdsStackInfo()
    launches = lib.launch_count()
    assert lib.dds_open_stack_raw(d_short.data_ptr(), file.size - 1, info) != 0 and "truncated" in lib.last_error()
    assert lib.launch_count() == launches and bytes(info) == bytes(B.DdsStackInfo())
