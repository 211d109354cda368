"""The open path for the block-compressed files itw_dds_open does not serve (include/itw_bcn.h section 15), on the CPU: the per-block
routines of the layer kernel and the alpha scan (emulated) against the reference's own _DecompressBC and _IsAlphaAllOpaqueBC, linked to
its D3DXDecodeBC2 / BC4S / BC5S; the scope against the compiled BitsPerColor / IsSRGB / HasAlpha; the refusals (all before any CUDA
call) and the layout."""
import numpy as np
import pytest

import itw_testlib as T
import open_other_bc_lib as L
import open_uncompressed_lib as U
import test_dds_open_uncompressed as TU       # g_LegacyDDSMap's header forms

B = T.binding

pytestmark = pytest.mark.skipif(L.ref() is None or U.ref() is None, reason="oracle/_ref/libitw_ref_open_other_bc.so not built")

RNG = np.random.default_rng(15)


def index_bits(idx, bits):
    return sum(int(v) << (bits * k) for k, v in enumerate(idx))


def bc4s_every_pair():
    """One block per (red_0, red_1) byte pair, its sixteen indices 0..7 twice: every (red_0, red_1, index), -128 on either side included."""
    r = np.arange(65536, dtype=np.uint32)
    blk = np.zeros((65536, 8), np.uint8)
    blk[:, 0], blk[:, 1] = r & 255, r >> 8
    blk[:, 2:] = np.frombuffer(index_bits(np.arange(16) % 8, 3).to_bytes(6, "little"), np.uint8)
    return blk


def test_bc4s_every_endpoint_pair_and_index():
    blk = bc4s_every_pair()
    assert np.array_equal(L.emu_blocks(81, blk.tobytes()), L.ref_blocks(81, blk.tobytes(), 28))


def test_bc5s_both_halves():
    pairs = bc4s_every_pair()
    for g in (np.roll(pairs, 1, 0), pairs[RNG.permutation(65536)]):
        blk = np.concatenate([pairs, g], 1)
        assert np.array_equal(L.emu_blocks(84, blk.tobytes()), L.ref_blocks(84, blk.tobytes(), 28))
        swapped = np.concatenate([g, pairs], 1)
        assert np.array_equal(L.emu_blocks(84, swapped.tobytes()), L.ref_blocks(84, swapped.tobytes(), 28))


def bc2_nibble_blocks():
    """Every alpha nibble in every slot (the other slots random), over colour halves of both endpoint orders."""
    out = []
    for slot in range(16):
        for n in range(16):
            for order in range(2):
                a = RNG.integers(0, 16, 16)
                a[slot] = n
                c = RNG.integers(0, 65536, 2)
                c0, c1 = (max(c), min(c)) if order == 0 else (min(c), max(c))
                colour = int(c0) | (int(c1) << 16) | (int(RNG.integers(0, 1 << 32)) << 32)
                out.append(index_bits(a, 4).to_bytes(8, "little") + colour.to_bytes(8, "little"))
    return b"".join(out)


@pytest.mark.parametrize("fmt", [74, 73, 75])
def test_bc2_every_nibble_in_every_slot(fmt):
    blocks = bc2_nibble_blocks()
    assert np.array_equal(L.emu_blocks(74, blocks), L.ref_blocks(fmt, blocks, L.LOADED[fmt][2]))


def bc6h_blocks():
    """BC6H blocks of the HDR corpus's values (encoded by the oracle), and random blocks: every mode, values above 1.0."""
    import hdr_corpus
    o = T.oracle()
    img = np.asarray(hdr_corpus.log_uniform(16, 32, seed=9), np.uint16)
    img = np.ascontiguousarray(np.concatenate([img.reshape(16, 32, 4), np.asarray(hdr_corpus.boundary(16, 32), np.uint16).reshape(16, 32, 4)]))
    corpus = np.asarray(o.encode("BC6H", img, o.profile("bc6h_veryfast")), np.uint8).tobytes()
    return corpus + RNG.integers(0, 256, 16 * 8192, dtype=np.uint8).tobytes()


def test_bc6h_typeless_into_16_bit_unorm():
    blocks = bc6h_blocks()
    want = L.ref_blocks(94, blocks, 11)
    assert np.array_equal(L.emu_blocks(94, blocks), want)
    assert (want[..., :3] == 65535).any() and (want[..., 3] == 65535).all()     # values above 1.0 saturate


@pytest.mark.parametrize("typeless,twin", [(70, 71), (73, 74), (76, 77), (79, 80), (82, 83), (97, 98)])
def test_typeless_decodes_as_its_typed_twin(typeless, twin):
    bpb = L.LOADED[typeless][1]
    blocks = RNG.integers(0, 256, 4096 * bpb, dtype=np.uint8).tobytes()
    want = L.ref_blocks(typeless, blocks, 28)
    assert np.array_equal(want, L.ref_blocks(twin, blocks, 28))
    assert np.array_equal(L.emu_blocks(L.LOADED[typeless][0], blocks), want)


def test_alpha_predicate_bc2_nibbles_14_and_15_in_every_slot():
    blocks = []
    for slot in range(16):
        for n in (14, 15):
            a = np.full(16, 15)
            a[slot] = n
            blocks.append(index_bits(a, 4).to_bytes(8, "little") + RNG.integers(0, 256, 8, dtype=np.uint8).tobytes())
    blocks = b"".join(blocks)
    for cols in range(1, 5):
        for rows in range(1, 5):
            want = L.blocks_opaque("ref", 74, blocks, cols, rows)
            assert np.array_equal(L.blocks_opaque("emu", 74, blocks, cols, rows), want)
            assert np.array_equal(L.blocks_opaque("ref", 73, blocks, cols, rows), want)
    assert set(L.blocks_opaque("ref", 74, blocks)) == {0, 1}


def test_alpha_predicate_bc1_typeless_punch_through_inside_and_outside_ragged_edges():
    blocks = []
    for k in range(16):                                  # one punch-through texel at k, three-colour mode
        idx = np.zeros(16, int)
        idx[k] = 3
        for c0, c1 in ((0x1234, 0x5678), (0x5678, 0x1234), (0x4444, 0x4444)):
            blocks.append((c0 | (c1 << 16) | (index_bits(idx, 2) << 32)).to_bytes(8, "little"))
    blocks = b"".join(blocks) + RNG.integers(0, 256, 8 * 4096, dtype=np.uint8).tobytes()
    for cols in range(1, 5):
        for rows in range(1, 5):
            want = L.blocks_opaque("ref", 70, blocks, cols, rows)
            assert np.array_equal(L.blocks_opaque("emu", 71, blocks, cols, rows), want), (cols, rows)
    assert set(L.blocks_opaque("ref", 70, blocks)) == {0, 1}


@pytest.mark.parametrize("fmt,decoder", [(76, 77), (97, 98)])
def test_alpha_predicate_bc3_bc7_typeless(fmt, decoder):
    blocks = RNG.integers(0, 256, 16 * 4096, dtype=np.uint8).tobytes() + L.opaque_blocks(fmt, 64).tobytes()
    for cols, rows in ((4, 4), (1, 3), (2, 2)):
        assert np.array_equal(L.blocks_opaque("emu", decoder, blocks, cols, rows), L.blocks_opaque("ref", fmt, blocks, cols, rows))


def verdict(file):
    """Open the header alone (every accepted header then fails at its size check, before any CUDA call)."""
    lib = T.product()
    dx10 = file.size >= 148 and bytes(file[84:88]) == b"DX10"
    f = np.ascontiguousarray(file[:min(file.size, 148 if dx10 else 128)])
    info = B.DdsOtherBcInfo()
    before = bytes(info)
    assert lib.dds_open_other_bc_raw(f.ctypes.data, f.size, info) != 0
    assert bytes(info) == before
    msg = lib.last_error()
    assert msg.startswith("itw_dds_open_other_bc: "), msg
    if "truncated file" in msg:
        return True, int(msg.split("needs ")[1].rstrip(")")), msg
    return False, None, msg


def test_scope_against_bits_per_color_is_srgb_has_alpha():
    """Every DXGI id in a 'DX10' header and every legacy form: the product opens the file iff its loaded format and form are in the
    table; its target, depth and alpha rule are the compiled BitsPerColor / IsSRGB / HasAlpha with the BC1 exclusion; every refusal
    names its reason."""
    for f in range(1, 121):
        file = np.frombuffer(U.header(4, 4, dx10=(f, 3, 0, 1)) + bytes(64), np.uint8).copy()
        m = U.ref_header(file)
        ok, need, msg = verdict(file)
        served = f in L.DX10
        assert ok == served, (f, msg)
        decoder, target, depth, has_alpha, bpb = L.emu_scope(f)
        assert (decoder >= 0) == (f in L.LOADED), f
        if served:
            assert need == 148 + bpb
            assert (target, depth) == L.ref_target(f), f
            assert has_alpha == (L.ref().ref_has_alpha(f) and f not in (71, 72)), f
        elif m is None or f in (0,) or f > 120 or 111 <= f <= 114:
            assert "unknown or palettised" in msg, (f, msg)
        elif 70 <= f <= 84 or 94 <= f <= 99:
            assert "itw_dds_open" in msg and "opened by" in msg, (f, msg)
        else:
            assert "itw_dds_open_uncompressed or itw_dds_open_converted" in msg, (f, msg)
    served = set()
    for pf in TU.legacy_table():
        head = U.header(4, 4, 1, pf)
        m = U.ref_header(np.frombuffer(head + bytes(64), np.uint8).copy())
        ok, need, msg = verdict(np.frombuffer(head + bytes(64), np.uint8).copy())
        name = pf[1].to_bytes(4, "little").decode("latin1") if pf[0] == U.FOURCC else None
        assert ok == (name in L.LEGACY), (pf, msg)
        if ok:
            assert m["format"] == L.LEGACY[name][1] and need == 128 + L.LOADED[m["format"]][1]
            served.add(name)
        elif m is not None and (70 <= m["format"] <= 84 or 94 <= m["format"] <= 99):
            assert "opened by itw_dds_open" in msg, (pf, msg)
        elif m is not None and m["conv"] & 0x1:                                   # CONV_FLAGS_EXPAND (R8G8B8 is section 13's)
            assert "expansion" in msg or "itw_dds_open_uncompressed" in msg, (pf, msg)
        elif m is not None:
            assert "itw_dds_open_uncompressed or itw_dds_open_converted" in msg, (pf, msg)
    assert served == set(L.LEGACY)


@pytest.mark.parametrize("label,fmt,writer", L.FORMS, ids=[f[0] for f in L.FORMS])
def test_header_forms_against_decode_header(label, fmt, writer):
    for w, h, mips, cube in ((1, 1, 1, False), (5, 3, 3, False), (4, 4, 3, True)):
        file = writer(w, h, mips, cube)
        m = U.ref_header(file)
        assert m is not None and m["format"] == fmt
        ok, need, msg = verdict(file)
        assert ok and need == file.size, msg


def test_shape_refusals_leave_info_untouched():
    cases = [(np.frombuffer(U.header(4, 4, dx10=(74, 4, 0, 1)) + bytes(16), np.uint8).copy(), "volume"),
             (np.frombuffer(U.header(4, 4, dx10=(74, 3, 0, 2)) + bytes(32), np.uint8).copy(), "array"),
             (np.frombuffer(U.header(4, 4, dx10=(74, 3, 0x4, 2)) + bytes(16 * 12), np.uint8).copy(), "array of 2 cube maps"),
             (np.frombuffer(U.header(4, 4, pf=(U.FOURCC, U.fourcc("DXT3"), 0, 0, 0, 0, 0), caps2=0x600) + bytes(16), np.uint8).copy(),
              "six faces"),
             (L.legacy_file("DXT3", 8, 8)[:-1], "truncated"),
             (np.frombuffer(U.header(0, 4, dx10=(81, 3, 0, 1)) + bytes(16), np.uint8).copy(), "width or height 0"),
             (np.frombuffer(U.header(1 << 25, 4, dx10=(81, 3, 0, 1)) + bytes(16), np.uint8).copy(), "above 16777216"),
             (np.frombuffer(U.header(4, 4, 4, dx10=(81, 3, 0, 1)) + bytes(64), np.uint8).copy(), "mip levels")]
    for file, text in cases:
        info = B.DdsOtherBcInfo()
        assert T.product().dds_open_other_bc_raw(file.ctypes.data, file.size, info) != 0
        assert text in T.product().last_error(), (text, T.product().last_error())
        assert bytes(info) == bytes(B.DdsOtherBcInfo())


@pytest.mark.parametrize("options", L.OPTIONS)
@pytest.mark.parametrize("label,cube", [("BC4S", False), ("BC5S", True), ("DX10-94", False), ("DX10-94", True), ("DX10-79", False),
                                        ("DX10-82", True), ("DX10-81", False), ("DX10-84", False)])
def test_layout_for_every_option(label, cube, options):
    """Formats without alpha: the open is host-only (no scan), so the layout can be checked on the CPU."""
    lib = T.product()
    _, fmt, writer = next(f for f in L.FORMS if f[0] == label)
    file = writer(6, 5, 3 if not cube else 1, cube)
    info = lib.dds_other_bc_layout(lib.dds_open_other_bc(file.ctypes.data, file.size), options)
    m, start, _ = L.oracle_open(file, options)
    assert L.info_fields(info) == {k: start[k] for k in L.info_fields(info)}
    assert info.desc.dxgi_format == fmt and info.payload_offset == m["offset"]
    assert info.form == (L.LEGACY[label][0] if label in L.LEGACY else B.OBC_DX10)


def test_layout_and_read_refusals_before_any_cuda_call():
    lib = T.product()
    file = L.legacy_file("BC5S", 8, 8, 4)
    info = lib.dds_other_bc_layout(lib.dds_open_other_bc(file.ctypes.data, file.size), B.OPEN_MIPS)
    dst = np.full(8 * 8 * 4, 0x5A, np.uint8)
    bad = B.DdsOtherBcInfo.from_buffer_copy(info)
    bad.form = B.OBC_DXT3                                   # a form whose loaded format is not the description's
    assert lib.dds_other_bc_layout_raw(bad, 0) != 0 and "not a description" in lib.last_error()
    bad = B.DdsOtherBcInfo.from_buffer_copy(info)
    bad.desc.dxgi_format = 77                               # BC3 is a DX10 format of itw_dds_open
    assert lib.dds_other_bc_layout_raw(bad, 0) != 0
    assert lib.dds_other_bc_layout_raw(B.DdsOtherBcInfo.from_buffer_copy(info), 4) != 0 and "option" in lib.last_error()
    for call, row, text in ((4, 0, "call out of range"), (-1, 0, "call out of range"), (0, 8 * 4 - 1, "row_bytes")):
        assert lib.dds_read_other_bc_layer_raw(file.ctypes.data, file.size, info, call, dst.ctypes.data, row) != 0
        assert text in lib.last_error()
    assert lib.dds_read_other_bc_layer_raw(file.ctypes.data, file.size - 1, info, 0, dst.ctypes.data) != 0
    assert "truncated" in lib.last_error()
    other = L.legacy_file("BC5S", 8, 8, 3)
    assert lib.dds_read_other_bc_layer_raw(other.ctypes.data, other.size, info, 0, dst.ctypes.data) != 0
    assert "does not match" in lib.last_error()
    fresh = lib.dds_open_other_bc(file.ctypes.data, file.size)
    assert lib.dds_read_other_bc_layer_raw(file.ctypes.data, file.size, fresh, 0, dst.ctypes.data) != 0
    assert "not laid out" in lib.last_error()
    assert (dst == 0x5A).all()


def test_other_calls_keep_refusing_these_files():
    lib = T.product()
    for label, _, writer in L.FORMS:
        f = writer(4, 4)
        assert lib.dds_open_uncompressed_raw(f.ctypes.data, f.size, B.DdsUncompressedInfo()) != 0, label
        assert lib.dds_open_converted_raw(f.ctypes.data, f.size, B.DdsConvertedInfo()) != 0, label
        assert lib.lib.itw_dds_read_header(f.ctypes.data, f.size, ctypes_desc()) == 0, label


def ctypes_desc():
    import ctypes
    lib = T.product().lib
    lib.itw_dds_read_header.restype = ctypes.c_size_t
    lib.itw_dds_read_header.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(B.DdsDesc)]
    return ctypes.byref(B.DdsDesc())
