"""Parity tests proper: the CUDA path, called through the C-ABI, against the oracle (bit-exact)."""
import numpy as np
import pytest

import itw_testlib as T

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fmt,prof", T.ALL_CASES, ids=[f"{f}-{p}" for f, p in T.ALL_CASES])
def test_corpus_bit_exact(fmt, prof):
    lib, oracle = T.product(), T.oracle()
    bpb = T.binding.FORMATS[fmt][1]
    for name, img in T.corpus_for(fmt).items():
        got = T.run(lib, fmt, img, prof)
        want = T.run(oracle, fmt, img, prof)
        assert T.differing_blocks(got, want, bpb) == 0, f"{fmt}/{prof}/{name}"


def _rand_img(fmt, h, w, seed, pad=0):
    rng = np.random.default_rng(seed)
    if fmt == "BC6H":
        buf = rng.integers(0, 0x7C00, (h, w + pad, 4)).astype(np.uint16)
    else:
        buf = rng.integers(0, 256, (h, w + pad, 4), dtype=np.uint8)
    return buf[:, :w]


SHAPE_CASES = [("BC1", None), ("BC3", None), ("BC4", None), ("BC5", None), ("BC7", "basic"), ("BC7", "alpha_fast"),
               ("BC6H", "bc6h_basic")]


@pytest.mark.parametrize("fmt,prof", SHAPE_CASES, ids=[f"{f}-{p}" for f, p in SHAPE_CASES])
def test_ragged_sizes_and_padded_strides(fmt, prof):
    """Non-square surfaces, block counts that do not fill a warp batch or a CTA, row stride > row bytes,
    and sub-surfaces made by bumping ptr (what the plug-in does per slice/band, IntelPlugin.cpp:868-870)."""
    lib, oracle = T.product(), T.oracle()
    for h, w, pad in ((4, 4, 0), (4, 12, 3), (12, 20, 5), (8, 4, 1), (36, 132, 0), (260, 4, 2)):
        img = _rand_img(fmt, h, w, seed=h * 131 + w, pad=pad)
        got = T.run(lib, fmt, img, prof)
        want = T.run(oracle, fmt, np.ascontiguousarray(img), prof)
        assert np.array_equal(got, want), (h, w, pad)
    big = _rand_img(fmt, 64, 64, seed=99)
    sub = big[16:48]                                         # ptr bumped by 16 rows, same stride
    assert np.array_equal(T.run(lib, fmt, sub, prof), T.run(oracle, fmt, np.ascontiguousarray(sub), prof))


@pytest.mark.parametrize("fmt,prof", [("BC3", None), ("BC7", "fast"), ("BC6H", "bc6h_fast")])
def test_row_band_split_equals_whole_image(fmt, prof):
    """Encoding row bands separately (CompressImageMT, win32Threads.cpp:217-230) gives the whole-image bytes."""
    import importlib
    sharding = importlib.import_module("intel-texture-works-plugin_b200.sharding")
    lib = T.product()
    img = _rand_img(fmt, 128, 64, seed=5)
    whole = T.run(lib, fmt, img, prof)
    parts = []
    for i in range(5):
        y0, y1 = sharding.band_rows(128, 5, i)
        if y1 > y0:
            parts.append(T.run(lib, fmt, img[y0:y1], prof))
    assert np.array_equal(np.concatenate(parts), whole)


def test_device_pointer_paths_match_host_path():
    """src and dst may be device memory (auto-detected), and itw_encode_device enqueues on a caller stream."""
    import torch
    lib = T.product()
    for fmt, prof in (("BC1", None), ("BC7", "veryfast"), ("BC6H", "bc6h_veryfast")):
        img = _rand_img(fmt, 64, 96, seed=17)
        settings = lib.profile(prof) if prof else None
        want = lib.encode(fmt, img, settings)
        d_in = torch.from_numpy(img.copy().view(np.uint8).reshape(-1)).cuda()
        d_out = torch.zeros(want.size, dtype=torch.uint8, device="cuda")
        texel = T.binding.FORMATS[fmt][2]
        # CompressBlocks* with device src + device dst
        lib.encode_raw(fmt, d_in.data_ptr(), 96, 64, 96 * texel, d_out.data_ptr(), settings)
        torch.cuda.synchronize()
        assert np.array_equal(d_out.cpu().numpy(), want), fmt
        # device src + host dst
        h_out = np.zeros_like(want)
        lib.encode_raw(fmt, d_in.data_ptr(), 96, 64, 96 * texel, h_out.ctypes.data, settings)
        assert np.array_equal(h_out, want), fmt
        # explicit stream entry
        d_out.zero_()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            lib.encode_device(fmt, d_in.data_ptr(), 96, 64, 96 * texel, d_out.data_ptr(), settings, s.cuda_stream)
        s.synchronize()
        assert np.array_equal(d_out.cpu().numpy(), want), fmt
        # misaligned device dst (+8 bytes) goes through the internal staging buffer
        if T.binding.FORMATS[fmt][1] == 16:
            raw = torch.zeros(want.size + 16, dtype=torch.uint8, device="cuda")
            lib.encode_raw(fmt, d_in.data_ptr(), 96, 64, 96 * texel, raw.data_ptr() + 8, settings)
            torch.cuda.synchronize()
            assert np.array_equal(raw[8:8 + want.size].cpu().numpy(), want), fmt


def test_unaligned_source_pointer():
    """A source whose address / stride is not 16-byte aligned takes the byte-safe load path."""
    lib, oracle = T.product(), T.oracle()
    raw = np.random.default_rng(3).integers(0, 256, 64 * 68 * 4 + 64, dtype=np.uint8)
    img = raw[4:4 + 64 * 68 * 4].reshape(64, 68, 4)[:, :64]          # address % 16 == 4, stride 272
    for fmt in ("BC1", "BC3", "BC4", "BC5"):
        assert np.array_equal(T.run(lib, fmt, img, None), T.run(oracle, fmt, np.ascontiguousarray(img), None)), fmt


@pytest.mark.parametrize("prof", ["veryfast", "alpha_fast"])
def test_bc7_sixteen_block_rounds_ragged_and_unaligned(prof):
    """A launch runs BC7 in full rounds of sixteen blocks per warp (SMs x 16 x 16 blocks, 33 792 on a 132-SM H100); the blocks
    left over are dealt over all warps of the grid as one last round of 1, 2, 4, 8 or 16 per warp.  A host surface of 65 535
    blocks goes through the band pipeline (four launches of whole block rows, each ending in such a last round with a ragged
    last warp and CTA tile), from a host source that is 16-byte aligned and from one that is not, against the oracle.  The
    bands are staged into tight device rows, so both take the TMA-staged kernel; test_gpu_stress.py runs one launch over a
    surface of more than a wave, and reaches the plain-load kernel from a device source 4 bytes off."""
    lib, oracle = T.product(), T.oracle()
    h, w = 1020, 1028                                        # 255 x 257 = 65535 blocks
    raw = np.random.default_rng(17).integers(0, 256, h * (w + 4) * 4 + 64, dtype=np.uint8)
    off = (-raw.ctypes.data) % 16
    raw[off + 3::4][: raw.size // 8] = 255                   # first half opaque
    aligned = raw[off:off + h * (w + 4) * 4].reshape(h, w + 4, 4)[:, :w]
    shifted = raw[off + 4:off + 4 + h * (w + 4) * 4].reshape(h, w + 4, 4)[:, :w]
    assert aligned.ctypes.data % 16 == 0 and shifted.ctypes.data % 16 == 4
    for img in (aligned, shifted):
        got = T.run(lib, "BC7", img, prof)
        want = T.run(oracle, "BC7", np.ascontiguousarray(img), prof)
        assert T.differing_blocks(got, want, 16) == 0


def test_errors_are_reported_not_swallowed():
    lib = T.product()
    img = np.zeros((6, 8, 4), np.uint8)                                # height not a multiple of 4
    with pytest.raises(RuntimeError, match="multiples of 4"):
        lib.encode("BC1", img)
    bad = lib.profile("slow")
    bad.fastSkipTreshold_mode1 = 65
    with pytest.raises(RuntimeError, match="fastSkipTreshold"):
        lib.encode("BC7", np.zeros((4, 4, 4), np.uint8), bad)
    lib.encode("BC1", np.zeros((4, 4, 4), np.uint8))                   # and the error state clears
    assert lib.last_error() == ""


def test_concurrent_callers():
    """The reference is called from up to 64 pool threads at once (win32Threads.cpp:211-274)."""
    import threading
    lib, oracle = T.product(), T.oracle()
    imgs = [_rand_img("BC7", 32, 32, seed=100 + i) for i in range(8)]
    want = [T.run(oracle, "BC7", im, "veryfast") for im in imgs]
    got = [None] * 8

    def work(i):
        got[i] = lib.encode("BC7", imgs[i], lib.profile("veryfast"))
    ts = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_full_size_properties():
    """At BASELINE sizes the oracle is too slow to run whole; check size-independent properties instead:
    determinism, tile independence (a 4096^2 encode equals its 512-row bands encoded alone) and an
    oracle spot check on a band."""
    import torch
    lib, oracle = T.product(), T.oracle()
    img = T.synth.random_rgba8(4096, 4096)
    for fmt, prof in (("BC1", None), ("BC3", None), ("BC7", "basic")):
        settings = lib.profile(prof) if prof else None
        a = lib.encode(fmt, img, settings)
        b = lib.encode(fmt, img, settings)
        assert np.array_equal(a, b), "non-deterministic"
        bpb = T.binding.FORMATS[fmt][1]
        band = lib.encode(fmt, img[2048:2560], settings)
        off = (2048 // 4) * (4096 // 4) * bpb
        assert np.array_equal(a[off:off + band.size], band)
        rows = 8
        want = T.run(oracle, fmt, np.ascontiguousarray(img[1000:1000 + rows]), prof)
        off = (1000 // 4) * (4096 // 4) * bpb
        assert np.array_equal(a[off:off + want.size], want)


def test_batch_entry_streams_independent_tiles():
    """itw_encode_batch (config C5's tile stream): results equal the one-at-a-time encodes, for pageable,
    pinned and device-resident tiles, with tiles of different sizes in one batch."""
    import torch
    lib = T.product()
    fmt, prof = "BC7", "veryfast"
    settings = lib.profile(prof)
    sizes = [(64, 64), (32, 128), (64, 64), (128, 32), (4, 4), (64, 64), (64, 64)]
    tiles = [_rand_img(fmt, h, w, seed=200 + i) for i, (h, w) in enumerate(sizes)]
    want = [lib.encode(fmt, t, settings) for t in tiles]
    # pageable host memory
    outs = [np.zeros_like(w) for w in want]
    lib.encode_batch(fmt, [(t.ctypes.data, t.shape[1], t.shape[0], t.strides[0]) for t in tiles], [o.ctypes.data for o in outs], settings)
    assert all(np.array_equal(o, w) for o, w in zip(outs, want))
    # pinned host memory
    pins = [torch.from_numpy(t.copy().reshape(-1)).pin_memory() for t in tiles]
    pouts = [torch.zeros(w.size, dtype=torch.uint8).pin_memory() for w in want]
    lib.encode_batch(fmt, [(p.data_ptr(), t.shape[1], t.shape[0], t.shape[1] * 4) for p, t in zip(pins, tiles)],
                     [o.data_ptr() for o in pouts], settings)
    assert all(np.array_equal(o.numpy(), w) for o, w in zip(pouts, want))
    # device-resident
    devs = [p.cuda() for p in pins]
    douts = [torch.zeros(w.size, dtype=torch.uint8, device="cuda") for w in want]
    lib.encode_batch(fmt, [(d.data_ptr(), t.shape[1], t.shape[0], t.shape[1] * 4) for d, t in zip(devs, tiles)],
                     [o.data_ptr() for o in douts], settings)
    torch.cuda.synchronize()
    assert all(np.array_equal(o.cpu().numpy(), w) for o, w in zip(douts, want))


def test_banded_host_path_equals_device_path_and_oracle():
    """Host surfaces of 256+ rows go through the band pipeline of the compute-bound encoders (copy-in, kernels and
    copy-out on three streams): same bytes as the single-launch device path, and as the oracle on a crop."""
    import torch
    lib, oracle = T.product(), T.oracle()
    for fmt, prof, h, w, pad in (("BC7", "veryfast", 1024, 512, 0), ("BC7", "alpha_veryfast", 260, 64, 16), ("BC6H", "bc6h_veryfast", 516, 256, 8)):
        texel = T.binding.FORMATS[fmt][2]
        img = _rand_img(fmt, h, w, seed=h + w)
        settings = lib.profile(prof)
        d_in = torch.from_numpy(img.copy().view(np.uint8).reshape(-1)).cuda()
        d_out = torch.zeros((h // 4) * (w // 4) * 16, dtype=torch.uint8, device="cuda")
        lib.encode_raw(fmt, d_in.data_ptr(), w, h, w * texel, d_out.data_ptr(), settings)
        want = d_out.cpu().numpy()
        assert np.array_equal(lib.encode(fmt, img, settings), want), (fmt, "tight rows")
        if pad:                                                        # padded host stride
            wide = np.zeros((h, w * texel + pad), np.uint8)
            wide[:, :w * texel] = img.view(np.uint8).reshape(h, w * texel)
            got = np.zeros_like(want)
            lib.encode_raw(fmt, wide.ctypes.data, w, h, wide.strides[0], got.ctypes.data, settings)
            assert np.array_equal(got, want), (fmt, "padded stride")
        crop = np.ascontiguousarray(img[:64, :64])
        rows = want.reshape(h // 4, (w // 4) * 16)[:16, :16 * 16].reshape(-1)
        assert np.array_equal(T.run(oracle, fmt, crop, prof), rows), (fmt, "oracle crop")
    bad = lib.profile("slow")                                          # an error inside the pipeline leaves nothing in flight
    bad.fastSkipTreshold_mode1 = 65
    with pytest.raises(RuntimeError, match="fastSkipTreshold"):
        lib.encode("BC7", np.zeros((512, 64, 4), np.uint8), bad)
    assert np.array_equal(lib.encode("BC7", _rand_img("BC7", 256, 64, seed=1), lib.profile("veryfast")),
                          lib.encode("BC7", _rand_img("BC7", 256, 64, seed=1), lib.profile("veryfast")))


def test_release_frees_and_next_call_recreates():
    """itw_release drops the thread's device buffers / streams; later calls (all three host paths) still give the same bytes."""
    lib = T.product()
    img = _rand_img("BC7", 512, 64, seed=9)
    s = lib.profile("veryfast")
    want = lib.encode("BC7", img, s)                      # banded path
    small = lib.encode("BC1", img[:64])                   # single-launch path
    lib.lib.itw_release.restype = None
    lib.lib.itw_release()
    lib.lib.itw_release()                                 # idempotent
    assert np.array_equal(lib.encode("BC7", img, s), want)
    assert np.array_equal(lib.encode("BC1", img[:64]), small)


def test_baseline_configs_c1_c2_c3_against_the_oracle():
    """SURVEY.md 8d / BASELINE configs.  C1 (BC1, 512^2 gradient): the whole image against the oracle.  C2 / C3 (4096^2 random
    RGBA8 / RGBA16F, the seeded generators of synth.py): full-size encodes through the C-ABI, every 64th block row against the
    oracle (the oracle needs seconds per band at these profiles)."""
    lib, oracle = T.product(), T.oracle()
    c1 = T.synth.gradient_rgba8(512, 512)
    assert c1[0, 511, 0] == 255 and c1[511, 0, 1] == 255 and c1[511, 511, 2] == 255
    assert np.array_equal(lib.encode("BC1", c1), T.run(oracle, "BC1", c1, None))
    c2 = T.synth.random_rgba8(4096, 4096)
    c3 = T.synth.random_rgba16f(4096, 4096)
    for fmt, prof, img in (("BC7", "slow", c2), ("BC7", "alpha_slow", c2), ("BC6H", "bc6h_slow", c3)):
        got = lib.encode(fmt, img, lib.profile(prof)).reshape(1024, 1024 * 16)
        for row in (0, 448, 1023):
            band = np.ascontiguousarray(img[4 * row:4 * row + 4, :512])          # 128 blocks of that block row
            want = T.run(oracle, fmt, band, prof)
            assert np.array_equal(got[row, :128 * 16], want), (fmt, prof, row)
