"""The structured stress corpus (tests/stress_corpus.py, 66 560 blocks per surface) through the CUDA kernels, against the
reference build's recorded digests (tests/golden/stress_digests.json):
  * every case (all BC7 and BC6H presets and the non-preset settings) through the host C ABI, chunk by chunk;
  * four profiles from device memory in one launch -- the multi-round schedule with its dealt last round, not the band
    pipeline of host surfaces -- from a 16-byte aligned source (TMA-staged kernel) and from a source 4 bytes off (plain loads);
  * the real-content crops of tests/golden/real_content_texels.npz for every case of test_real_content.py.
No oracle runs unless a chunk differs; then the oracle encodes the first bad chunk and the message names the first differing
block, the (mode, partition) the reference gives it and where it falls in the launch schedule on this device."""
import hashlib

import numpy as np
import pytest

import itw_testlib as T
import test_real_content as R
import test_stress_corpus as C

pytestmark = pytest.mark.gpu

BC7_WARPS_PER_CTA, BC7_FULL_PER_WARP = 16, 16


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def schedule_position(fmt, block, nblocks):
    """Where block `block` of a one-launch encode of `nblocks` blocks falls in the BC7 kernel's schedule (bc7.cuh: full rounds
    of 16 blocks per warp on every warp, then one last round of 1, 2, 4, 8 or 16 per warp over all warps)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if fmt != "BC7":
        return f"{sms} SMs"
    warps = min(sms, -(-nblocks // BC7_WARPS_PER_CTA)) * BC7_WARPS_PER_CTA
    wave = warps * BC7_FULL_PER_WARP
    nfull, rem = divmod(nblocks, wave)
    if block < nfull * wave:
        return f"full round {block // wave} of {nfull} ({sms} SMs)"
    p = 1
    while p < BC7_FULL_PER_WARP and -(-rem // p) > warps:
        p *= 2
    return f"last round {nfull}, {p} blocks per warp, warp {(block - nfull * wave) // p} ({sms} SMs)"


def explain(case, got, where):
    """The first chunk whose digest differs, re-encoded by the oracle: the first differing block and what it should be."""
    fmt = C.CASES[case][0]
    want = C.GOLDEN["cases"][case]["chunks"]
    n = C.nchunks(fmt)
    bpb = T.binding.FORMATS[fmt][1]
    row = (C.surface(fmt).shape[1] // 4) * bpb
    bad = [j for j in range(n) if sha(got[j * C.ROWS * row:(j + 1) * C.ROWS * row]) != want[j]]
    if not bad:
        return None
    j = bad[0]
    ref = C.encode_chunks(T.oracle(), case, [j])[j].reshape(-1, bpb)
    mine = got[j * C.ROWS * row:(j + 1) * C.ROWS * row].reshape(-1, bpb)
    k = int(np.flatnonzero((ref != mine).any(1))[0]) if (ref != mine).any() else -1
    if k < 0:
        return f"{case} ({where}): chunks {bad} differ from the reference digests, but chunk {j} equals the oracle"
    block = j * C.ROWS * (row // bpb) + k
    hdr = C.bc7_header(ref[k])[:2] if fmt == "BC7" else C.bc6h_header(ref[k])
    nblocks = C.surface(fmt).size // 64
    return (f"{case} ({where}): {len(bad)} of {n} chunks differ, first at chunk {j}; first differing block {block} "
            f"(family {C.S.block_family(block, C.S.SEED_HDR if fmt == 'BC6H' else C.S.SEED_LDR, fmt == 'BC6H')}), "
            f"reference (mode, partition) = {hdr}, got {(C.bc7_header(mine[k])[:2] if fmt == 'BC7' else C.bc6h_header(mine[k]))}; "
            f"{schedule_position(fmt, block, nblocks)}")


@pytest.mark.parametrize("case", list(C.CASES))
def test_host_path_equals_the_reference(case):
    lib = T.product()
    fmt = C.CASES[case][0]
    img = C.surface(fmt)
    got = lib.encode(fmt, img, C.G.settings(lib, case))
    msg = explain(case, got, "host path")
    assert msg is None, msg
    assert sha(got) == C.GOLDEN["cases"][case]["sha256"]


@pytest.mark.parametrize("case", ["slow", "alpha_slow", "basic", "bc6h_slow"])
def test_device_source_one_launch_aligned_and_offset(case):
    import torch
    lib = T.product()
    fmt = C.CASES[case][0]
    img = C.surface(fmt)
    h, w = img.shape[:2]
    texel = T.binding.FORMATS[fmt][2]
    raw = np.ascontiguousarray(img).view(np.uint8).reshape(-1)
    buf = torch.zeros(raw.size + 16, dtype=torch.uint8, device="cuda")
    out = torch.zeros(C.GOLDEN["cases"][case]["bytes"], dtype=torch.uint8, device="cuda")
    settings = C.G.settings(lib, case)
    before = lib.launch_count()
    for off, where in ((0, "device source, 16-byte aligned: TMA-staged kernel"), (4, "device source, 4 bytes off: plain-load kernel")):
        src = buf[off:off + raw.size]
        assert (src.data_ptr() % 16 == 0) == (off == 0)
        src.copy_(torch.from_numpy(raw))
        out.zero_()
        lib.encode_raw(fmt, src.data_ptr(), w, h, w * texel, out.data_ptr(), settings)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        msg = explain(case, got, where)
        assert msg is None, msg
        assert sha(got) == C.GOLDEN["cases"][case]["sha256"], where
    assert lib.launch_count() - before == 2, "each encode is one launch"


def test_real_content_crops_equal_the_reference():
    lib = T.product()
    images, digests = R.stored()
    for name, _ in R.LDR:
        for fmt, prof in R.LDR_CASES:
            assert sha(T.run(lib, fmt, images[name], prof)) == digests[R.key(name, fmt, prof)], (name, fmt, prof)
    for fmt, prof in R.HDR_CASES:
        assert sha(T.run(lib, fmt, images[R.HDR[0]], prof)) == digests[R.key(R.HDR[0], fmt, prof)], (R.HDR[0], fmt, prof)
