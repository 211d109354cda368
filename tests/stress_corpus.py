"""A large, deterministic, structured corpus for the BC7 and BC6H encoders: surfaces built block by block, every block drawn
from a family of content that steers the encoder to one particular decision (a mode, a partition shape, a rotation, an index
selection, a degenerate or special-valued block).  Test infrastructure only; numpy only.

Block i of a surface is generated from its own generator, seeded with (seed, i), so any block can be regenerated from its
index alone (`block_rgba8(i, seed)`, `block_rgba16f(i, seed)`) and a mismatch can be traced back to the content that made it.

Surface size: 1024 x 1040 texels = 256 x 260 = 66 560 blocks.  The BC7 kernel runs one 16-warp CTA per SM and gives every
warp 16 blocks per full round, so a wave is SMs x 256 blocks:
  * 132 SMs (H100 SXM): wave 33 792 -> one full round, then 32 768 blocks left over 2 112 warps -> a last round of 16 per warp;
  * 114 SMs (H100 PCIe): wave 29 184 -> two full rounds, then 8 192 blocks over 1 824 warps -> a last round of 8 per warp.
So one launch over the surface runs both full rounds and the dealt last round on every SM."""
import numpy as np

import bcn_decode

HEIGHT, WIDTH = 1040, 1024
BLOCKS_X = WIDTH // 4
SEED_LDR, SEED_HDR = 1, 2

SHAPE2, SHAPE3 = bcn_decode.SHAPE2, bcn_decode.SHAPE3


def subsets2(shape):
    return np.array([(SHAPE2[shape] >> k) & 1 for k in range(16)])


def subsets3(shape):
    return np.array([(SHAPE3[shape] >> (2 * k)) & 3 for k in range(16)])


# ---------------------------------------------------------------------------------------------------------------------------
# LDR (RGBA8) families.  Each returns 16 x 4 integer texels (texel k = row k // 4, column k % 4), clipped to 0..255 by the caller.
# ---------------------------------------------------------------------------------------------------------------------------
NOISE = (0, 1, 4, 16)


def _colours(rng, n, style):
    """n subset colours: random, far apart on a coarse palette (tied shape errors), or on the 5-bit grid of modes 0 / 2."""
    if style == 0:
        return rng.integers(0, 256, (n, 4))
    if style == 1:
        return rng.integers(0, 3, (n, 4)) * 120 + rng.integers(0, 2) * 15
    q = rng.integers(0, 32, (n, 4))
    return (q << 3) | (q >> 2)


def _partitioned(rng, sub, n):
    """Colours laid out on a partition shape: flat subsets or a ramp inside every subset, plus noise of a chosen amplitude."""
    col = _colours(rng, n, int(rng.integers(0, 3)))
    px = col[sub].astype(np.int64)
    if rng.random() < 0.4:                                   # a ramp along a direction inside each subset: 3-bit indices pay
        step = rng.integers(-12, 13, (n, 4))
        t = np.arange(16) % 4 + np.arange(16) // 4
        px += step[sub] * t[:, None]
    amp = NOISE[int(rng.integers(0, 4))]
    if amp:
        px += rng.integers(-amp, amp + 1, (16, 4))
    return px


def _alpha_for_shape(rng, px, sub, n):
    r = rng.random()
    if r < 0.6:
        px[:, 3] = 255
    elif r < 0.85:                                           # alpha per subset (mode 7 on alpha profiles)
        px[:, 3] = rng.integers(0, 256, n)[sub] + rng.integers(-2, 3, 16)
    return px


def fam_shape2(rng):
    shape = int(rng.integers(0, 64))
    sub = subsets2(shape)
    return _alpha_for_shape(rng, _partitioned(rng, sub, 2), sub, 2)


def fam_shape3(rng):
    shape = int(rng.integers(0, 16)) if rng.random() < 0.4 else int(rng.integers(0, 64))     # mode 0 only has shapes 0-15
    sub = subsets3(shape)
    px = _partitioned(rng, sub, 3)
    px[:, 3] = 255
    return px


def fam_tied(rng):
    """Two or three far-apart values per channel spread over a random shape: many shapes tie on error."""
    sub = subsets2(int(rng.integers(0, 64))) if rng.random() < 0.6 else subsets3(int(rng.integers(0, 64)))
    pal = rng.integers(0, 3, (3, 4)) * 120
    px = pal[sub].astype(np.int64)
    px[:, 3] = 255 if rng.random() < 0.7 else px[:, 3]
    return px


def _line(rng):
    """A smooth one-subset block: a ramp between two random colours along a random direction, with small noise."""
    a, b = rng.integers(0, 256, 4), rng.integers(0, 256, 4)
    d = rng.integers(0, 4)
    k = np.arange(16)
    t = [k % 4, k // 4, k % 4 + k // 4, 3 - k % 4 + k // 4][d] / (6.0 if d >= 2 else 3.0)
    px = np.rint(a[None] + (b - a)[None] * t[:, None]).astype(np.int64)
    return px + rng.integers(-2, 3, (16, 4))


def fam_alpha_const(rng):
    px = _line(rng)
    px[:, 3] = 255
    return px


def fam_alpha_independent(rng):
    """Alpha (or, for a rotation, one colour channel) independent of the other three: modes 4 / 5 with every rotation and
    index selection."""
    px = _line(rng)
    ch = int(rng.integers(0, 4))
    lo, hi = sorted(rng.integers(0, 256, 2))
    px[:, ch] = rng.integers(lo, hi + 1, 16) if rng.random() < 0.5 else rng.permutation(np.linspace(lo, hi, 16).astype(np.int64))
    if ch != 3 and rng.random() < 0.5:
        px[:, 3] = 255
    if rng.random() < 0.5:                                   # colours with little variation next to a busy scalar channel
        others = [c for c in range(3) if c != ch]
        px[:, others] = px[0, others] + rng.integers(-1, 2, (16, len(others)))
    return px


def fam_alpha_correlated(rng):
    px = _line(rng)
    c = int(rng.integers(0, 3))
    px[:, 3] = (px[:, c] if rng.random() < 0.5 else 255 - px[:, c]) + rng.integers(-3, 4, 16)
    return px


def fam_alpha_punch(rng):
    px = _line(rng) if rng.random() < 0.5 else rng.integers(0, 256, (16, 4))
    px[:, 3] = np.where(rng.random(16) < 0.5, 0, 255)
    return px


def fam_alpha_single(rng):
    px = _line(rng)
    px[:, 3] = 255
    px[int(rng.integers(0, 16)), 3] = int(rng.integers(0, 255))
    return px


def fam_degenerate(rng):
    kind = int(rng.integers(0, 8))
    k = np.arange(16)
    if kind == 0:                                            # flat
        px = np.tile(rng.integers(0, 256, 4), (16, 1))
    elif kind == 1:                                          # flat subsets inside a partitioned block
        sub = subsets2(int(rng.integers(0, 64))) if rng.random() < 0.5 else subsets3(int(rng.integers(0, 64)))
        px = rng.integers(0, 256, (3, 4))[sub]
    elif kind == 2:                                          # one-texel outlier in a flat block
        px = np.tile(rng.integers(0, 256, 4), (16, 1))
        px[int(rng.integers(0, 16)), : int(rng.integers(1, 5))] = rng.integers(0, 256)
    elif kind == 3:                                          # single-channel ramp
        px = np.tile(rng.integers(0, 256, 4), (16, 1))
        px[:, int(rng.integers(0, 4))] = rng.integers(0, 64) + k * int(rng.integers(1, 13))
    elif kind == 4:                                          # grey ramp
        g = rng.integers(0, 128) + k * int(rng.integers(1, 9))
        px = np.stack([g, g, g, np.full(16, 255)], 1)
    elif kind == 5:                                          # 0 / 255 extremes
        px = rng.integers(0, 2, (16, 4)) * 255
    elif kind == 6:                                          # +-1 around one value
        px = rng.integers(1, 255, 4)[None] + rng.integers(-1, 2, (16, 4))
    else:                                                    # extremes on a shape
        px = (rng.integers(0, 2, (2, 4)) * 255)[subsets2(int(rng.integers(0, 64)))]
    if kind != 4 and rng.random() < 0.5:
        px = px.copy()
        px[:, 3] = 255
    return px


LDR_FAMILIES = ((fam_shape2, 30), (fam_shape3, 30), (fam_tied, 6), (fam_alpha_const, 4), (fam_alpha_independent, 12),
                (fam_alpha_correlated, 4), (fam_alpha_punch, 3), (fam_alpha_single, 3), (fam_degenerate, 8))


# ---------------------------------------------------------------------------------------------------------------------------
# HDR (RGBA16F half bits) families.  Values are worked on as half bit patterns: the BC6H endpoints are quantised from them.
# ---------------------------------------------------------------------------------------------------------------------------
HMAX = 0x7BFF
# two-region modes: endpoint bits and delta bits (r, g, b) -- the largest endpoint spread per channel each one can hold,
# in half-bit units, is about 2^(delta bits - 1) quanta of 0x7C00 / 2^(endpoint bits)
BC6_TWO = ((10, (5, 5, 5)), (7, (6, 6, 6)), (11, (5, 4, 4)), (11, (4, 5, 4)), (11, (4, 4, 5)), (9, (5, 5, 5)), (8, (6, 5, 5)),
           (8, (5, 6, 5)), (8, (5, 5, 6)), (6, (7, 7, 7)))
BC6_ONE = ((10, 10), (11, 9), (12, 8), (16, 4))


def _spread(epb, nb):
    return int(2 ** (nb - 1) * 0x7C00 / 2 ** epb)


def fam_hdr_shape(rng):
    """Two colours on one of the 32 two-region shapes, all four endpoints inside one mode's delta range per channel."""
    sub = subsets2(int(rng.integers(0, 32)))
    epb, nb = BC6_TWO[int(rng.integers(0, 10))]
    span = [int(_spread(epb, b) * rng.uniform(0.3, 0.95)) for b in nb]
    px = np.zeros((16, 4), np.int64)
    for c in range(3):
        base = int(rng.integers(0, HMAX - span[c]))
        cols = base + rng.integers(0, span[c] + 1, 4)
        t = np.arange(16) % 4 / 3.0 if rng.random() < 0.5 else np.zeros(16)
        lo, hi = cols[2 * sub], cols[2 * sub + 1]
        px[:, c] = np.rint(lo + (hi - lo) * t)
    amp = (0, 1, 4, 16)[int(rng.integers(0, 4))]
    px[:, :3] += rng.integers(0, amp + 1, (16, 3))
    px[:, 3] = 0x3C00
    return px


def fam_hdr_one(rng):
    """One smooth region whose span fits one of the one-region modes."""
    epb, nb = BC6_ONE[int(rng.integers(0, 4))]
    px = np.zeros((16, 4), np.int64)
    k = np.arange(16)
    t = (k % 4 + k // 4) / 6.0
    for c in range(3):
        span = int(_spread(epb, nb) * rng.uniform(0.2, 0.95)) if nb < 10 else int(rng.integers(0, HMAX))
        base = int(rng.integers(0, HMAX - span + 1))
        px[:, c] = base + np.rint(span * t)
    px[:, 3] = 0x3C00
    return px


def fam_hdr_span(rng):
    """Narrow and wide spans per channel around a base (as in the small corpus): per-channel delta widths."""
    base = int(rng.integers(0x0400, 0x7000))
    px = base + rng.integers(0, 40, (16, 4))
    for c in range(3):
        if rng.random() < 0.4:
            px[:, c] += rng.integers(0, int(rng.choice([200, 1500, 6000])), 16)
    return px


def fam_hdr_special(rng):
    kind = int(rng.integers(0, 6))
    if kind == 0:                                            # denormal halves
        px = rng.integers(0, 0x0400, (16, 4))
    elif kind == 1:                                          # next to the largest finite half
        px = HMAX - rng.integers(0, 64, (16, 4))
    elif kind == 2:                                          # arbitrary sign-bit patterns
        px = rng.integers(0, 0x10000, (16, 4))
    elif kind == 3:                                          # Inf / NaN bit patterns among ordinary values
        px = rng.integers(0x3000, 0x5000, (16, 4))
        m = rng.random((16, 4)) < 0.3
        px[m] = rng.choice([0x7C00, 0x7C01, 0x7E00, 0x7FFF, 0xFC00, 0xFE00, 0xFFFF], int(m.sum()))
    elif kind == 4:                                          # negative values next to positive ones
        px = rng.integers(0x2000, 0x6000, (16, 4)) | np.where(rng.random((16, 4)) < 0.5, 0x8000, 0)
    else:                                                    # zeros and the largest half
        px = np.where(rng.random((16, 4)) < 0.5, 0, HMAX)
    return px


def fam_hdr_ramp(rng):
    """A smooth exponent ramp: values 2^(a + b t) over the block."""
    k = np.arange(16)
    t = (k % 4 + k // 4) / 6.0
    a, b = rng.uniform(-14, 12), rng.uniform(-6, 6)
    v = np.exp2(np.clip(a + b * t, -24, 15.9))[:, None] * (1 + rng.uniform(0, 1, 4))[None]
    return np.clip(v, 0, 65504).astype(np.float16).view(np.uint16).astype(np.int64)


HDR_FAMILIES = ((fam_hdr_shape, 50), (fam_hdr_one, 14), (fam_hdr_span, 12), (fam_hdr_special, 12), (fam_hdr_ramp, 12))


# ---------------------------------------------------------------------------------------------------------------------------
def _pick(families, rng):
    w = np.array([f[1] for f in families], np.float64)
    return families[int(np.searchsorted(np.cumsum(w) / w.sum(), rng.random(), side="right"))][0]


def block_family(i, seed, hdr=False):
    return _pick(HDR_FAMILIES if hdr else LDR_FAMILIES, np.random.default_rng((seed, i))).__name__


def block_rgba8(i, seed=SEED_LDR):
    """Block i of structured_rgba8(..., seed): 4 x 4 x 4 uint8."""
    rng = np.random.default_rng((seed, i))
    px = _pick(LDR_FAMILIES, rng)(rng)
    return np.clip(px, 0, 255).astype(np.uint8).reshape(4, 4, 4)


def block_rgba16f(i, seed=SEED_HDR):
    """Block i of structured_rgba16f(..., seed): 4 x 4 x 4 uint16 half bit patterns."""
    rng = np.random.default_rng((seed, i))
    px = _pick(HDR_FAMILIES, rng)(rng)
    return np.clip(px, 0, 0xFFFF).astype(np.uint16).reshape(4, 4, 4)


def _surface(h, w, make, seed, dtype):
    assert h % 4 == 0 and w % 4 == 0
    out = np.zeros((h // 4, 4, w // 4, 4, 4), dtype)
    for i in range((h // 4) * (w // 4)):
        out[i // (w // 4), :, i % (w // 4)] = make(i, seed)
    return out.reshape(h, w, 4)


def structured_rgba8(h=HEIGHT, w=WIDTH, seed=SEED_LDR):
    return _surface(h, w, block_rgba8, seed, np.uint8)


def structured_rgba16f(h=HEIGHT, w=WIDTH, seed=SEED_HDR):
    return _surface(h, w, block_rgba16f, seed, np.uint16)
