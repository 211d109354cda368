"""HDR inputs of the BC6H save and preview paths: seeded numpy generators, deterministic, no files read except the committed
real-content crop.  Test infrastructure only.

Every family is built as RGBA16F half bit patterns (H x W x 4 uint16); `planes(bits)` gives the float32 planes of the same
values (half -> float32 is exact), so one family feeds both the RGBA16F entry points and the 32-bit Photoshop-plane ones.  The
boundary family is the exception: most of its values are not halves, so it is built as float planes and its halves are their
conversion.

Two domains, kept apart (DESIGN.md section 2):
  * PINNED: every half a family holds, and every half the save path computes from it, is at most 65504 in magnitude.  There
    the half conversions are the reference's, and the tests compare with the reference's own bodies and their digests.
  * PRODUCT-DEFINED (`product_defined`): +-Inf, NaN, values that convert to exponent-31 halves (65520 and above) and those halves
    themselves.  The product restates DirectXMath 3.06 there (saturation to 0x7FFF, exponent 31 decoded as an ordinary binade
    65536 ... 131008); other DirectXMath generations differ, so these are compared with the oracle only.

The numpy restatements below (`half_from_float`, `float_from_half`, `box_level1`, `linear_level1`, `normalize`) let a CPU test
measure what the corpus reaches: how many stored halves change when the filter sums in another order, and how often each
conversion class occurs."""
import functools
import os

import numpy as np

HALF_MAX = 65504.0
BOX_ORDERS = ("reference", "row_pairs", "column_pairs")        # ((a+c)+b)+d, ((a+b)+c)+d, (a+c)+(b+d)


# ---- DirectXMath 3.06 half conversions (csrc/frontend.cuh) -------------------------------------------------------------
def half_from_float(x):
    """XMConvertFloatToHalf, 3.06 scalar path: RNE on the rebiased pattern, truncating denormal shift, 0x7FFF above 0x47FFEFFF."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.int64)
    sign = (b & 0x80000000) >> 16
    b = b & 0x7FFFFFFF
    shift = 113 - (b >> 23)
    den = np.where((shift > 0) & (shift < 32), (0x800000 | (b & 0x7FFFFF)) >> np.clip(shift, 0, 31), 0)
    v = np.where(b < 0x38800000, den, (b + 0xC8000000) & 0xFFFFFFFF)
    r = ((v + 0x0FFF + ((v >> 13) & 1)) >> 13) & 0x7FFF
    return (np.where(b > 0x47FFEFFF, 0x7FFF, r) | sign).astype(np.uint16)


def half_from_float_ieee(x):
    """IEEE round-to-nearest-even (numpy's float16) with 3.06's saturation: differs from `half_from_float` only on half denormals."""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        h = x.astype(np.float16).view(np.uint16)
    return np.where(np.abs(x) < 2.0 ** -14, h, half_from_float(x)).astype(np.uint16)


def float_from_half(h):
    """XMConvertHalfToFloat, 3.06 scalar path: exact for every half; exponent 31 is an ordinary binade (65536 ... 131008)."""
    h = np.asarray(h, np.uint16).astype(np.uint32)
    e, mant, sign = (h >> 10) & 31, h & 0x3FF, (h & 0x8000) << 16
    normal = (sign | ((e + 112) << 23) | (mant << 13)).astype(np.uint32).view(np.float32)
    den = (mant.astype(np.float32) * np.float32(2.0 ** -24)) * np.where(sign != 0, np.float32(-1), np.float32(1))
    return np.where(e > 0, normal, den).astype(np.float32)


def planes(bits):
    """RGBA16F bits -> the float32 planes of the same values (exact)."""
    return float_from_half(bits)


def halves(vals):
    return half_from_float(np.asarray(vals, np.float32))


# ---- families ----------------------------------------------------------------------------------------------------------
def _log_uniform(rng, shape, lo=-24.0, hi=np.log2(HALF_MAX), neg=0.2):
    mag = np.exp2(rng.uniform(lo, hi, shape)).astype(np.float32)
    mag = np.minimum(mag, np.float32(HALF_MAX))
    return np.where(rng.random(shape) < neg, -mag, mag).astype(np.float32)


def log_uniform(h, w, seed=1):
    """Signed magnitudes log-uniform over 2^-24 ... 65504, 20 % negative, every channel independent."""
    return halves(_log_uniform(np.random.default_rng(seed), (h, w, 4)))


def order_cells(h, w, seed=2):
    """2x2 cells on level 0's grid whose box / linear sum rounds differently in another order.  Per cell and channel one of
    (a = (row 0, col 0), b = (row 0, col 1), c = (row 1, col 0), d = (row 1, col 1)):
      0  a = X, c = -X (+ a few ulps of X), b, d tiny          cancellation inside the reference's first pair
      1  b = Y, d = -Y, a, c tiny                              cancellation inside its second column
      2  a = X, b = -X, c, d tiny                              cancellation along row 0
      3  c = X, d = -X, a, b tiny                              cancellation along row 1
      4  one bright texel, three tiny ones of either sign
      5  a = 2h, c = 2h' (h, h' adjacent halves: (a+c)/4 is a half rounding tie), b = f, d = -f with f near the float ulp
         of a + c, so whether the tie survives depends on the order
    X, Y are halves of 2^10 ... 65504, tiny ones 2^-24 ... 2^-4, signs random."""
    rng = np.random.default_rng(seed)
    ch, cw = (h + 1) // 2, (w + 1) // 2
    shp = (ch, cw, 4)
    kind = rng.integers(0, 6, shp)
    big = np.abs(halves(_log_uniform(rng, shp, 10.0, 15.99, 0.0)).astype(np.int64))
    big = np.minimum(big, 0x7BFF)
    sgn = np.where(rng.random(shp) < 0.5, 0x8000, 0)
    X = big | sgn
    negX = big | (sgn ^ 0x8000)
    delta = np.where(rng.random(shp) < 0.5, 0, rng.integers(1, 4, shp))
    Xd = np.where(big >= delta, (big - delta) | (sgn ^ 0x8000), negX)                       # -X + delta ulps, |.| < |X|
    t = [halves(_log_uniform(rng, shp, -24.0, -4.0, 0.5)).astype(np.int64) for _ in range(3)]
    # kind 5: h, h' adjacent positive halves of 2^-10 ... 2^14; f a half near ulp_f32(2h + 2h')
    hh = np.minimum(np.abs(halves(_log_uniform(rng, shp, -10.0, 14.0, 0.0)).astype(np.int64)), 0x7BFE)
    two_h, two_h1 = halves(2 * float_from_half(hh)), halves(2 * float_from_half(hh + 1))
    s = 2 * float_from_half(hh).astype(np.float64) + 2 * float_from_half(hh + 1)
    ulp = np.exp2(np.floor(np.log2(s)) - 23)
    f = halves((ulp * rng.choice([0.5, 0.75, 1.0, 1.5, 2.5, 3.0], shp)).astype(np.float32)).astype(np.int64)
    fneg = f ^ 0x8000
    pos = rng.integers(0, 4, shp)
    cells = np.zeros((ch, cw, 4, 4), np.int64)                  # last axis: a, b, c, d
    cases = {
        0: (X, t[0], Xd, t[1]), 1: (t[0], X, t[1], negX), 2: (X, negX, t[0], t[1]), 3: (t[0], t[1], X, negX),
        5: (two_h.astype(np.int64), f, two_h1.astype(np.int64), fneg),
    }
    for k, (a, b, c, d) in cases.items():
        m = kind == k
        for i, v in enumerate((a, b, c, d)):
            cells[..., i][m] = np.asarray(v)[m]
    m4 = kind == 4
    for i in range(4):
        cells[..., i][m4] = np.where(pos == i, X, t[i % 3] ^ (0x8000 * (i & 1)))[m4]
    out = np.empty((2 * ch, 2 * cw, 4), np.uint16)
    out[0::2, 0::2], out[0::2, 1::2] = cells[..., 0], cells[..., 1]
    out[1::2, 0::2], out[1::2, 1::2] = cells[..., 2], cells[..., 3]
    return np.ascontiguousarray(out[:h, :w])


def exposure_ramp(h, w, seed=3):
    """Smooth exposure ramps: 2^(a + b x / w + c y / h) over 20+ stops, a different ramp and tint per channel."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    ch = []
    for _ in range(4):
        a, span = rng.uniform(-20, -8), rng.uniform(20, 30)
        fx, fy = rng.uniform(0.3, 1.0), rng.uniform(0.0, 0.7)
        e = a + span * (fx * x / max(w - 1, 1) + fy * y / max(h - 1, 1)) / (fx + fy)
        ch.append(np.exp2(np.clip(e, -24, 15.99)) * rng.uniform(1, 1.9))
    v = np.minimum(np.stack(ch, -1), HALF_MAX).astype(np.float32)
    return halves(v)


def _boundary_pinned():
    """Float values whose half is at most 65504 in magnitude, at the edges of the conversion."""
    f32 = lambda bits: np.array(bits, np.uint32).view(np.float32)
    top = np.arange(65504, 65520, dtype=np.float32)                                  # 65504 ... 65519 -> 0x7BFF
    top = np.concatenate([top, f32([0x477FEFFF, 0x477FF000 - 1, 0x477FE000, 0x477FE001])])   # around the 65504 / 65520 midpoint
    d24 = np.float32(2.0 ** -24)
    tiny = np.array([d24, d24 / 2, d24 / 4, d24 * 1.5, d24 * 0.75, d24 * 2.5, np.nextafter(d24 / 2, np.float32(1)),
                     np.nextafter(d24 / 2, np.float32(0))], np.float32)
    n61 = np.float32(6.1e-5)
    near_min = np.concatenate([[np.nextafter(n61, np.float32(0)), n61, np.nextafter(n61, np.float32(1))],
                               np.float32(2.0 ** -14) + np.array([-1, 0, 1], np.float32) * np.float32(2.0 ** -37)])
    # half-denormal results where the truncating shift meets a tie that IEEE rounding would break upwards: exponent e, shift
    # 113 - e >= 1, the kept bits end in exactly 0x1000 over an even half mantissa, and a lost bit is set
    ties = []
    for e in range(103, 113):
        sh = 113 - e
        for k in range(0, 1024, 37):
            kept = ((2 * k) << 12) | 0x1000                                            # even half mantissa k*2, tie
            full = (kept << sh) | 1
            if full >= 0x800000 and full < 0x1000000:
                ties.append((e << 23) | (full & 0x7FFFFF))
    ties = f32(ties)
    vals = np.concatenate([top, tiny, near_min, ties, [0.0, 1.0, 0.5]]).astype(np.float32)
    return np.concatenate([vals, -vals, [np.float32(-0.0)]]).astype(np.float32)


def boundary_planes(h, w, seed=4):
    """32-bit planes: the pinned boundary values (65504 ... 65519, the 65504 / 65520 midpoint, 2^-24 and its halves, the
    neighbours of 6.1e-5 and of 2^-14, +-0, denormal ties of the truncating shift), shuffled over the surface."""
    rng = np.random.default_rng(seed)
    vals = _boundary_pinned()
    idx = rng.permutation(np.resize(np.arange(vals.size), h * w * 4))
    return vals[idx].reshape(h, w, 4)


def boundary(h, w, seed=4):
    return halves(boundary_planes(h, w, seed))


@functools.lru_cache(None)
def _reciprocal_sensitive(count=256, seed=55):
    """Half RGB vectors whose normalised halves change when x * (1 / m) is computed as x / m: a component lands within a float
    ulp of a half rounding tie.  Found by search over a fixed seeded stream (about 1 vector in 1 500 qualifies)."""
    rng = np.random.default_rng(seed)
    found, n = [], 0
    while n < count:
        v = rng.uniform(-2, 2, (1 << 17, 4)) * np.exp2(rng.uniform(-6, 6, (1 << 17, 1)))
        bits = halves(v.astype(np.float32))
        hit = bits[(normalize(bits) != normalize(bits, reciprocal=False))[:, :3].any(1)]
        found.append(hit)
        n += hit.shape[0]
    return np.concatenate(found)[:count, :3]


def normal_vectors(h, w, seed=5):
    """Normal-map RGB (alpha random): zero (+-0), near-zero (half denormals), huge (1e4 ... 65504), single-axis of every magnitude,
    random vectors in [-2, 2]^3, and vectors whose normalisation depends on multiplying by the reciprocal (`_reciprocal_sensitive`)."""
    rng = np.random.default_rng(seed)
    n = h * w
    kind = rng.integers(0, 6, n)
    pool = float_from_half(_reciprocal_sensitive())
    v = rng.uniform(-2, 2, (n, 3)).astype(np.float32)
    sz = (rng.random((n, 3)) < 0.5)
    v[kind == 0] = np.where(sz, np.float32(-0.0), np.float32(0.0))[kind == 0]
    v[kind == 1] = _log_uniform(rng, (n, 3), -24.0, -14.0, 0.5)[kind == 1]
    v[kind == 2] = _log_uniform(rng, (n, 3), 13.3, 15.99, 0.5)[kind == 2]
    axis = rng.integers(0, 3, n)
    single = np.zeros((n, 3), np.float32)
    single[np.arange(n), axis] = _log_uniform(rng, n, -24.0, 15.99, 0.5)
    v[kind == 3] = single[kind == 3]
    v[kind == 5] = pool[rng.integers(0, pool.shape[0], int((kind == 5).sum()))]
    rgba = np.concatenate([v, rng.uniform(0, 1, (n, 1)).astype(np.float32)], 1)
    return halves(rgba.reshape(h, w, 4))


def real_hdr(h=128, w=128):
    """The committed HDR crop (tests/golden/real_content_texels.npz, HDR.hdr: RGBA16F), tiled to h x w."""
    crop = np.load(os.path.join(os.path.dirname(__file__), "golden", "real_content_texels.npz"))["HDR.hdr"]
    reps = (-(-h // crop.shape[0]), -(-w // crop.shape[1]), 1)
    return np.ascontiguousarray(np.tile(crop, reps)[:h, :w])


FAMILIES = {"log_uniform": log_uniform, "order_cells": order_cells, "exposure_ramp": exposure_ramp, "boundary": boundary,
            "normal_vectors": normal_vectors, "real_hdr": lambda h, w, seed=0: real_hdr(h, w)}


def family(name, h, w, seed=0):
    """RGBA16F bits of family `name` at h x w (seeded from the size so every shape has its own draw)."""
    if name == "real_hdr":
        return real_hdr(h, w)
    return FAMILIES[name](h, w, seed=1000 * seed + 7 * h + w)


def family_planes(name, h, w, seed=0):
    """The same family as float32 planes (the boundary family's own floats, not their halves)."""
    if name == "boundary":
        return boundary_planes(h, w, seed=1000 * seed + 7 * h + w)
    return planes(family(name, h, w, seed))


# ---- the product-defined set (section B only) ----------------------------------------------------------------------------
PRODUCT_VALUES = np.concatenate([
    np.array([np.inf, -np.inf, np.nan, -np.nan, 1e9, -1e9, 70000.0, -70000.0, 131008.0, 131040.0, 65520.0, -65520.0, 1e30, 3.4e38],
             np.float32),
    np.array([0x47FFEFFF, 0x47FFEFFE, 0x47FFF000, 0x47FFF001, 0x477FF000, 0x477FF001, 0x7F800001, 0xFFC00000], np.uint32).view(np.float32)])


def product_defined_planes(h, w, seed=6):
    """32-bit planes: a third of the texels from PRODUCT_VALUES, the rest log-uniform halves (so filters mix both)."""
    rng = np.random.default_rng(seed)
    v = planes(log_uniform(h, w, seed)).copy()
    pick = rng.random((h, w, 4)) < 0.34
    v[pick] = rng.choice(PRODUCT_VALUES, int(pick.sum()))
    return v


def product_defined(h, w, seed=6):
    """RGBA16F bits: exponent-31 halves (0x7C00 ... 0x7FFF, both signs) mixed into log-uniform halves, plus the 3.06 conversion
    of PRODUCT_VALUES."""
    rng = np.random.default_rng(seed + 1)
    bits = halves(product_defined_planes(h, w, seed))
    pick = rng.random((h, w, 4)) < 0.2
    bits[pick] = (rng.integers(0x7C00, 0x8000, int(pick.sum())) | (rng.integers(0, 2, int(pick.sum())) << 15)).astype(np.uint16)
    return bits


# ---- numpy restatements of one filter step and of the normal-map pass (for the corpus' own power test) --------------------
def box_level1(bits, order="reference"):
    """Level 1 of a power-of-two RGBA16F level 0 (both sizes >= 2): AVERAGE4 in the reference's order or a reordering."""
    v = float_from_half(bits)
    a, b, c, d = v[0::2, 0::2], v[0::2, 1::2], v[1::2, 0::2], v[1::2, 1::2]
    s = {"reference": lambda: ((a + c) + b) + d, "row_pairs": lambda: ((a + b) + c) + d, "column_pairs": lambda: (a + c) + (b + d)}[order]()
    return half_from_float(s * np.float32(0.25))


def linear_taps(source, dest):
    """_CreateLinearFilter in float32 (Filters.h, clamp addressing): (u0, u1, w0, w1) arrays."""
    u = np.arange(dest, dtype=np.float32)
    scale = np.float32(source) / np.float32(dest)
    srcB = (u + np.float32(0.5)) * scale + np.float32(0.5)
    iB = srcB.astype(np.int64)
    iA = np.maximum(iB - 1, 0)
    iB = np.minimum(iB, source - 1)
    w0 = np.float32(1.0) + iB.astype(np.float32) - srcB
    return iA, iB, w0.astype(np.float32), (np.float32(1.0) - w0).astype(np.float32)


def linear_level1(bits, order="reference"):
    """Level 1 of a non-power-of-two RGBA16F level 0: BILINEAR_INTERPOLATE in the reference's association (rows first) or
    columns first."""
    h, w = bits.shape[:2]
    v = float_from_half(bits)
    xa, xb, xw0, xw1 = linear_taps(w, max(w >> 1, 1))
    ya, yb, yw0, yw1 = linear_taps(h, max(h >> 1, 1))
    a, b = v[ya][:, xa], v[ya][:, xb]
    c, d = v[yb][:, xa], v[yb][:, xb]
    X0, X1 = xw0[None, :, None], xw1[None, :, None]
    Y0, Y1 = yw0[:, None, None], yw1[:, None, None]
    if order == "reference":
        s = (Y0 * (a * X0 + b * X1)) + (Y1 * (c * X0 + d * X1))
    else:
        s = (X0 * (a * Y0 + c * Y1)) + (X1 * (b * Y0 + d * Y1))
    return half_from_float(s.astype(np.float32))


def normalize(bits, reciprocal=True):
    """NormalizeNormalMapChain on RGB halves: x * (1 / m) as the reference does, or x / m."""
    r, g, b = (float_from_half(bits[..., i]) for i in range(3))
    m = np.sqrt((r * r + g * g) + b * b)
    out = bits.copy()
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.float32(1.0) / m
        for i, x in enumerate((r, g, b)):
            out[..., i] = np.where(m > 0, half_from_float(x * inv if reciprocal else x / m), (0, 0, 0x3C00)[i])
    return out


# ---- the cases of tests/golden/hdr_digests.json (written by tests/golden/make_golden_hdr.py) ------------------------------
EXTRA_CHAIN_SHAPES = [(256, 256), (129, 255), (8, 512), (512, 8), (1, 256), (256, 1)]     # (h, w), next to test_mips_f16.SIZES
CONVERT_SHAPE = (21, 37)                                                                  # (h, w): padded along both axes
# (family, h, w) of the chains whose padded levels are encoded under every BC6H preset
BC6H_CHAINS = [("log_uniform", 64, 64), ("order_cells", 36, 60), ("boundary", 32, 32), ("normal_vectors", 12, 20),
               ("exposure_ramp", 16, 64), ("real_hdr", 128, 128)]


def sixteen_bit_planes(planes, seed=9):
    """256 x 256 x planes 16-bit planes, each plane a permutation of every value 0 ... 65535 (65535 / 32768 reaches 2.0)."""
    rng = np.random.default_rng(seed + planes)
    return np.stack([rng.permutation(65536).astype(np.uint16) for _ in range(planes)], -1).reshape(256, 256, planes)


def key(*parts):
    return ":".join(str(p) for p in parts)


def sha(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
