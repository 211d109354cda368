// bc7_pair_check.cpp -- TEST-ONLY: the routines of bc7.cuh that work on two subsets or two masks at once, against the
// per-subset routines they replace.  Compiled for the CPU like tests/emu/emu.cpp.
//
// pair_fit_check: for every two-subset shape of every given block
//   * bc7_fit_pair(mask0, 3 or 4 channels) equals bc7_fit of subset 0 and of subset 1, bit for bit;
//   * at three channels its bounds equal the split bounds of the two subsets (split_bound below), and the key formed from
//     them equals bc7_split_key;
//   * bc7_pair_error of the mode-1 / mode-3 endpoints equals bc7_assign's error of the same shape (three bits, and the
//     two-bit threshold form the shape phases use).
// mask3_pair_check: for every lane pair (masks 2i, 2i + 1 of itw_masks3.cuh) of every given block
//   * bc7_fit_masks2 equals bc7_fit(blk, 3, 1, mask, 3) of each mask, bit for bit;
//   * bc7_masks_error2 of the mode-2 endpoints (and of the mode-0 endpoints, as a second set of inputs) equals the error of
//     each mask alone, as subset_error below computes it.
// Both return the number of mismatches and describe the first one in `what`.
#include <cmath>
#include <cstdio>
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/bc7.cuh"

using namespace itw;

static Bc7Block block_of(const u32* tex)
{
    Bc7Block b;
    memset(&b, 0, sizeof(b));
    for (int k = 0; k < 16; k++) {
        b.tex[k] = tex[k];
        b.rgb[k] = tex[k] & 0x00FFFFFFu;
    }
    for (int c = 0; c < 4; c++)
        for (int i = 0; i < 4; i++) {
            u32 v = 0;
            for (int j = 0; j < 4; j++) v |= ((tex[4 * i + j] >> (8 * c)) & 255u) << (8 * j);
            b.plane[c][i] = v;
        }
    return b;
}

static u32 bits_of(float f)
{
    u32 u;
    memcpy(&u, &f, 4);
    return u;
}

// Split bound of one subset at three channels, written out on its own (K:907-939) so that it does not share the product's
// PCA-line code: the covariance scaled by 1/256^2 with eps on three diagonal slots, four power iterations from (1, 1, 1)
// renormalised every other one, then trace - lambda_max.
static float split_bound(const Bc7Block* blk, u32 mask)
{
    u32 P[4][4];
    load_planes(P, View{blk, 3, 1});
    int st[15];
    moments_u8(st, P, mask, 3);
    float m[10], mean[4];
    bc7_covariance<3>(m, mean, st);
    for (int i = 0; i < 10; i++) m[i] *= 1.0f / (256.0f * 256.0f);
    const float eps = 0.001f * 0.001f;
    m[0] += eps; m[4] += eps; m[7] += eps;
    float v0 = 1.0f, v1 = 1.0f, v2 = 1.0f;
    for (int it = 0; it < 4; it++) {
        const float a0 = m[0] * v0 + m[1] * v1 + m[2] * v2;
        const float a1 = m[1] * v0 + m[4] * v1 + m[5] * v2;
        const float a2 = m[2] * v0 + m[5] * v1 + m[7] * v2;
        v0 = a0; v1 = a1; v2 = a2;
        if (it & 1) {
            float n2 = a0 * a0;
            n2 += a1 * a1;
            n2 += a2 * a2;
            const float rn = 1.0f / sqrtf(n2);
            v0 *= rn; v1 *= rn; v2 *= rn;
        }
    }
    const float mv0 = m[0] * v0 + m[1] * v1 + m[2] * v2;
    const float mv1 = m[1] * v0 + m[4] * v1 + m[5] * v2;
    const float mv2 = m[2] * v0 + m[5] * v1 + m[7] * v2;
    float sum = 0.0f;
    sum += mv0 * mv0;
    sum += mv1 * mv1;
    sum += mv2 * mv2;
    float bound = m[0] + m[4] + m[7];
    bound -= sqrtf(sum);
    return bound > 0.0f ? bound : 0.0f;
}

// The single-mask mode-2 error the shape phases used before the pair walk: one counted loop over the mask's set bits.
static int subset_error(const Bc7Block* blk, u32 mask, u32 dec_a, u32 dec_b)
{
    const Bc7Sub2 s = bc7_sub2(dec_a, dec_b);
    const int n = popcount16(mask);
    int total = 0;
    u32 rest = mask;
    for (int i = 0; i < n; i++) {
        const u32 low = rest & (0u - rest);
        rest ^= low;
        total += bc7_texel_error2(s, blk->rgb[popcount32(low - 1u)]);
    }
    return total;
}

extern "C" int pair_fit_check(const u32* texels, int nblocks, char* what, int what_len)
{
    static u32 pal[40][32];
    int bad = 0;
    auto fail = [&](int blk, int shape, int ch, const char* item) {
        if (bad++ == 0) snprintf(what, what_len, "block %d shape %d channels %d: %s", blk, shape, ch, item);
    };
    for (int n = 0; n < nblocks; n++) {
        const Bc7Block b = block_of(texels + 16 * n);
        for (int shape = 0; shape < 64; shape++) {
            const u32 m0 = (u32)shape_mask(shape, 0), m1 = (u32)shape_mask(shape, 1);
            if (m1 != (~m0 & 0xFFFFu)) fail(n, shape, 0, "subset 1 is not the complement of subset 0");
            for (int ch = 3; ch <= 4; ch++) {
                const Bc7Pair f = bc7_fit_pair(&b, m0, ch);
                for (int j = 0; j < 2; j++) {
                    const Bc7Seg s = bc7_fit(&b, 3, 1, j ? m1 : m0, ch);
                    for (int i = 0; i < 8; i++)
                        if (bits_of(s.v[i]) != bits_of(f.seg[j].v[i])) fail(n, shape, ch, j ? "endpoints of subset 1" : "endpoints of subset 0");
                }
                if (ch == 4) continue;
                if (bits_of(f.bound[0]) != bits_of(split_bound(&b, m0))) fail(n, shape, ch, "split bound of subset 0");
                if (bits_of(f.bound[1]) != bits_of(split_bound(&b, m1))) fail(n, shape, ch, "split bound of subset 1");
                if (bc7_key_of(shape, f.bound[0], f.bound[1]) != bc7_split_key(&b, shape, 3)) fail(n, shape, ch, "ranking key");
                u32 e1[4], e3[4];
                for (int j = 0; j < 2; j++) {
                    const Bc7Packed p1 = bc7_quantise(f.seg[j], 1, 3), p3 = bc7_quantise(f.seg[j], 3, 3);
                    e1[2 * j] = p1.dec_a; e1[2 * j + 1] = p1.dec_b;
                    e3[2 * j] = p3.dec_a; e3[2 * j + 1] = p3.dec_b;
                }
                const Bc7PairErr e = bc7_pair_error(&b, m0, e1[0], e1[1], e1[2], e1[3], e3[0], e3[1], e3[2], e3[3]);
                const u32 pattern = shape_pattern(shape);
                const int want1 = bc7_assign(pal, 0, &b, 3, 1, 3, 2, pattern, e1[0], e1[1], e1[2], e1[3], 0u, 0u, 0x00FFFFFFu).err;
                const int want3 = bc7_assign(pal, 0, &b, 3, 1, 2 | kAssignThresholds, 2, pattern, e3[0], e3[1], e3[2], e3[3], 0u, 0u,
                                             0x00FFFFFFu).err;
                if (e.mode1 != want1) fail(n, shape, ch, "mode-1 error");
                if (e.mode3 != want3) fail(n, shape, ch, "mode-3 error");
            }
        }
    }
    return bad;
}

extern "C" int mask3_pair_count() { return ITW_MASK3_COUNT / 2; }

extern "C" int mask3_pair_check(const u32* texels, int nblocks, char* what, int what_len)
{
    int bad = 0;
    auto fail = [&](int blk, int pair, const char* item) {
        if (bad++ == 0) snprintf(what, what_len, "block %d lane pair %d: %s", blk, pair, item);
    };
    for (int n = 0; n < nblocks; n++) {
        const Bc7Block b = block_of(texels + 16 * n);
        for (int i = 0; i < ITW_MASK3_COUNT / 2; i++) {
            const u32 m[2] = {(u32)ITW_TABLE(mask3_unique)[2 * i], (u32)ITW_TABLE(mask3_unique)[2 * i + 1]};
            const Bc7Segs2 f = bc7_fit_masks2(&b, m[0], m[1]);
            for (int j = 0; j < 2; j++) {
                const Bc7Seg s = bc7_fit(&b, 3, 1, m[j], 3);
                for (int c = 0; c < 8; c++)
                    if (bits_of(s.v[c]) != bits_of(f.seg[j].v[c])) fail(n, i, j ? "endpoints of mask b" : "endpoints of mask a");
            }
            for (int mode = 0; mode <= 2; mode += 2) {
                const Bc7Packed pa = bc7_quantise(f.seg[0], mode, 3), pb = bc7_quantise(f.seg[1], mode, 3);
                const Bc7Err2 e = bc7_masks_error2(&b, m[0], m[1], pa.dec_a, pa.dec_b, pb.dec_a, pb.dec_b);
                if (e.a != subset_error(&b, m[0], pa.dec_a, pa.dec_b)) fail(n, i, "error of mask a");
                if (e.b != subset_error(&b, m[1], pb.dec_a, pb.dec_b)) fail(n, i, "error of mask b");
            }
        }
    }
    return bad;
}
