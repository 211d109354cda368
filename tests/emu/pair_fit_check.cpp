// pair_fit_check.cpp -- TEST-ONLY: the two-subset pair routines of bc7.cuh against the per-subset routines they replace.
//
// For every two-subset shape of every given block, compiled for the CPU like tests/emu/emu.cpp:
//   * bc7_fit_pair(mask0, 3 or 4 channels) equals bc7_fit of subset 0 and of subset 1, bit for bit;
//   * at three channels its bounds equal the split bounds of the two subsets (what bc7_split_key computes), and the key
//     formed from them equals bc7_split_key;
//   * bc7_pair_error of the mode-1 / mode-3 endpoints equals bc7_assign's error of the same shape (three bits, and the
//     two-bit threshold form the shape phases use).
// Returns the number of mismatches and describes the first one in `what`.
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

// split bound of one subset, as bc7_split_key_impl<3> computes it
static float split_bound(const Bc7Block* blk, u32 mask)
{
    u32 P[4][4];
    load_planes(P, View{blk, 3, 1});
    int st[15];
    moments_u8(st, P, mask, 3);
    float cov[10], mean[4];
    bc7_covariance<3>(cov, mean, st);
    return bc7_residual_bound<3>(cov);
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
