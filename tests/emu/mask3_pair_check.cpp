// mask3_pair_check.cpp -- TEST-ONLY: the two-mask routines of the three-subset shape phases of bc7.cuh against the
// per-mask routines they replace.
//
// For every lane pair (masks 2i, 2i + 1 of itw_masks3.cuh) of every given block, compiled for the CPU like tests/emu/emu.cpp:
//   * bc7_fit_masks2 equals bc7_fit(blk, 3, 1, mask, 3) of each mask, bit for bit;
//   * bc7_masks_error2 of the mode-2 endpoints (and of the mode-0 endpoints, as a second set of inputs) equals the error of
//     each mask alone, as the single-mask routine below computes it.
// Returns the number of mismatches and describes the first one in `what`.
#include <cstdio>
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/bc7.cuh"

using namespace itw;

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
