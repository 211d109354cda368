// bc7.cuh -- BC7 encoder (reference: kernel.ispc:616-2037, cited as K:line).
//
// Mapping.  One WARP owns kBc7Super = 16 consecutive 4x4 blocks per full round (the last round of a launch deals what is left
// over every warp of the grid, 1 to 16 blocks each; bc7_kernel).  The shape / ranking phases hold one HALF of eight blocks at
// a time, as two GROUPS of kBc7Slots = 4 that reuse the per-group scratch; the chain phase -- 14 to 18 roles per block in 8 to
// 10 units, a third of the work -- runs ONCE for all sixteen blocks, two lanes per block, so that a pass is two equally long
// units wide (DESIGN.md section 4 has the numbers).
// The 32 lanes are spread over the blocks' independent work items instead of over texels:
//   * shape phases: a shape's error is the sum of its subsets' errors, and a subset's fit, endpoints and error depend on its
//     texel mask alone (the reference refits per shape and mode, K:1279-1297, with identical results).  So the three-subset
//     shapes go lane <-> (block, two distinct masks) over the four blocks of a group: one routine fits both masks
//     (bc7_fit_masks2: two moment passes, two independent PCA lines, one projection loop), quantises them for modes 0
//     and 2, and one walk over both masks' texels searches them for mode 2; then lane <-> (block, shape) adds three stored
//     mode-2 errors and searches mode 0 from the stored endpoints.  A two-subset shape
//     (modes 1, 3, 7) belongs to one lane.  When the profile searches all 64 of them for modes 1 / 3, lane <-> (block, shape)
//     over the four blocks of a group, shapes in popcount order: one routine fits both subsets (bc7_fit_pair: subset 1's
//     moments are the block's minus subset 0's, two independent PCA lines, one projection loop) and gives the split keys,
//     and one walk over each subset's texels scores modes 1 and 3.  For shorter lists and for mode 7 a lane evaluates
//     one ranked shape: it fits each subset and searches the shape for both modes of the pair (the pair fit measured slower
//     there: it raises the register pressure of bc7_eval_shape);
//   * ranking phase: lane <-> (block slot, two-subset shape) for the 64 PCA split bounds, only where a list of 0 < t < 64
//     shapes needs it to choose its members;
//   * winner phases: lane <-> (block slot, list, strip of 16 entries), then lane <-> (block slot, list);
//   * chain phase: lane <-> (block slot, unit of roles).  The per-mode refinement chains, the mode 4/5
//     rotation / index-swap candidates and mode 6 are independent of one another in the reference
//     (they only meet in a strict `<` on the final error, K:1358, :1638, :1650, :1684), so they
//     all run side by side in units: a partitioned mode, the mode 4/5 roles of one rotation (one fit, one texel walk for
//     the three searches, the three refinements interleaved), mode 6; the block's winner is the first minimum in the
//     reference's order: mode 0, 2, 1, 3, 7, 4(rotation, swap), 5(rotation), 6.
//
// Exactness.  BC7 texels are 8-bit integers, so most of the reference's float arithmetic is exact
// integer arithmetic in disguise.  Wherever every intermediate is an integer below 2^24 the kernel
// uses packed-byte integer instructions instead -- same values, ~6x fewer instructions:
//   * raw moments of a subset (K:763-803): IDP.4A dot products over channel-planar packed bytes;
//   * index search (K:1133-1193): the projection numerator / denominator are integer dot
//     products (then ONE float division, evaluated as the FMA-corrected quotient that equals the
//     IEEE one -- tests/test_exact_division.py, tests/test_gpu_division.py; the two-bit search of the shape phases by two
//     integer thresholds instead), the two candidate palette entries are integer interpolations (the reference truncates
//     them through int, K:1172-1173) and their squared errors are VABSDIFF4 + IDP.4A;
//   * least-squares sums (K:1198-1230): IDP.4A over index bytes.
// Everything that rounds (covariance, power iteration, endpoint solve, quantisation) follows the
// reference's float expression order exactly (DESIGN.md "Canonical float model").  Every fit goes through one PCA-line
// routine (bc7_line, bc7_project, bc7_ends) and every index search through one texel step (bc7_num, bc7_q1_quotient /
// bc7_steps, bc7_pick), so the variants cannot round differently.
//
// Structure for speed (DESIGN.md section 4): the non-inlined routines exchange their results BY VALUE (small structs stay
// in registers across calls; arrays passed by pointer would live in local memory), the inner routines are branch-free
// (rotation views via PRMT selectors, the fourth component via zero operands), and chain tasks are scheduled role-major.
//
// The phases are per-lane functions separated by barriers; tests/emu drives the same
// functions lane by lane on the CPU (test-only).
#pragma once
#include "bc67_core.cuh"
#include "itw_masks3.cuh"
#include "itw_order2.cuh"

// unroll factors of the two hottest loops; on H100 (tools/tune_unroll.sh) BC7 slow / basic take 33.65 / 13.51 ms at
// 16 / 8 against 34.28 / 13.59 (assign 8), 34.81 / 13.85 (assign 4), 33.95 / 13.64 (power 4), 33.90 / 13.60 (power 2)
#ifndef ITW_BC7_ASSIGN_UNROLL
#define ITW_BC7_ASSIGN_UNROLL 16
#endif
#ifndef ITW_BC7_POWER_UNROLL
#define ITW_BC7_POWER_UNROLL 8
#endif

namespace itw {

// distinct subset masks of the three-subset shapes and the mask ids of each shape (tools/gen_mask_tables.py)
ITW_TABLE_DECL(uint16_t, mask3_unique, ITW_MASK3_COUNT)
ITW_TABLE_DECL(uint8_t, shape3_mask_id, 64 * 3)
// the two-subset shapes in ascending popcount of subset 0 (tools/gen_mask_tables.py)
ITW_TABLE_DECL(uint8_t, shape2_order, 64)

// bc7_enc_settings (ispc_texcomp.h:27-41) flattened to ints for the device
struct Bc7Params {
    int sel[4];
    int refine[8];
    int skip2, t1, t3, t7, ch0, rch, channels;
};

constexpr int kBc7Slots = 4;          // blocks per group (ranking / shape phases share per-group scratch)
constexpr int kBc7Batch = 8;          // blocks per HALF: what the shape phases hold in Bc7Warp::blk at a time (two groups)
constexpr int kBc7Super = 16;         // blocks per warp in a full round: two halves, ONE chain phase
constexpr int kBc7MaxRoles = 18;      // 5 partitioned modes + up to 8 mode-4 + 4 mode-5 + mode 6
constexpr int kBc7Strips = 4;         // a candidate list of up to 64 entries is reduced in four strips of 16
constexpr int kErrNone = 0x7fffffff;  // "no result": loses every strict < comparison

// One 4x4 block in shared memory
struct Bc7Block {
    u32 tex[16];       // packed RGBA8 of texel k (R in byte 0)
    u32 plane[4][4];   // plane[c][i] = channel c of texels 4i..4i+3, one byte each
    u32 rgb[16];       // tex[k] & 0x00FFFFFF: what the three-channel index searches read (three quarters of all searches)
    u32 pad;           // 49 words: word k of the eight blocks of a half lands in eight different banks (in the chain phase
                       // adjacent lanes hold different blocks; with 32 words every block read was a bank conflict)
};
// Per-warp scratch in shared memory
struct Bc7Warp {
    Bc7Block blk[kBc7Batch];                   // the half the shape phases are working on
    union {
        // per-GROUP scratch (slot = block index inside the group), reused by every group in turn
        int cand_err[kBc7Slots][2][64];        // errors of the mode-slot pair being evaluated: [first/second][list position,
                                               // or shape id on the full two-subset path (bc7_full_two)]
        // end of the chain phase -> store phase (the shape phases are over by then)
        struct {
            int err[32], role[32];             // best (error, role) of the roles a lane ran for ITS block ...
            u32 code[32][4];                   // ... and the 128 bits of that candidate
        } fin;
    };
    uint8_t order[kBc7Slots][2][64];           // shapes in ascending key order: [0] RGB (modes 1,3), [1] profile channels (mode 7)
    int win_shape[kBc7Super][5];               // winning shape id per block of the round and mode slot, -1 = none
    union {
        u32 palette[40][32];                   // lane-private scratch of the index search, [entry][lane]: 24 palette
                                               // entries, then 5 per-subset constants x 3 subsets
        // winner selection (no index search runs then): the best (error, list position) of each strip of 16 list entries
        struct {
            int err[kBc7Strips][kBc7Slots][2], pos[kBc7Strips][kBc7Slots][2];
        } strip;
    };
    union {
        // every DISTINCT three-subset mask, for the four blocks of the group (bc7_phase_masks3 -> bc7_phase_shapes3): the
        // mode-2 subset error of all 140 masks, the decoded mode-0 endpoints (A, B as RGBA bytes) of the 36 masks of shapes 0..15
        struct {
            int err2[kBc7Slots][ITW_MASK3_COUNT];
            u32 ends0[kBc7Slots][ITW_MASK3_FIRST][2];
        } masks3;
        // two-subset shapes of the group, after its three-subset phases
        struct {
            int keys[kBc7Slots][64];           // split-bound keys of the set being ranked: dead once `order` is written
        } two;
        // chain phase of a two-half round: the FIRST half again (re-read from the staged tile once its slot in blk[] has
        // been taken by the second half; the mask tables are dead by then)
        Bc7Block parked[kBc7Batch];
    };
    int nvalid;                                // valid blocks in blk[]
    int half;                                  // which half of the round blk[] holds (0 / 1)
    int ntotal;                                // valid blocks of the round (chain and store phases)
    int nparked;                               // blocks in parked[]: the round's blocks [0, nparked); blk[] holds the rest
};
// mode slots m = 0..4 <-> BC7 modes {0, 2, 1, 3, 7}: the reference's evaluation order
ITW_HD int bc7_slot_mode(int m) { return (m == 0) ? 0 : ((m == 1) ? 2 : ((m == 2) ? 1 : ((m == 3) ? 3 : 7))); }
ITW_HD int bc7_mode_bits(int mode) { return (mode == 0 || mode == 1) ? 3 : ((mode == 6) ? 4 : 2); }

// number of candidates mode slot m evaluates under the profile; K:1386-1435
ITW_HD int bc7_slot_count(const Bc7Params& P, int m)
{
    if (m == 0) return P.sel[0] ? 16 : 0;
    if (m == 1) return (P.sel[0] && !P.skip2) ? 64 : 0;
    if (m == 2) return P.sel[1] ? P.t1 : 0;
    if (m == 3) return P.sel[1] ? P.t3 : 0;
    return P.sel[1] ? P.t7 : 0;
}
// A two-subset list that holds all 64 shapes is walked in shape order and never ranked: its winner, the first minimum in
// ranked (ascending key) order, is the minimum of (error, key), since the keys are unique (bc7_phase_strips).
ITW_HD bool bc7_shape_order(const Bc7Params& P, int m) { return m >= 2 && bc7_slot_count(P, m) == 64; }
// shape id of list position n of mode slot m
ITW_HD int bc7_slot_shape(const Bc7Warp& W, const Bc7Params& P, int slot, int m, int n)
{
    if (m <= 1) return 64 + n;                                  // modes 0/2 walk the 3-subset table in order
    if (bc7_shape_order(P, m)) return n;
    return W.order[slot][(m == 4) ? 1 : 0][n] & 63;             // shorter lists of modes 1/3/7 walk the ranked list
}

// ---------------------------------------------------------------------------------------------
// Views.  Modes 4/5 encode the block with one colour channel swapped with alpha ("rotation");
// for RGB profiles the swapped-in plane is the constant 255 (K:1579-1584).  rot = 3: no swap.
// ---------------------------------------------------------------------------------------------
struct View {
    const Bc7Block* b;
    int rot;      // 0..2 rotated channel, 3 = identity
    int alpha;    // 1: the swapped-in plane is alpha; 0: it is 255
};
ITW_HD u32 view_tex(const View& v, int k)
{
    const u32 t = v.b->tex[k];
    // byte `rot` <- byte 3 of the 2nd operand; rot = 3 with alpha reproduces t, so only "rot = 3 without alpha" (identity
    // views of RGB profiles) needs the plain selector
    const u32 swap_sel = (0x3210u & ~(0xFu << (4 * v.rot))) | (7u << (4 * v.rot));
    const u32 sel = (v.rot < 3) ? swap_sel : 0x3210u;
    return byte_perm(t, v.alpha ? t : 0xFFFFFFFFu, sel);
}
ITW_HD u32 view_plane(const View& v, int c, int i)          // branch-free: one load from a selected plane, one select
{
    const bool swapped = (c == v.rot);
    const u32 p = v.b->plane[swapped ? 3 : c][i];
    return (swapped && !v.alpha) ? 0xFFFFFFFFu : p;
}
ITW_HD u32 nibble_to_bytemask(u32 nib) { return (((nib & 15u) * 0x00204081u) & 0x01010101u) * 0xFFu; }

// ---------------------------------------------------------------------------------------------
// raw moments of the masked texels as exact integers; slots as K:763-803
// ---------------------------------------------------------------------------------------------
ITW_HD void moments_u8(int (&st)[15], const u32 (&P)[4][4], u32 mask, int channels)
{
    u32 s[15];
#pragma unroll
    for (int i = 0; i < 15; i++) s[i] = 0u;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const u32 bm = nibble_to_bytemask(mask >> (4 * i));
        const u32 r = P[0][i] & bm, g = P[1][i] & bm, b = P[2][i] & bm;
        s[10] = dp4a_u8(r, 0x01010101u, s[10]);
        s[11] = dp4a_u8(g, 0x01010101u, s[11]);
        s[12] = dp4a_u8(b, 0x01010101u, s[12]);
        s[0] = dp4a_u8(r, P[0][i], s[0]);
        s[1] = dp4a_u8(r, P[1][i], s[1]);
        s[2] = dp4a_u8(r, P[2][i], s[2]);
        s[4] = dp4a_u8(g, P[1][i], s[4]);
        s[5] = dp4a_u8(g, P[2][i], s[5]);
        s[7] = dp4a_u8(b, P[2][i], s[7]);
        if (channels == 4) {
            const u32 a = P[3][i] & bm;
            s[13] = dp4a_u8(a, 0x01010101u, s[13]);
            s[3] = dp4a_u8(r, P[3][i], s[3]);
            s[6] = dp4a_u8(g, P[3][i], s[6]);
            s[8] = dp4a_u8(b, P[3][i], s[8]);
            s[9] = dp4a_u8(a, P[3][i], s[9]);
        }
    }
    s[14] = (u32)popcount16(mask & 0xFFFFu);
#pragma unroll
    for (int i = 0; i < 15; i++) st[i] = (int)s[i];
}
ITW_HD void load_planes(u32 (&P)[4][4], const View& v)
{
#pragma unroll
    for (int c = 0; c < 4; c++)
#pragma unroll
        for (int i = 0; i < 4; i++) P[c][i] = view_plane(v, c, i);
}

// Power iteration on a packed symmetric matrix [xx xy xz xw yy yz yw zz zw ww]; K:207-229.  Continues from the vector in
// `axis` (the reference starts from (1, 1, 1, 1)); kIterations is even, so the renormalisation keeps the reference's parity
// when a run is split in two.  Unroll factor measured (tools/tune_unroll.sh): rolled by 4 in round 1, when the kernel was
// instruction-cache bound; fully unrolled is 0.4 % faster now.
template <int CH, int kIterations>
ITW_HD void bc7_power_axis(float (&axis)[4], const float (&m)[10])
{
    static_assert(kIterations % 2 == 0, "renormalisation parity");
    float v0 = axis[0], v1 = axis[1], v2 = axis[2], v3 = axis[3];
    ITW_UNROLL(ITW_BC7_POWER_UNROLL)
    for (int it = 0; it < kIterations; it++) {
        float a0, a1, a2, a3 = 0.0f;
        if (CH == 3) {
            a0 = m[0] * v0 + m[1] * v1 + m[2] * v2;
            a1 = m[1] * v0 + m[4] * v1 + m[5] * v2;
            a2 = m[2] * v0 + m[5] * v1 + m[7] * v2;
        } else {
            a0 = m[0] * v0 + m[1] * v1 + m[2] * v2 + m[3] * v3;
            a1 = m[1] * v0 + m[4] * v1 + m[5] * v2 + m[6] * v3;
            a2 = m[2] * v0 + m[5] * v1 + m[7] * v2 + m[8] * v3;
            a3 = m[3] * v0 + m[6] * v1 + m[8] * v2 + m[9] * v3;
        }
        v0 = a0; v1 = a1; v2 = a2; v3 = a3;
        if (it & 1) {                                  // renormalise every other iteration: 1/sqrt, two exact ops
            float n2 = a0 * a0;
            n2 += a1 * a1;
            n2 += a2 * a2;
            if (CH == 4) n2 += a3 * a3;
            const float rn = 1.0f / sqrtf(n2);
            v0 *= rn; v1 *= rn; v2 *= rn; v3 *= rn;
        }
    }
    axis[0] = v0; axis[1] = v1; axis[2] = v2; axis[3] = v3;
}
// cov = sum(xy) - sum(x)*sum(y)/n on exact integer moments; K:805-823.  sum(x)*sum(y) < 2^24 is an
// exact integer, so the division by the count can use the slow-path-free exact quotient.
template <int CH>
ITW_HD void bc7_covariance(float (&cov)[10], float (&mean)[4], const int (&st)[15])
{
    const float n = (float)st[14], rn = 1.0f / n;
    float s[4];
#pragma unroll
    for (int c = 0; c < 4; c++) s[c] = (float)st[10 + c];
#pragma unroll
    for (int i = 0; i < 10; i++) cov[i] = 0.0f;
    cov[0] = (float)st[0] - div_by_rcp(s[0] * s[0], n, rn);
    cov[1] = (float)st[1] - div_by_rcp(s[0] * s[1], n, rn);
    cov[2] = (float)st[2] - div_by_rcp(s[0] * s[2], n, rn);
    cov[4] = (float)st[4] - div_by_rcp(s[1] * s[1], n, rn);
    cov[5] = (float)st[5] - div_by_rcp(s[1] * s[2], n, rn);
    cov[7] = (float)st[7] - div_by_rcp(s[2] * s[2], n, rn);
    if (CH == 4) {
        cov[3] = (float)st[3] - div_by_rcp(s[0] * s[3], n, rn);
        cov[6] = (float)st[6] - div_by_rcp(s[1] * s[3], n, rn);
        cov[8] = (float)st[8] - div_by_rcp(s[2] * s[3], n, rn);
        cov[9] = (float)st[9] - div_by_rcp(s[3] * s[3], n, rn);
    }
#pragma unroll
    for (int c = 0; c < 4; c++) mean[c] = (c < CH) ? div_by_rcp(s[c], n, rn) : 0.0f;
}
// By-value working set of the shape and chain phases: nvcc keeps these small structs in registers across the
// non-inlined calls, whereas arrays handed over by pointer live in local memory (see bc6h.cuh).
struct Bc7Seg { float v[8]; };                       // endpoints A (r,g,b,a) and B (r,g,b,a) of one subset
struct Bc7Packed { u32 dec_a, dec_b, q_a, q_b; };    // decoded A, B and quantised A, B as RGBA bytes
struct Bc7Search { int err; u32 idx0, idx1; };

// trace - lambda_max of a scaled covariance, from the axis of its power iteration; K:925-938
template <int CH>
ITW_HD float bc7_bound_from_axis(const float (&cov)[10], const float (&axis)[4])
{
    float mv[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (CH == 3) {
        mv[0] = cov[0] * axis[0] + cov[1] * axis[1] + cov[2] * axis[2];
        mv[1] = cov[1] * axis[0] + cov[4] * axis[1] + cov[5] * axis[2];
        mv[2] = cov[2] * axis[0] + cov[5] * axis[1] + cov[7] * axis[2];
    } else {
        mv[0] = cov[0] * axis[0] + cov[1] * axis[1] + cov[2] * axis[2] + cov[3] * axis[3];
        mv[1] = cov[1] * axis[0] + cov[4] * axis[1] + cov[5] * axis[2] + cov[6] * axis[3];
        mv[2] = cov[2] * axis[0] + cov[5] * axis[1] + cov[7] * axis[2] + cov[8] * axis[3];
        mv[3] = cov[3] * axis[0] + cov[6] * axis[1] + cov[8] * axis[2] + cov[9] * axis[3];
    }
    float sum = 0.0f;
#pragma unroll
    for (int c = 0; c < CH; c++) sum += sq(mv[c]);
    float bound = cov[0] + cov[4] + cov[7];
    if (CH == 4) bound += cov[9];
    bound -= sqrtf(sum);
    return max_sse(bound, 0.0f);
}
// Scales a covariance by 1/256^2 and adds eps to its diagonal.  The fit puts eps on all four diagonal slots (K:842-852); the
// split bound on three only (K:911-920), so a four-channel bound differs from the fit's in slot 9.
template <bool kEps9>
ITW_HD void bc7_scale_covariance(float (&cov)[10])
{
    const float inv_var = 1.0f / (256.0f * 256.0f);
#pragma unroll
    for (int i = 0; i < 10; i++) cov[i] *= inv_var;
    const float eps = 0.001f * 0.001f;
    cov[0] += eps; cov[4] += eps; cov[7] += eps;
    if (kEps9) cov[9] += eps;
}
// The PCA line of a set of moments (K:834-855): mean and principal axis after eight power iterations.  kBound: also the split
// bound of the mask (bc7_residual_bound).  At three channels the fit's scaled covariance equals the bound's (slot 9 is never
// read), and the bound's four power iterations are the fit's first four.
struct Bc7Line { float axis[4], mean[4], bound; };
template <int CH, bool kBound>
ITW_HD Bc7Line bc7_line(const int (&st)[15])
{
    static_assert(!kBound || CH == 3, "the four-channel fit adds eps to slot 9, the split bound does not");
    Bc7Line l;
    float cov[10];
    bc7_covariance<CH>(cov, l.mean, st);
    bc7_scale_covariance<true>(cov);
#pragma unroll
    for (int c = 0; c < 4; c++) l.axis[c] = 1.0f;
    bc7_power_axis<CH, 4>(l.axis, cov);
    l.bound = kBound ? bc7_bound_from_axis<CH>(cov, l.axis) : 0.0f;
    bc7_power_axis<CH, 4>(l.axis, cov);
    return l;
}
// Position of texel k along a line through `mean` (K:874-876).  The reference starts the sum from 0.0f; 0 + x differs from
// x only in the sign of a zero, which nothing downstream can observe (bc7_fit), so the sum starts from the first product.
template <int CH>
ITW_HD float bc7_project(const float (&axis)[4], const float (&mean)[4], const u32 (&P)[4][4], int k)
{
    float d = axis[0] * ((float)((P[0][k >> 2] >> (8 * (k & 3))) & 255u) - mean[0]);
#pragma unroll
    for (int c = 1; c < CH; c++) d += axis[c] * ((float)((P[c][k >> 2] >> (8 * (k & 3))) & 255u) - mean[c]);
    return d;
}
// Endpoints of the line's span [lo, hi], widened to one unit when shorter and clamped to [0,255]; K:882-905.  v[0..3] = A,
// v[4..7] = B; components >= CH are zero (the reference's never-written slots, rule F6).
template <int CH>
ITW_HD Bc7Seg bc7_ends(const Bc7Line& l, float lo, float hi)
{
    if (hi - lo < 1.0f) { lo -= 0.5f; hi += 0.5f; }
    Bc7Seg seg;
#pragma unroll
    for (int i = 0; i < 8; i++) seg.v[i] = 0.0f;
#pragma unroll
    for (int c = 0; c < CH; c++) {
        seg.v[c] = clamp_sse(lo * l.axis[c] + l.mean[c], 0.0f, 255.0f);
        seg.v[4 + c] = clamp_sse(hi * l.axis[c] + l.mean[c], 0.0f, 255.0f);
    }
    return seg;
}
template <int CH>
ITW_HD Bc7Seg bc7_fit_impl(const View& v, u32 mask)
{
    u32 P[4][4];
    load_planes(P, v);
    int st[15];
    moments_u8(st, P, mask, CH);
    const Bc7Line l = bc7_line<CH, false>(st);
    float lo = inf_f(), hi = -inf_f();
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const float d = bc7_project<CH>(l.axis, l.mean, P, k);
        // d is finite here (8-bit texels, finite axis), so the reference's (a<b)?a:b equals fminf/fmaxf up to
        // the sign of a zero, which the affine map of bc7_ends cannot observe: one FMNMX instead of FSETP+FSEL
        if ((mask >> k) & 1u) {
            lo = fminf(lo, d);
            hi = fmaxf(hi, d);
        }
    }
    return bc7_ends<CH>(l, lo, hi);
}
// PCA line through the masked texels, clamped to [0,255]; K:834-905.
ITW_HD_NOINLINE Bc7Seg bc7_fit(const Bc7Block* blk, int rot, int alpha, u32 mask, int channels)
{
    const View v{blk, rot, alpha};
    return (channels == 4) ? bc7_fit_impl<4>(v, mask) : bc7_fit_impl<3>(v, mask);
}
// bc7_fit of all sixteen texels (the one-subset chains): the constant mask folds the masking out of the moments and the
// mask test out of the projection loop; the line and its rounding are bc7_fit's.
ITW_HD_NOINLINE Bc7Seg bc7_fit_full(const Bc7Block* blk, int rot, int alpha, int channels)
{
    const View v{blk, rot, alpha};
    return (channels == 4) ? bc7_fit_impl<4>(v, 0xFFFFu) : bc7_fit_impl<3>(v, 0xFFFFu);
}
// Both subsets of a two-subset shape of an untransformed block: the same values as bc7_fit of mask0 and of its complement
// (and, at three channels, their split bounds), with the work the two fits share done once.  Subset 1's integer moments are
// the block's minus subset 0's (exact); the two lines are independent, so the scheduler can interleave them; one projection
// loop sends every texel to its own subset's line.  That loop reads the texels from the register planes and selects the line
// per texel: one set-bit walk per subset with its line in registers (texel words from shared memory, as bc7_pair_error) made
// the `slow` profile 1.1 % slower on H100.
struct Bc7Pair { Bc7Seg seg[2]; float bound[2]; };
template <int CH>
ITW_HD Bc7Pair bc7_fit_pair_impl(const Bc7Block* blk, u32 mask0)
{
    u32 P[4][4];
    load_planes(P, View{blk, 3, 1});
    int full[15], part[15], rest[15];
    moments_u8(full, P, 0xFFFFu, CH);
    moments_u8(part, P, mask0, CH);
#pragma unroll
    for (int i = 0; i < 15; i++) rest[i] = full[i] - part[i];
    const Bc7Line l0 = bc7_line<CH, CH == 3>(part), l1 = bc7_line<CH, CH == 3>(rest);
    float lo0 = inf_f(), hi0 = -inf_f(), lo1 = inf_f(), hi1 = -inf_f();
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const bool in0 = (mask0 >> k) & 1u;
        float axis[4], mean[4];
#pragma unroll
        for (int c = 0; c < 4; c++) { axis[c] = in0 ? l0.axis[c] : l1.axis[c]; mean[c] = in0 ? l0.mean[c] : l1.mean[c]; }
        const float d = bc7_project<CH>(axis, mean, P, k);
        if (in0) { lo0 = fminf(lo0, d); hi0 = fmaxf(hi0, d); }
        else     { lo1 = fminf(lo1, d); hi1 = fmaxf(hi1, d); }
    }
    return Bc7Pair{{bc7_ends<CH>(l0, lo0, hi0), bc7_ends<CH>(l1, lo1, hi1)}, {l0.bound, l1.bound}};
}
// mask0 = subset 0 of a two-subset shape; bound[] is set at three channels only
ITW_HD_NOINLINE Bc7Pair bc7_fit_pair(const Bc7Block* blk, u32 mask0, int channels)
{
    return (channels == 4) ? bc7_fit_pair_impl<4>(blk, mask0) : bc7_fit_pair_impl<3>(blk, mask0);
}
// Two subset masks of an untransformed block at three channels (a lane pair of the three-subset masks): the same values as
// bc7_fit(blk, 3, 1, mask, 3) of each.  The masks are not complements, so each has its own moment pass; the two lines are
// independent, so the scheduler can interleave them; one projection loop converts every texel once and projects it onto
// both.  Inlined into bc7_phase_masks3, like bc7_masks_error2: as non-inlined routines they moved ptxas's register
// assignment of the shared callees so that bc7_chain spilled 160 bytes instead of 4 to 20 (-Xptxas -v), and basic /
// alpha_basic ran 0.4 / 1.4 % slower on H100.
struct Bc7Segs2 { Bc7Seg seg[2]; };
ITW_HD Bc7Segs2 bc7_fit_masks2(const Bc7Block* blk, u32 mask_a, u32 mask_b)
{
    u32 P[4][4];
    load_planes(P, View{blk, 3, 1});
    int sta[15], stb[15];
    moments_u8(sta, P, mask_a, 3);
    moments_u8(stb, P, mask_b, 3);
    const Bc7Line la = bc7_line<3, false>(sta), lb = bc7_line<3, false>(stb);
    float loa = inf_f(), hia = -inf_f(), lob = inf_f(), hib = -inf_f();
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const float da = bc7_project<3>(la.axis, la.mean, P, k), db = bc7_project<3>(lb.axis, lb.mean, P, k);
        if ((mask_a >> k) & 1u) { loa = fminf(loa, da); hia = fmaxf(hia, da); }
        if ((mask_b >> k) & 1u) { lob = fminf(lob, db); hib = fmaxf(hib, db); }
    }
    return Bc7Segs2{{bc7_ends<3>(la, loa, hia), bc7_ends<3>(lb, lob, hib)}};
}

// trace - lambda_max of a covariance after four power iterations; K:907-939
template <int CH>
ITW_HD float bc7_residual_bound(float (&cov)[10])
{
    bc7_scale_covariance<false>(cov);
    float axis[4] = {1.0f, 1.0f, 1.0f, 1.0f};
    bc7_power_axis<CH, 4>(axis, cov);
    return bc7_bound_from_axis<CH>(cov, axis);
}
// Ranking key of a two-subset shape from the bounds of its subsets; K:952-971, :1403-1410
ITW_HD int bc7_key_of(int shape, float bound0, float bound1)
{
    float b = 0.0f;
    b += bound0;
    b += bound1;
    return shape + (int)((unsigned)cvt_x86(sqrtf(b) * 256.0f) * 64u);
}
// subset 1 = full - subset 0
template <int CH>
ITW_HD int bc7_split_key_impl(const Bc7Block* blk, int shape)
{
    const View v{blk, 3, 1};
    u32 P[4][4];
    load_planes(P, v);
    int full[15], part[15], rest[15];
    moments_u8(full, P, 0xFFFFu, CH);
    moments_u8(part, P, (u32)shape_mask(shape, 0), CH);
#pragma unroll
    for (int i = 0; i < 15; i++) rest[i] = full[i] - part[i];            // exact: the reference subtracts exact floats
    float c1[10], c2[10], mean[4];
    bc7_covariance<CH>(c1, mean, part);
    bc7_covariance<CH>(c2, mean, rest);
    const float b0 = bc7_residual_bound<CH>(c1);
    return bc7_key_of(shape, b0, bc7_residual_bound<CH>(c2));
}
ITW_HD_NOINLINE int bc7_split_key(const Bc7Block* blk, int shape, int channels)
{
    return (channels == 4) ? bc7_split_key_impl<4>(blk, shape) : bc7_split_key_impl<3>(blk, shape);
}

// Quantise one endpoint pair; K:983-1128.  out[0],out[1] = decoded A,B as RGBA bytes, out[2],out[3] =
// quantised A,B as RGBA bytes.  `channels` = components that vote on the p-bit (K:1011-1020); all four
// components are always produced (a never-written component is quantised from 0, rule F6).
// One rolled loop over the 8 components serves all three families:
//   modes 0,3,6,7  one p-bit per endpoint   K:983-1022   (the vote compares against the RAW quantised value
//                                                         except in mode 0 -- reference behaviour, K:1003-1009)
//   mode 1         one p-bit per pair        K:1024-1052  (a single running error sum over both endpoints)
//   modes 2,4,5    no p-bit                  K:1054-1065
// decodes four quantised bytes of `bits` bits at once (K:1093-1122): v << (8-d) | that >> d, bytewise
ITW_HD u32 bc7_decode_packed(u32 q, int bits)
{
    const u32 vv = q << (8 - bits);
    return vv + ((vv >> bits) & (0x01010101u * (0xFFu >> bits)));
}
ITW_HD Bc7Packed bc7_quantise_impl(const Bc7Seg& seg, int mode, int channels)
{
    const float (&ep)[8] = seg.v;
    // per-mode constants from nibble tables (mode 0 in the low nibble): nested conditionals on `mode` compile to a jump table
    // that cost more than a tenth of this routine
    const int family = (int)((0x00220210u >> (4 * mode)) & 3u);           // 1: mode 1; 2: modes 2, 4, 5; else 0
    // stored bits per component including the p-bit: 2^qbits - 1 is K's `levels2` (p-bit modes) or `levels-1`
    const int qbits = (int)((0x68758575u >> (4 * mode)) & 15u);           // modes 0,2,4: 5; 1,5: 7; 7: 6; 3,6: 8
    const int top = (1 << qbits) - 1;
    const float ftop = (float)top;
    const int vote_bits = (int)((0x88888875u >> (4 * mode)) & 15u);       // mode 0: 5; mode 1: 7; else 8 (expand_bits(v, 8) == v)
    const int votes = (mode == 1) ? 3 : channels;
    // Conversions: |ep| < 2^31 always holds here -- the fit clamps to [0,255] and the least-squares
    // solve divides by an exact non-zero INTEGER determinant (bc7_solve), which bounds |ep| by ~1.2e7 --
    // so the x86 overflow rule of cvt_x86() can never trigger and a plain truncation is identical.
    // t*0.5 and (t-1)*0.5 are exact (power-of-two scaling), so fusing the +0.5 rounds once, exactly like
    // the reference's separate multiply and add.
    // Modes 0-3 never emit a 4th component and their index search ignores it; it only matters when it votes
    // (alpha profiles refining modes 0/3, quirk Q1).  Otherwise it is skipped (its byte stays 0).
    const bool four = !(mode <= 3 && votes <= 3);
    // Branch-free per component: the no-p-bit family is the p-bit formula with scale 1 instead of 1/2 (t*1 + 0.5 rounds
    // once, like t + 0.5) and both candidates equal.  Components 0..2 always take part and always vote (votes >= 3);
    // only the fourth is conditional.
    const bool plain = (family == 2);
    const float half = plain ? 1.0f : 0.5f;
    const int step = plain ? 1 : 2, top0 = plain ? top : top - 1;
    u32 cand0[2] = {0u, 0u}, cand1[2] = {0u, 0u};
    bool pick1[2] = {false, false};
    float e0 = 0.0f, e1 = 0.0f;
    if (plain) {
        // no p-bit (modes 2, 4, 5; K:1054-1065): one candidate per component, no vote -- a third of all quantisations
#pragma unroll
        for (int i = 0; i < 2; i++) {
            u32 c0 = 0u;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                if (c == 3 && !four) continue;
                const float t = div255(ep[4 * i + c]) * ftop;
                c0 |= (u32)clampi(trunc_i(fma_rn(t, 1.0f, 0.5f)), 0, top) << (8 * c);
            }
            cand0[i] = c0;
        }
    } else
#pragma unroll
    for (int i = 0; i < 2; i++) {
        if (family == 0) { e0 = 0.0f; e1 = 0.0f; }
        u32 c0 = 0u, c1 = 0u;
#pragma unroll
        for (int c = 0; c < 4; c++) {
            if (c == 3 && !four) continue;
            const float x = ep[4 * i + c];
            const float t = div255(x) * ftop;
            const int v0 = clampi(trunc_i(fma_rn(t, half, 0.5f)) * step, 0, top0);
            const int v1p = clampi(trunc_i(fma_rn(t - 1.0f, 0.5f, 0.5f)) * 2 + 1, 1, top);      // ((t - 1)/2 + 0.5) truncated, *2 + 1
            const int v1 = plain ? v0 : v1p;
            c0 |= (u32)v0 << (8 * c);
            c1 |= (u32)v1 << (8 * c);
            const float d0 = sq(x - (float)expand_bits(v0, vote_bits)), d1 = sq(x - (float)expand_bits(v1, vote_bits));
            if (c < 3 || votes == 4) { e0 += d0; e1 += d1; }
        }
        const bool p = !(e0 < e1);
        if (i == 0) { cand0[0] = c0; cand1[0] = c1; pick1[0] = p; }
        else        { cand0[1] = c0; cand1[1] = c1; pick1[1] = p; }
    }
    if (family == 1) pick1[0] = pick1[1];                                // decided after both endpoints
    if (family == 2) pick1[0] = pick1[1] = false;
    u32 dec[2], qq[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        qq[i] = pick1[i] ? cand1[i] : cand0[i];
        dec[i] = bc7_decode_packed(qq[i], qbits);                        // every mode decodes the bits it stores
    }
    return Bc7Packed{dec[0], dec[1], qq[0], qq[1]};
}
ITW_HD_NOINLINE Bc7Packed bc7_quantise(Bc7Seg seg, int mode, int channels) { return bc7_quantise_impl(seg, mode, channels); }
// One three-channel segment for modes 1 and 3 (the full two-subset lists): the same code with the mode and the channel count
// known at compile time, so that the per-mode constants, the no-p-bit branch and the fourth component fold away.
struct Bc7Packed13 { Bc7Packed m1, m3; };
ITW_HD_NOINLINE Bc7Packed13 bc7_quantise13(Bc7Seg seg)
{
    return Bc7Packed13{bc7_quantise_impl(seg, 1, 3), bc7_quantise_impl(seg, 3, 3)};
}
// The same code for one mode and voting channel count known at compile time: the three-subset masks phase (modes 0 and 2)
// and the mode-6 chain.  The rotation units inline bc7_quantise_impl for modes 4 and 5 (no p-bit, so nothing votes and the
// channel count does not matter to them).
template <int kMode, int kChannels>
ITW_HD_NOINLINE Bc7Packed bc7_quantise_m(Bc7Seg seg) { return bc7_quantise_impl(seg, kMode, kChannels); }

// Index search; K:1133-1193.  ends[2j], ends[2j+1] = decoded endpoints A,B of subset j (RGBA bytes);
// chmask zeroes the channels that do not take part (0x00FFFFFF for three-channel modes).
// Returns the summed error (exact integer) and the sixteen 4-bit indices in idx[0..1].
// bits_flags = index bits, plus kAssignThresholds when the caller allows the integer-threshold form of the two-bit search.
// The shape phases do: there every lane of the warp searches the same mode at the same time.  The partitioned chains do
// not: their passes pair mode 0 with mode 2 and mode 1 with mode 3, and two texel loops would run one after the other.
constexpr int kAssignThresholds = 8;
// Palette, K:1172: ((64 - w) a + w b + 32) >> 6 per channel, two channels per 32-bit word.  Written as (64 a + 32) + w (b - a):
// the packed difference may borrow across the 16-bit lanes, but every lane of the SUM is the non-negative 14-bit value above,
// so the word arithmetic is exact.  w = 0 and w = 64 give the endpoints.
struct Bc7Lerp {
    u32 base_rb, base_ga, d_rb, d_ga;
    ITW_HD u32 entry(u32 w) const
    {
        return (((base_rb + w * d_rb) >> 6) & 0x00FF00FFu) | (((base_ga + w * d_ga) << 2) & 0xFF00FF00u);
    }
};
ITW_HD Bc7Lerp bc7_lerp(u32 a, u32 b)
{
    const u32 m = 0x00FF00FFu;
    const u32 a_rb = a & m, a_ga = (a >> 8) & m;
    return Bc7Lerp{(a_rb << 6) + 0x00200020u, (a_ga << 6) + 0x00200020u, (b & m) - a_rb, ((b >> 8) & m) - a_ga};
}
// Per-subset constants of a search with endpoints a, b (channels that do not take part already zeroed): the numerator offset
// cj = a.(b - a) and the squared length idiv = |b - a|^2, exact integers, and the palette interpolation.
struct Bc7Sub { u32 a, b; int cj, idiv; Bc7Lerp lerp; };
ITW_HD Bc7Sub bc7_sub(u32 a, u32 b)
{
    const u32 aa = dp4a_u8(a, a, 0u), ab = dp4a_u8(a, b, 0u), bb = dp4a_u8(b, b, 0u);
    return Bc7Sub{a, b, (int)(ab - aa), (int)(bb - 2u * ab + aa), bc7_lerp(a, b)};
}
// Projection numerator of texel t, sum_c (t_c - a_c)(b_c - a_c): an integer, |value| < 2^18, so the float it converts to is
// the reference's float sum (K:1148-1156)
ITW_HD int bc7_num(u32 t, u32 a, u32 b, int cj) { return (int)dp4a_u8(t, b, 0u) - (int)dp4a_u8(t, a, 0u) - cj; }
// q1 by the quotient num / div of K:1158, evaluated as the exact FMA-corrected quotient (proved equal to IEEE num/div on this
// integer domain, tests/test_exact_division.py).  |proj*levels| < 2^23, so truncation never overflows; NaN (coincident
// endpoints, 0/0) becomes INT_MIN on x86 and 0 here -- both clamp to 1 (K:1160-1161).  proj*levels is exact, so the fused
// form rounds once like the reference's multiply-then-add.
ITW_HD int bc7_q1_quotient(int num, float fdiv, float rdiv, float flevels, int levels)
{
    const float proj = div_by_rcp((float)num, fdiv, rdiv);
    return clampi(trunc_i(fma_rn(proj, flevels, 0.5f)), 1, levels - 1);
}
// Two-bit search by thresholds: q1 = 1 + (num >= t2) + (num >= t3), t2 <= t3.  The reference's
// q1 = clamp((int)(RN(RN(num / div) * 4) + 0.5), 1, 3) is a non-decreasing step function of the integer num; with
// tau = (2m - 1) / 8 (a float): RN(p * 4 + 0.5) >= m <=> p >= tau (the sum is exact below the next binade, and the binade
// boundary itself is an integer m), and RN(num / div) >= tau <=> num / div >= tau because a quotient below tau stays at
// least 1 / (8 div) > 2^-21 away from it while half an ulp of tau is below 2^-24 (div <= 4 * 255^2 < 2^18).  So
// q1 >= m  <=>  8 num >= (2m - 1) div  <=>  num >= ceil((2m - 1) div / 8), m = 2, 3; coincident endpoints give 0/0 = NaN ->
// q1 = 1 in the reference: thresholds out of reach.  tests/test_exact_division.py checks both sides of every step for every
// possible div.
struct Bc7Thresholds { int t2, t3; };
ITW_HD Bc7Thresholds bc7_thresholds(int idiv)
{
    return Bc7Thresholds{idiv ? (3 * idiv + 7) >> 3 : 0x7fffffff, idiv ? (5 * idiv + 7) >> 3 : 0x7fffffff};
}
struct Bc7Steps {
    bool ge2, ge3;
    ITW_HD int q1() const { return 1 + (ge2 ? 1 : 0) + (ge3 ? 1 : 0); }
};
ITW_HD Bc7Steps bc7_steps(int num, int t2, int t3) { return Bc7Steps{num >= t2, num >= t3}; }
// The better of palette entries q1 - 1 (`lo`) and q1 (`hi`) for texel t: VABSDIFF4 + IDP.4A errors, q1 on a tie (K:1163-1184)
struct Bc7Pick { int err; bool first; };
ITW_HD Bc7Pick bc7_pick(u32 lo, u32 hi, u32 t)
{
    const u32 d0 = absdiff_u8x4(lo, t), d1 = absdiff_u8x4(hi, t);
    const int e0 = (int)dp4a_u8(d0, d0, 0u), e1 = (int)dp4a_u8(d1, d1, 0u);
    const bool first = e0 < e1;
    return Bc7Pick{first ? e0 : e1, first};
}
// bc7_assign's texel loop: palette and per-subset constants from lane-private shared memory.  kThresholds: the two-bit
// search by thresholds; kIdentity: the texel words are read as stored (every shape-phase search and the partitioned
// chains), else through the rotated view.  Separate instantiations, not a branch inside the loop.  The one-subset chains
// search with bc7_assign_rotation and bc7_assign_one.
template <bool kThresholds, bool kIdentity>
ITW_HD Bc7Search bc7_assign_texels(const u32 (*pal)[32], int lane, const View& v, int levels, u32 pattern, u32 chmask)
{
    const u32* tx = (chmask == 0x00FFFFFFu) ? v.b->rgb : v.b->tex;
    const int lv = kThresholds ? 4 : levels;
    const float flevels = (float)levels;
    int total = 0;
    u32 out0 = 0u, out1 = 0u;
    ITW_UNROLL(ITW_BC7_ASSIGN_UNROLL)
    for (int k = 0; k < 16; k++) {
        const u32 t = kIdentity ? tx[k] : (view_tex(v, k) & chmask);
        const int j = (int)((pattern >> (2 * k)) & 3u);
        const int num = bc7_num(t, pal[24 + 5 * j + 0][lane], pal[24 + 5 * j + 1][lane], (int)pal[24 + 5 * j + 2][lane]);
        const int q1 = kThresholds ? bc7_steps(num, (int)pal[24 + 5 * j + 3][lane], (int)pal[24 + 5 * j + 4][lane]).q1()
                                   : bc7_q1_quotient(num, bits_float(pal[24 + 5 * j + 3][lane]), bits_float(pal[24 + 5 * j + 4][lane]),
                                                     flevels, levels);
        const Bc7Pick p = bc7_pick(pal[j * lv + q1 - 1][lane], pal[j * lv + q1][lane], t);
        total += p.err;
        const u32 bq = (u32)(p.first ? q1 - 1 : q1) << (4 * (k & 7));
        if (k < 8) out0 += bq; else out1 += bq;
    }
    return Bc7Search{total, out0, out1};
}
ITW_HD_NOINLINE Bc7Search bc7_assign(u32 (*pal)[32], int lane, const Bc7Block* blk, int rot, int alpha, int bits_flags, int pairs,
                                     u32 pattern, u32 e0, u32 e1, u32 e2, u32 e3, u32 e4, u32 e5, u32 chmask)
{
    const View v{blk, rot, alpha};
    const int bits = bits_flags & 7;
    const bool thresholds = (bits_flags == (2 | kAssignThresholds)) && rot == 3;
    const int levels = 1 << bits;
    // per-subset constants go to lane-private shared memory too and are fetched by subset id in the texel
    // loop: the load/store pipe is nearly idle in this kernel while the ALU pipe (selects) is the busiest
    u32 cur_a = e0, cur_b = e1, next_a = e2, next_b = e3;        // endpoints walk through two register pairs: no select by j
    for (int j = 0; j < pairs; j++) {
        const Bc7Sub s = bc7_sub(cur_a & chmask, cur_b & chmask);
        cur_a = next_a; cur_b = next_b; next_a = e4; next_b = e5;
        pal[24 + 5 * j + 0][lane] = s.a;
        pal[24 + 5 * j + 1][lane] = s.b;
        pal[24 + 5 * j + 2][lane] = (u32)s.cj;
        if (thresholds) {
            const Bc7Thresholds th = bc7_thresholds(s.idiv);
            pal[24 + 5 * j + 3][lane] = (u32)th.t2;
            pal[24 + 5 * j + 4][lane] = (u32)th.t3;
        } else {
            const float fdiv = (float)s.idiv;
            pal[24 + 5 * j + 3][lane] = float_bits(fdiv);
            pal[24 + 5 * j + 4][lane] = float_bits(1.0f / fdiv);  // inf when the endpoints coincide (-> NaN, as 0/0)
        }
        pal[j * levels][lane] = s.a;
        pal[j * levels + levels - 1][lane] = s.b;
        for (int q = 1; q < levels - 1; q++) pal[j * levels + q][lane] = s.lerp.entry((u32)bc7_weight(bits, q));
    }
    if (thresholds) return bc7_assign_texels<true, true>(pal, lane, v, levels, pattern, chmask);
    if (rot == 3) return bc7_assign_texels<false, true>(pal, lane, v, levels, pattern, chmask);
    return bc7_assign_texels<false, false>(pal, lane, v, levels, pattern, chmask);
}
// Shape-phase searches without index bits (three channels, untransformed block): bc7_assign's texel step with each subset's
// constants and palette in registers.  The error of a shape is the sum of the errors of its subsets (exact integers).
// Two-bit constants of one subset (thresholds as in bc7_assign)
struct Bc7Sub2 { u32 a, b; int cj, t2, t3; u32 p1, p2; };
ITW_HD Bc7Sub2 bc7_sub2(u32 dec_a, u32 dec_b)
{
    const Bc7Sub s = bc7_sub(dec_a & 0x00FFFFFFu, dec_b & 0x00FFFFFFu);
    const Bc7Thresholds th = bc7_thresholds(s.idiv);
    return Bc7Sub2{s.a, s.b, s.cj, th.t2, th.t3, s.lerp.entry((u32)bc7_weight(2, 1)), s.lerp.entry((u32)bc7_weight(2, 2))};
}
ITW_HD Bc7Pick bc7_pick2(const Bc7Sub2& s, const Bc7Steps& q, u32 t)
{
    const u32 lo = q.ge3 ? s.p2 : (q.ge2 ? s.p1 : s.a), hi = q.ge3 ? s.b : (q.ge2 ? s.p2 : s.p1);      // entries q1 - 1, q1
    return bc7_pick(lo, hi, t);
}
ITW_HD int bc7_texel_error2(const Bc7Sub2& s, u32 t)
{
    return bc7_pick2(s, bc7_steps(bc7_num(t, s.a, s.b, s.cj), s.t2, s.t3), t).err;
}
// Three-bit constants of one subset
struct Bc7Sub3 { u32 a, b; int cj; float fdiv, rdiv; Bc7Lerp lerp; };
ITW_HD Bc7Sub3 bc7_sub3(u32 dec_a, u32 dec_b)
{
    const Bc7Sub s = bc7_sub(dec_a & 0x00FFFFFFu, dec_b & 0x00FFFFFFu);
    const float fdiv = (float)s.idiv;
    return Bc7Sub3{s.a, s.b, s.cj, fdiv, 1.0f / fdiv, s.lerp};
}
ITW_HD int bc7_texel_error3(const Bc7Sub3& s, u32 t)
{
    const int q1 = bc7_q1_quotient(bc7_num(t, s.a, s.b, s.cj), s.fdiv, s.rdiv, 8.0f, 8);
    return bc7_pick(s.lerp.entry((u32)bc7_weight(3, q1 - 1)), s.lerp.entry((u32)bc7_weight(3, q1)), t).err;
}
// Index searches of the one-subset chains: bc7_assign's texel step with the subset's constants in registers, no subset
// lookup, all sixteen texels.
ITW_HD void bc7_put_index(u32& out0, u32& out1, int k, int q)
{
    const u32 bq = (u32)q << (4 * (k & 7));
    if (k < 8) out0 += bq; else out1 += bq;
}
// Mode 6 (four-bit, identity view): q1 by the quotient, the palette in lane-private shared memory.  ea, eb = decoded
// endpoints A, B; chmask as in bc7_assign.
ITW_HD_NOINLINE Bc7Search bc7_assign_one(u32 (*pal)[32], int lane, const Bc7Block* blk, u32 ea, u32 eb, u32 chmask)
{
    const Bc7Sub s = bc7_sub(ea & chmask, eb & chmask);
    const int levels = 16;
    pal[0][lane] = s.a;
    pal[levels - 1][lane] = s.b;
    for (int q = 1; q < levels - 1; q++) pal[q][lane] = s.lerp.entry((u32)bc7_weight(4, q));
    const u32* tx = (chmask == 0x00FFFFFFu) ? blk->rgb : blk->tex;
    const float fdiv = (float)s.idiv, rdiv = 1.0f / fdiv;           // inf when the endpoints coincide (-> NaN, as 0/0)
    int total = 0;
    u32 out0 = 0u, out1 = 0u;
    ITW_UNROLL(ITW_BC7_ASSIGN_UNROLL)
    for (int k = 0; k < 16; k++) {
        const u32 t = tx[k];
        const int q1 = bc7_q1_quotient(bc7_num(t, s.a, s.b, s.cj), fdiv, rdiv, (float)levels, levels);
        const Bc7Pick p = bc7_pick(pal[q1 - 1][lane], pal[q1][lane], t);
        total += p.err;
        bc7_put_index(out0, out1, k, p.first ? q1 - 1 : q1);
    }
    return Bc7Search{total, out0, out1};
}
// The three searches of a rotation (bc7_chain_rotation; three channels, rotated view): mode 4 with index swap 0 and mode 5
// take q1 by the thresholds and their two entries from registers (bc7_pick2), mode 4 with swap 1 takes the three-bit
// quotient and computes its two entries from the interpolation (bc7_texel_error3).  One walk over the sixteen texels reads
// each rotated texel once for all three, as bc7_pair_error does for modes 1 and 3.
struct Bc7Search3 { Bc7Search s[3]; };                // mode 4 swap 0, mode 4 swap 1, mode 5
ITW_HD Bc7Search3 bc7_assign_rotation(const View& v, u32 a40, u32 b40, u32 a41, u32 b41, u32 a5, u32 b5)
{
    const Bc7Sub2 s40 = bc7_sub2(a40, b40), s5 = bc7_sub2(a5, b5);
    const Bc7Sub3 s41 = bc7_sub3(a41, b41);
    Bc7Search3 r;
#pragma unroll
    for (int j = 0; j < 3; j++) r.s[j] = Bc7Search{0, 0u, 0u};
    ITW_UNROLL(ITW_BC7_ASSIGN_UNROLL)
    for (int k = 0; k < 16; k++) {
        const u32 t = view_tex(v, k) & 0x00FFFFFFu;
        const Bc7Steps qa = bc7_steps(bc7_num(t, s40.a, s40.b, s40.cj), s40.t2, s40.t3);
        const Bc7Steps qc = bc7_steps(bc7_num(t, s5.a, s5.b, s5.cj), s5.t2, s5.t3);
        const int q1 = bc7_q1_quotient(bc7_num(t, s41.a, s41.b, s41.cj), s41.fdiv, s41.rdiv, 8.0f, 8);
        const Bc7Pick pa = bc7_pick2(s40, qa, t), pc = bc7_pick2(s5, qc, t);
        const Bc7Pick pb = bc7_pick(s41.lerp.entry((u32)bc7_weight(3, q1 - 1)), s41.lerp.entry((u32)bc7_weight(3, q1)), t);
        r.s[0].err += pa.err;
        r.s[1].err += pb.err;
        r.s[2].err += pc.err;
        bc7_put_index(r.s[0].idx0, r.s[0].idx1, k, pa.first ? qa.q1() - 1 : qa.q1());
        bc7_put_index(r.s[1].idx0, r.s[1].idx1, k, pb.first ? q1 - 1 : q1);
        bc7_put_index(r.s[2].idx0, r.s[2].idx1, k, pc.first ? qc.q1() - 1 : qc.q1());
    }
    return r;
}
// Mode-2 errors of the two subset masks of a lane pair: a subset's endpoints depend on its mask alone, so the three-subset
// phases search every distinct mask once.  One counted loop walks the set bits of both masks, so that the two error chains
// interleave; it is unrolled so that the texel loads of several iterations are in flight at once (a rolled loop waits for
// each load: four warps per scheduler do not hide that latency).  Each mask uses its own constants (e*a, e*b = decoded
// endpoints A, B).
struct Bc7Err2 { int a, b; };
ITW_HD Bc7Err2 bc7_masks_error2(const Bc7Block* blk, u32 mask_a, u32 mask_b, u32 ea_a, u32 ea_b, u32 eb_a, u32 eb_b)
{
    const Bc7Sub2 sa = bc7_sub2(ea_a, ea_b), sb = bc7_sub2(eb_a, eb_b);
    const int n = mini(popcount16(mask_a), popcount16(mask_b));
    int ta = 0, tb = 0;
    u32 ra = mask_a, rb = mask_b;
#pragma unroll 4
    for (int i = 0; i < n; i++) {
        const u32 la = ra & (0u - ra), lb = rb & (0u - rb);
        ra ^= la;
        rb ^= lb;
        ta += bc7_texel_error2(sa, blk->rgb[popcount32(la - 1u)]);
        tb += bc7_texel_error2(sb, blk->rgb[popcount32(lb - 1u)]);
    }
    // the rest of the longer mask: only one pair of the table has unequal popcounts (tools/gen_mask_tables.py)
#pragma unroll 1
    for (; ra; ra &= ra - 1u) ta += bc7_texel_error2(sa, blk->rgb[popcount32((ra & (0u - ra)) - 1u)]);
#pragma unroll 1
    for (; rb; rb &= rb - 1u) tb += bc7_texel_error2(sb, blk->rgb[popcount32((rb & (0u - rb)) - 1u)]);
    return Bc7Err2{ta, tb};
}
// Mode-1 (three-bit) and mode-3 (two-bit) errors of one two-subset shape, mask0 = its subset 0: a walk over subset 0's texels
// with its constants in registers, then one over subset 1's (the errors are exact integers, so the order of the sums does not
// matter).  Subset 1's constants are built after the first walk, so that only its four endpoint words are live across it.
// e1 / e3 = decoded endpoints A, B of subsets 0 and 1 for mode 1 / mode 3.
struct Bc7PairErr { int mode1, mode3; };
ITW_HD void bc7_subset_error13(Bc7PairErr& e, const Bc7Block* blk, u32 mask, u32 e1a, u32 e1b, u32 e3a, u32 e3b)
{
    const Bc7Sub3 s1 = bc7_sub3(e1a, e1b);
    const Bc7Sub2 s3 = bc7_sub2(e3a, e3b);
    const int n = popcount16(mask);
    u32 rest = mask;
    // unrolled so that the texel loads of several iterations are in flight at once (as bc7_masks_error2; 4 measured faster
    // than 2 or 8 on H100, and faster than walking both subsets in one loop)
#pragma unroll 4
    for (int i = 0; i < n; i++) {
        const u32 low = rest & (0u - rest);
        rest ^= low;
        const u32 t = blk->rgb[popcount32(low - 1u)];
        e.mode1 += bc7_texel_error3(s1, t);
        e.mode3 += bc7_texel_error2(s3, t);
    }
}
ITW_HD_NOINLINE Bc7PairErr bc7_pair_error(const Bc7Block* blk, u32 mask0, u32 e1a0, u32 e1b0, u32 e1a1, u32 e1b1, u32 e3a0,
                                          u32 e3b0, u32 e3a1, u32 e3b1)
{
    Bc7PairErr e{0, 0};
    bc7_subset_error13(e, blk, mask0, e1a0, e1b0, e3a0, e3b0);
    bc7_subset_error13(e, blk, ~mask0 & 0xFFFFu, e1a1, e1b1, e3a1, e3b1);
    return e;
}

// Least-squares endpoints of one subset from its indices; K:1198-1262.  The sums are exact integers.
// Components >= channels are zero.
ITW_HD u32 bc7_index_bytes(u32 idx0, u32 idx1, int i)                     // 4-bit indices of texels 4i..4i+3, one per byte
{
    u32 n = (((i < 2) ? idx0 : idx1) >> (16 * (i & 1))) & 0xFFFFu;
    n = (n | (n << 8)) & 0x00FF00FFu;
    return (n | (n << 4)) & 0x0F0F0F0Fu;
}
// The endpoints from the integer sums: count texels, sq1 = sum q, sqq = sum q^2, sum[c] = sum x_c, atb1[c] = sum (top - q) x_c
ITW_HD Bc7Seg bc7_solve_ends(u32 top, float count, u32 sq1, u32 sqq, const u32 (&sum)[4], const u32 (&atb1)[4], int channels)
{
    Bc7Seg seg;
    float (&ep)[8] = seg.v;
    const float ftop = (float)top;
    const float fsq1 = (float)sq1, fsqq = (float)sqq;
    float cxx = count * sq(ftop) - (2.0f * ftop) * fsq1 + fsqq;
    float cyy = fsqq;
    float cxy = ftop * fsq1 - fsqq;
    float det = cxx * cyy - cxy * cxy;
    float scale = ftop / det;
    bool flat = fabsf(det) < 0.001f;
    const float rcount = 1.0f / count;
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const float fs = (float)sum[c], fa1 = (float)atb1[c];
        float atb2 = ftop * fs - fa1;
        float a = (fa1 * cyy - atb2 * cxy) * scale;
        float b = (atb2 * cxx - fa1 * cxy) * scale;
        // integer sum / integer count (1..16): the exact FMA-corrected quotient (tests/test_exact_division.py); a plain
        // IEEE division would take its slow path for every zero sum
        if (flat) { a = div_by_rcp(fs, count, rcount); b = a; }
        const bool used = (c < 3 || channels == 4);
        ep[c] = used ? a : 0.0f;
        ep[4 + c] = used ? b : 0.0f;
    }
    return seg;
}
ITW_HD_NOINLINE Bc7Seg bc7_solve(const Bc7Block* blk, int rot, int alpha, int bits, u32 idx0, u32 idx1, u32 mask, int channels)
{
    const View v{blk, rot, alpha};
    const u32 top = (1u << bits) - 1u;
    u32 sq1 = 0u, sqq = 0u, sum[4] = {0u, 0u, 0u, 0u}, atb1[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const u32 n = bc7_index_bytes(idx0, idx1, i);
        const u32 bm = nibble_to_bytemask(mask >> (4 * i));
        const u32 qm = n & bm, ones = bm & 0x01010101u;
        const u32 xm = ((top * 0x01010101u) & bm) - qm;                    // (levels-1) - q, bytewise, no borrows
        sq1 = dp4a_u8(qm, 0x01010101u, sq1);
        sqq = dp4a_u8(qm, qm, sqq);
#pragma unroll
        for (int c = 0; c < 4; c++) {                           // channels >= 3; an unused fourth channel sums zeros
            const u32 p = (c < 3 || channels == 4) ? view_plane(v, c, i) : 0u;
            sum[c] = dp4a_u8(ones, p, sum[c]);
            atb1[c] = dp4a_u8(xm, p, atb1[c]);
        }
    }
    return bc7_solve_ends(top, (float)popcount16(mask & 0xFFFFu), sq1, sqq, sum, atb1, channels);
}

// ---------------------------------------------------------------------------------------------
// 128-bit layouts; K:1694-1964.  Q[j][0/1] = quantised endpoints A/B of subset j as RGBA bytes.
// ---------------------------------------------------------------------------------------------
ITW_HD u32 qcomp(u32 packed, int c) { return (packed >> (8 * c)) & 255u; }

ITW_HD void bc7_write_partitioned(u32* out, u32 (&Q)[3][2], u32 idx0, u32 idx1, int shape, int mode)
{
    const int bits = bc7_mode_bits(mode), pairs = bc7_pairs(mode), channels = (mode == 7) ? 4 : 3;
    const int half = (1 << bits) / 2;
    int flips = 0;
#pragma unroll
    for (int j = 0; j < 3; j++) {                               // anchor index MSB must be 0; K:1708-1733
        if (j >= pairs) continue;
        const int k0 = shape_anchor(shape, j);
        const int vv = (int)(((k0 < 8 ? idx0 : idx1) >> (4 * (k0 & 7))) & 15u);
        if (vv >= half) {
            const u32 t = Q[j][0]; Q[j][0] = Q[j][1]; Q[j][1] = t;
            flips |= shape_mask(shape, j);
        }
    }
    BitSink s;
    s.reset();
    s.put(mode + 1, 1u << mode);
    s.put(mode == 0 ? 4 : 6, (u32)(shape & (mode == 0 ? 15 : 63)));
    const int width = (mode == 0) ? 4 : ((mode == 1) ? 6 : ((mode == 3) ? 7 : 5));
    const int drop = (mode == 2) ? 0 : 1;                      // p-bit modes store the value without its LSB
    for (int c = 0; c < channels; c++) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (j >= pairs) continue;
            s.put(width, qcomp(Q[j][0], c) >> drop);
            s.put(width, qcomp(Q[j][1], c) >> drop);
        }
    }
    if (mode == 1) { s.put(1, Q[0][0] & 1u); s.put(1, Q[1][0] & 1u); }
    if (mode == 0 || mode == 3 || mode == 7) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (j >= pairs) continue;
            s.put(1, Q[j][0] & 1u);
            s.put(1, Q[j][1] & 1u);
        }
    }
    put_indices(s, idx0, idx1, bits, flips, shape_anchor(shape, 1), (pairs == 3) ? shape_anchor(shape, 2) : -1);
    out[0] = s.w0; out[1] = s.w1; out[2] = s.w2; out[3] = s.w3;
}
// single-subset orientation on packed endpoints; K:1694-1706
ITW_HD void orient_packed(u32& qa, u32& qb, u32& idx0, u32& idx1, int bits)
{
    const int levels = 1 << bits;
    if ((int)(idx0 & 15u) >= levels / 2) {
        const u32 t = qa; qa = qb; qb = t;
        const u32 all = 0x11111111u * (u32)(levels - 1);
        idx0 = all - idx0;
        idx1 = all - idx1;
    }
}
ITW_HD void bc7_write_mode45(u32* out, u32 qa, u32 qb, u32 i0, u32 i1, int aq0, int aq1, u32 a0, u32 a1, int mode,
                             int rotation, int swap)
{
    const int epbits = (mode == 4) ? 5 : 7, aepbits = (mode == 4) ? 6 : 8;
    const int cbits = 2, sbits = (mode == 4) ? 3 : 2;          // widths of the first / second index set
    int aq[2] = {aq0, aq1};
    if (!swap) {
        orient_packed(qa, qb, i0, i1, cbits);
        orient_single(aq, 1, a0, a1, sbits);
    } else {                                                    // the two index sets trade places; K:1903-1908
        u32 t0 = i0, t1 = i1;
        i0 = a0; i1 = a1;
        a0 = t0; a1 = t1;
        orient_single(aq, 1, i0, i1, cbits);
        orient_packed(qa, qb, a0, a1, sbits);
    }
    BitSink s;
    s.reset();
    s.put(mode + 1, 1u << mode);
    s.put(2, (u32)((rotation + 1) & 3));
    if (mode == 4) s.put(1, (u32)swap);
    for (int c = 0; c < 3; c++) { s.put(epbits, qcomp(qa, c)); s.put(epbits, qcomp(qb, c)); }
    s.put(aepbits, (u32)aq[0]);
    s.put(aepbits, (u32)aq[1]);
    put_indices(s, i0, i1, cbits, 0, -1, -1);
    put_indices(s, a0, a1, sbits, 0, -1, -1);
    out[0] = s.w0; out[1] = s.w1; out[2] = s.w2; out[3] = s.w3;
}
ITW_HD void bc7_write_mode6(u32* out, u32 qa, u32 qb, u32 i0, u32 i1)
{
    orient_packed(qa, qb, i0, i1, 4);
    BitSink s;
    s.reset();
    s.put(7, 64u);
    for (int c = 0; c < 4; c++) { s.put(7, qcomp(qa, c) >> 1); s.put(7, qcomp(qb, c) >> 1); }
    s.put(1, qa & 1u);
    s.put(1, qb & 1u);
    put_indices(s, i0, i1, 4, 0, -1, -1);
    out[0] = s.w0; out[1] = s.w1; out[2] = s.w2; out[3] = s.w3;
}

// ---------------------------------------------------------------------------------------------
// scalar channel of modes 4/5; K:1437-1563.  `a` = byte `shift/8` of the ORIGINAL texels.
// ---------------------------------------------------------------------------------------------
// After quantisation the two endpoints are integers, the texels are integers and the weights are
// integers, so the index search and the least-squares sums are exact integer arithmetic; the projection
// (x - e0)/(e1 - e0 + 0.001f) keeps the reference's float expression (K:1510) with the exact quotient
// (domain proved in tests/test_exact_division.py).
// The sixteen texels of the channel are the four packed words of its plane (pl[i] byte j = texel 4i+j); the palette
// (at most 8 byte-sized entries) is packed into one 64-bit register and read with a shift.
ITW_HD void scalar_quantise(int (&q)[2], int (&e)[2], const float (&ep)[2], int epbits)
{
    const int top = (1 << epbits) - 1;
#pragma unroll
    for (int i = 0; i < 2; i++) {
        q[i] = clampi(trunc_i(div255(ep[i]) * (float)top + 0.5f), 0, top);   // ep in [0,255]: no overflow
        e[i] = expand_bits(q[i], epbits);
    }
}
// The three scalar channels of a rotation (bc7_chain_rotation), side by side: role r has index bits scalar_bits(r), its
// endpoints e[r] and gets its indices in idx0[r], idx1[r] and its error in err[r].  One loop reads each plane word once.
ITW_HD int scalar_bits(int r) { return (r == 0) ? 3 : 2; }            // r = 0, 1, 2: mode 4 swap 0, mode 4 swap 1, mode 5
ITW_HD int scalar_epbits(int r) { return (r == 2) ? 8 : 6; }
ITW_HD void scalar_assign3(u32 (&idx0)[3], u32 (&idx1)[3], int (&err)[3], const u32 (&pl)[4], const int (&e)[3][2])
{
    float den[3], rden[3];
    unsigned long long pal[3];
    u32 out[3][2];
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const int bits = scalar_bits(r), levels = 1 << bits;
        den[r] = (float)(e[r][1] - e[r][0]) + 0.001f;
        rden[r] = 1.0f / den[r];
        pal[r] = 0ull;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int w = bc7_weight(bits, q);
            const u32 v = (q < levels) ? (u32)(((64 - w) * e[r][0] + w * e[r][1] + 32) >> 6) : 0u;
            pal[r] |= (unsigned long long)v << (8 * q);
        }
        out[r][0] = out[r][1] = 0u;
        err[r] = 0;
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
#pragma unroll 1
        for (int i = 0; i < 2; i++) {                          // one plane word = four texels per iteration
            const u32 word = i ? pl[2 * h + 1] : pl[2 * h];     // a select: pl[] indexed at run time would be local memory
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int a = (int)((word >> (8 * j)) & 255u);
#pragma unroll
                for (int r = 0; r < 3; r++) {
                    const int levels = 1 << scalar_bits(r);
                    const float proj = div_by_rcp((float)(a - e[r][0]), den[r], rden[r]);
                    const int q1 = clampi(trunc_i(fma_rn(proj, (float)levels, 0.5f)), 1, levels - 1);
                    const u32 two = (u32)(pal[r] >> (8 * (q1 - 1)));  // entries q1-1 and q1
                    const int d0 = (int)(two & 255u) - a, d1 = (int)((two >> 8) & 255u) - a;
                    const int err0 = d0 * d0, err1 = d1 * d1;
                    const bool first = err0 < err1;
                    err[r] += first ? err0 : err1;
                    out[r][h] += (u32)(first ? q1 - 1 : q1) << (16 * i + 4 * j);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 3; r++) { idx0[r] = out[r][0]; idx1[r] = out[r][1]; }
}
ITW_HD void scalar_solve(float (&ep)[2], const u32 (&pl)[4], int bits, u32 idx0, u32 idx1)
{
    const u32 utop = (1u << bits) - 1u;
    u32 usq1 = 0u, usqq = 0u, usum = 0u, uatb1 = 0u;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        u32 n = (((i < 2) ? idx0 : idx1) >> (16 * (i & 1))) & 0xFFFFu;     // four 4-bit indices ...
        n = (n | (n << 8)) & 0x00FF00FFu;
        n = (n | (n << 4)) & 0x0F0F0F0Fu;                                  // ... one per byte
        const u32 xm = utop * 0x01010101u - n;                             // (levels-1) - q, bytewise, no borrows
        usq1 = dp4a_u8(n, 0x01010101u, usq1);
        usqq = dp4a_u8(n, n, usqq);
        usum = dp4a_u8(pl[i], 0x01010101u, usum);
        uatb1 = dp4a_u8(xm, pl[i], uatb1);
    }
    const float top = (float)utop, atb1 = (float)uatb1, sq1 = (float)usq1, sqq = (float)usqq, sum = (float)usum;
    float atb2 = top * sum - atb1;
    float cxx = 16.0f * sq(top) - (2.0f * top) * sq1 + sqq;
    float cyy = sqq;
    float cxy = top * sq1 - sqq;
    float det = cxx * cyy - cxy * cxy;
    float scale = top / det;
    ep[0] = clamp_sse((atb1 * cyy - atb2 * cxy) * scale, 0.0f, 255.0f);
    ep[1] = clamp_sse((atb2 * cxx - atb1 * cxy) * scale, 0.0f, 255.0f);
    if (fabsf(det) < 0.001f) {
        ep[0] = sum * 0.0625f;                                             // sum / 16, exact
        ep[1] = ep[0];
    }
}
// The scalar channels of mode 4 with swap 0 and 1 and of mode 5 at one rotation: one plane read and one min/max (K:1542-1548)
// serve all three, the first quantisation of the two mode-4 roles is the same, and the refinements run side by side.  cerr
// = the errors of the three roles' colour channels; returns the role r (0, 1, 2 as scalar_bits) whose summed error is the
// first strict minimum, that error and r's scalar channel.
struct Bc7Scalar { int r, err, q0, q1; u32 idx0, idx1; };
ITW_HD_NOINLINE Bc7Scalar bc7_scalar_rotation(const Bc7Block* blk, int rotation, int rch, int cerr0, int cerr1, int cerr2)
{
    u32 pl[4];
#pragma unroll
    for (int i = 0; i < 4; i++) pl[i] = blk->plane[rotation][i];
    int lo = 255, hi = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int a = (int)((pl[i] >> (8 * j)) & 255u);
            lo = mini(lo, a);
            hi = maxi(hi, a);
        }
    float ep[3][2];
    int q[3][2], e[3][2], err[3];
    u32 idx0[3], idx1[3];
    ep[0][0] = (float)lo; ep[0][1] = (float)hi;
    scalar_quantise(q[0], e[0], ep[0], scalar_epbits(0));
    scalar_quantise(q[2], e[2], ep[0], scalar_epbits(2));
#pragma unroll
    for (int i = 0; i < 2; i++) { q[1][i] = q[0][i]; e[1][i] = e[0][i]; }
    scalar_assign3(idx0, idx1, err, pl, e);
#pragma unroll 1
    for (int it = 0; it < rch; it++) {
#pragma unroll
        for (int r = 0; r < 3; r++) {
            scalar_solve(ep[r], pl, scalar_bits(r), idx0[r], idx1[r]);
            scalar_quantise(q[r], e[r], ep[r], scalar_epbits(r));
        }
        scalar_assign3(idx0, idx1, err, pl, e);
    }
    const int t0 = cerr0 + err[0], t1 = cerr1 + err[1], t2 = cerr2 + err[2];
    Bc7Scalar s{0, t0, q[0][0], q[0][1], idx0[0], idx1[0]};
    if (t1 < s.err) s = Bc7Scalar{1, t1, q[1][0], q[1][1], idx0[1], idx1[1]};
    if (t2 < s.err) s = Bc7Scalar{2, t2, q[2][0], q[2][1], idx0[2], idx1[2]};
    return s;
}

// ---------------------------------------------------------------------------------------------
// The chains: initial fit + refinement + encode of one (block, role).  Roles r = 0..4 are the mode slots (modes 0, 2, 1, 3,
// 7), then mode 4 by (rotation, swap), mode 5 by rotation, mode 6: the reference's order, which decides ties.  The chain
// phase runs them in UNITS, one routine each: a partitioned mode (K:1299-1363: modes 0-3, 7), a rotation (K:1565-1655: the
// roles of modes 4 and 5 at one rotation) and mode 6 (K:1657-1689).  Units u = 0..4 are the mode slots, then one per
// rotation, then mode 6.
// ---------------------------------------------------------------------------------------------
ITW_HD int bc7_rotations(const Bc7Params& P) { return P.sel[2] ? maxi(P.channels - P.ch0, 0) : 0; }
ITW_HD int bc7_unit_count(const Bc7Params& P) { return 5 + bc7_rotations(P) + (P.sel[3] ? 1 : 0); }
// The chain phase walks only the units that can produce a candidate: a partitioned mode whose list is empty under the profile
// (mode 7 of the RGB profiles, ...) would otherwise idle one lane of every pass.
ITW_HD int bc7_active_units(const Bc7Params& P)
{
    int n = bc7_unit_count(P) - 5;
    for (int m = 0; m < 5; m++) n += (bc7_slot_count(P, m) > 0) ? 1 : 0;
    return n;
}
// i-th active unit in RUN order, which groups units that take the same routine, so that the two units of a sixteen-block
// pass match: the partitioned modes (0, 2, 1, 3, 7), then the rotations and mode 6.  When the partitioned units are odd in
// number, the last of them shares a pass with a one-subset unit anyway; mode 6 takes that place, so that the rotations
// after it stay paired.
ITW_HD int bc7_active_unit(const Bc7Params& P, int i)
{
    int nparts = 0;
    for (int m = 0; m < 5; m++)
        if (bc7_slot_count(P, m) > 0) { if (i == 0) return m; i--; nparts++; }
    const int nrot = bc7_rotations(P), six = 5 + nrot;
    if (P.sel[3] && (nparts & 1)) { if (i == 0) return six; i--; }
    return (i < nrot) ? 5 + i : six;                             // mode 6, when not placed above
}
ITW_HD const Bc7Block* bc7_chain_block(const Bc7Warp& W, int slot)
{
    return (slot < W.nparked) ? &W.parked[slot] : &W.blk[slot - W.nparked];
}

// the best candidate of a unit: its error, role number and 128 bits
struct Bc7Result { int err, role; u32 code[4]; };
// Partitioned roles r = 0..4: the winning shape of mode slot r, identity view.
ITW_HD_NOINLINE Bc7Result bc7_chain_parts(Bc7Warp& W, const Bc7Params& P, int lane, int slot, int r)
{
    Bc7Result res;
    res.err = kErrNone;
    res.role = r;
    res.code[0] = res.code[1] = res.code[2] = res.code[3] = 0u;
    const int shape = W.win_shape[slot][r];
    if (shape < 0) return res;
    const Bc7Block* blk = bc7_chain_block(W, slot);
    const int mode = bc7_slot_mode(r);
    const int pairs = bc7_pairs(mode), bits = bc7_mode_bits(mode);
    // channels fitted / searched, and the count that votes on p-bits during refinement (K:1343)
    const int channels = (mode == 7) ? 4 : 3;
    const u32 chmask = (channels == 4) ? 0xFFFFFFFFu : 0x00FFFFFFu;
    const int alpha = (P.channels == 4) ? 1 : 0;
    const u32 pattern = shape_pattern(shape);

    u32 ends[6], Q[3][2];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        Q[j][0] = Q[j][1] = 0u;
        ends[2 * j] = ends[2 * j + 1] = 0u;
    }
#pragma unroll
    for (int j = 0; j < 3; j++) {
        if (j >= pairs) continue;
        const Bc7Seg seg = bc7_fit(blk, 3, alpha, (u32)shape_mask(shape, j), channels);   // slots >= channels are zero (F6)
        const Bc7Packed pk = bc7_quantise(seg, mode, channels);
        ends[2 * j] = pk.dec_a; ends[2 * j + 1] = pk.dec_b;
        Q[j][0] = pk.q_a; Q[j][1] = pk.q_b;
    }
    Bc7Search best = bc7_assign(W.palette, lane, blk, 3, alpha, bits, pairs, pattern, ends[0], ends[1], ends[2], ends[3], ends[4],
                                ends[5], chmask);

    const int refine = P.refine[mode];
    for (int it = 0; it < refine; it++) {
        u32 nQ[3][2];
#pragma unroll
        for (int j = 0; j < 3; j++) nQ[j][0] = nQ[j][1] = 0u;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (j >= pairs) continue;
            const Bc7Seg seg = bc7_solve(blk, 3, alpha, bits, best.idx0, best.idx1, (u32)shape_mask(shape, j), channels);
            const Bc7Packed pk = bc7_quantise(seg, mode, P.channels);
            ends[2 * j] = pk.dec_a; ends[2 * j + 1] = pk.dec_b;
            nQ[j][0] = pk.q_a; nQ[j][1] = pk.q_b;
        }
        const Bc7Search found = bc7_assign(W.palette, lane, blk, 3, alpha, bits, pairs, pattern, ends[0], ends[1], ends[2], ends[3],
                                           ends[4], ends[5], chmask);
        // the best iterate is kept (K:1348)
        if (found.err < best.err) {
#pragma unroll
            for (int j = 0; j < 3; j++) { Q[j][0] = nQ[j][0]; Q[j][1] = nQ[j][1]; }
            best = found;
        }
    }
    int best_err = best.err;
    if (mode != 7 && P.channels != 3) {                           // opaque error of the dropped alpha; K:1267-1277, :1356
        int opaque = 0;
        for (int k = 0; k < 16; k++) { const int d = (int)(blk->tex[k] >> 24) - 255; opaque += d * d; }
        best_err += opaque;
    }
    bc7_write_partitioned(res.code, Q, best.idx0, best.idx1, shape, mode);
    res.err = best_err;
    return res;
}
// The roles of modes 4 and 5 at one rotation (mode 4 with index swap 0 and 1, mode 5; three channels, all sixteen texels,
// the view rotated unless the rotation is 3, alpha with itself).  The three share one fit, the two mode-4 roles their first
// quantisation, and each step of the refinement holds one solve, quantisation and search per role as independent code: the
// plane sums of the solve are index-free and taken once per step for all three roles (held across the steps they added 4
// bytes of kernel spills), and one walk over the texels searches all three (bc7_assign_rotation).  Rule F6 and the carried fourth slot (quirk Q5) apply to each role separately.
// The steps are non-inlined routines that exchange the three roles' state BY VALUE: their quantised endpoints (the decoded
// ones, and with them the carried fourth slot, follow from those) and their searches.  Nothing else is live across a step,
// so the chain's call does not raise the registers the chain phase needs around it: with the search as the only call
// inside the refinement loop, the kernel spilled 112 / 132 bytes instead of 16 / 12 (-Xptxas -v).
struct Bc7RotState { u32 q[3][2]; Bc7Search3 best; };
ITW_HD int bc7_rotation_bits(int r) { return (r == 2) ? 7 : 5; }    // stored bits per component, modes 4 and 5
// the three searches from quantised endpoints
ITW_HD Bc7Search3 bc7_rotation_search(const View& v, const u32 (&q)[3][2])
{
    u32 dec[3][2];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int i = 0; i < 2; i++) dec[r][i] = bc7_decode_packed(q[r][i], bc7_rotation_bits(r));
    return bc7_assign_rotation(v, dec[0][0], dec[0][1], dec[1][0], dec[1][1], dec[2][0], dec[2][1]);
}
// fit, first quantisations, first searches
ITW_HD_NOINLINE Bc7RotState bc7_rotation_start(const Bc7Block* blk, int rot, int alpha)
{
    const Bc7Seg seg = bc7_fit_full(blk, rot, alpha, 3);        // slots >= 3 are zero (F6)
    const Bc7Packed p4 = bc7_quantise_impl(seg, 4, 3), p5 = bc7_quantise_impl(seg, 5, 3);
    Bc7RotState st;
    st.q[0][0] = st.q[1][0] = p4.q_a; st.q[0][1] = st.q[1][1] = p4.q_b;
    st.q[2][0] = p5.q_a; st.q[2][1] = p5.q_b;
    st.best = bc7_rotation_search(View{blk, rot, alpha}, st.q);
    return st;
}
// One refinement step of the roles whose refinement is not over (do4: both mode-4 roles, do5: mode 5); the others keep their
// state.  s0..s2 = the channel sums of the solve (K:1198-1230), index-free.
ITW_HD_NOINLINE Bc7RotState bc7_rotation_refine(const Bc7Block* blk, int rot, int alpha, Bc7RotState st, bool do4, bool do5)
{
    const View v{blk, rot, alpha};
    u32 sum[4] = {0u, 0u, 0u, 0u}, sq1[3] = {0u, 0u, 0u}, sqq[3] = {0u, 0u, 0u}, atb1[3][4];
#pragma unroll
    for (int r = 0; r < 3; r++) atb1[r][0] = atb1[r][1] = atb1[r][2] = atb1[r][3] = 0u;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        u32 p[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            p[c] = view_plane(v, c, i);
            sum[c] = dp4a_u8(0x01010101u, p[c], sum[c]);
        }
#pragma unroll
        for (int r = 0; r < 3; r++) {
            const u32 top = (r == 1) ? 7u : 3u;                  // index bits 2, 3, 2
            const u32 n = bc7_index_bytes(st.best.s[r].idx0, st.best.s[r].idx1, i);
            const u32 xm = top * 0x01010101u - n;                // (levels-1) - q, bytewise, no borrows
            sq1[r] = dp4a_u8(n, 0x01010101u, sq1[r]);
            sqq[r] = dp4a_u8(n, n, sqq[r]);
#pragma unroll
            for (int c = 0; c < 3; c++) atb1[r][c] = dp4a_u8(xm, p[c], atb1[r][c]);
        }
    }
    Bc7RotState nst;
#pragma unroll
    for (int r = 0; r < 3; r++) {
        Bc7Seg seg = bc7_solve_ends((r == 1) ? 7u : 3u, 16.0f, sq1[r], sqq[r], sum, atb1[r], 3);
        // ep[3], ep[7] are carried between iterations (quirk Q5): a fourth slot the solve does not write keeps the previous
        // iteration's decoded value
        seg.v[3] = (float)(bc7_decode_packed(st.q[r][0], bc7_rotation_bits(r)) >> 24);
        seg.v[7] = (float)(bc7_decode_packed(st.q[r][1], bc7_rotation_bits(r)) >> 24);
        const Bc7Packed pk = bc7_quantise_impl(seg, (r == 2) ? 5 : 4, 3);
        nst.q[r][0] = pk.q_a;
        nst.q[r][1] = pk.q_b;
    }
    nst.best = bc7_rotation_search(v, nst.q);
    // the last iterate is kept (K:1598-1603)
#pragma unroll
    for (int r = 0; r < 3; r++)
        if (!((r == 2) ? do5 : do4)) { nst.q[r][0] = st.q[r][0]; nst.q[r][1] = st.q[r][1]; nst.best.s[r] = st.best.s[r]; }
    return nst;
}
// The scalar channels (bc7_scalar_rotation), then the 128 bits of the best of the three roles: mode 4 with swap 0 and 1 are
// roles r4 and r4 + 1, mode 5 is role r5 (r4 < r4 + 1 < r5).
ITW_HD_NOINLINE Bc7Result bc7_rotation_finish(const Bc7Block* blk, int rotation, int rch, int r4, int r5, Bc7RotState st)
{
    const Bc7Scalar sc = bc7_scalar_rotation(blk, rotation, rch, st.best.s[0].err, st.best.s[1].err, st.best.s[2].err);
    const int w = sc.r;
    const u32 qa = (w == 0) ? st.q[0][0] : ((w == 1) ? st.q[1][0] : st.q[2][0]);
    const u32 qb = (w == 0) ? st.q[0][1] : ((w == 1) ? st.q[1][1] : st.q[2][1]);
    const Bc7Search s = (w == 0) ? st.best.s[0] : ((w == 1) ? st.best.s[1] : st.best.s[2]);
    Bc7Result res;
    res.err = sc.err;
    res.role = (w == 2) ? r5 : r4 + w;
    bc7_write_mode45(res.code, qa, qb, s.idx0, s.idx1, sc.q0, sc.q1, sc.idx0, sc.idx1, (w == 2) ? 5 : 4, rotation, (w == 1) ? 1 : 0);
    return res;
}
// One rotation (0..3) of a block; n4, n5 = refinement steps of modes 4 and 5, rch = of the scalar channel; roles as in
// bc7_rotation_finish.  Takes the profile's values by value: a Bc7Params by reference is read from local memory.  Returns
// the best candidate of the three, the minimum of (error, role).
ITW_HD_NOINLINE Bc7Result bc7_chain_rotation(const Bc7Block* blk, int rotation, int alpha, int n4, int n5, int rch, int r4, int r5)
{
    const int rot = (rotation < 3) ? rotation : 3;              // rotation 3 (alpha "with itself") is the identity
    Bc7RotState st = bc7_rotation_start(blk, rot, alpha);
#pragma unroll 1
    for (int it = 0; it < maxi(n4, n5); it++) st = bc7_rotation_refine(blk, rot, alpha, st, it < n4, it < n5);
    return bc7_rotation_finish(blk, rotation, rch, r4, r5, st);
}
// Mode 6 (role 5 + 3 nrot): all sixteen texels and the profile's channels, identity view.
ITW_HD_NOINLINE Bc7Result bc7_chain_mode6(Bc7Warp& W, const Bc7Params& P, int lane, int slot)
{
    const Bc7Block* blk = bc7_chain_block(W, slot);
    const int channels = P.channels;                            // fitted, searched and voting (K:1657-1689)
    const u32 chmask = (channels == 4) ? 0xFFFFFFFFu : 0x00FFFFFFu;
    const int alpha = (P.channels == 4) ? 1 : 0;

    Bc7Seg seg = bc7_fit_full(blk, 3, alpha, channels);         // slots >= channels are zero (F6)
    if (channels == 3) seg.v[3] = seg.v[7] = 255.0f;            // K:1664-1667
    Bc7Packed pk = (channels == 4) ? bc7_quantise_m<6, 4>(seg) : bc7_quantise_m<6, 3>(seg);
    // ep[3], ep[7] are carried between iterations (quirk Q5), as in bc7_chain_rotation
    float tail_a = (float)(pk.dec_a >> 24), tail_b = (float)(pk.dec_b >> 24);
    Bc7Search best = bc7_assign_one(W.palette, lane, blk, pk.dec_a, pk.dec_b, chmask);
    const int refine = P.refine[6];
    for (int it = 0; it < refine; it++) {
        Bc7Seg s = bc7_solve(blk, 3, alpha, 4, best.idx0, best.idx1, 0xFFFFu, channels);
        if (channels < 4) { s.v[3] = tail_a; s.v[7] = tail_b; }
        pk = (channels == 4) ? bc7_quantise_m<6, 4>(s) : bc7_quantise_m<6, 3>(s);
        tail_a = (float)(pk.dec_a >> 24); tail_b = (float)(pk.dec_b >> 24);
        // the last iterate is kept (K:1677-1682)
        best = bc7_assign_one(W.palette, lane, blk, pk.dec_a, pk.dec_b, chmask);
    }
    Bc7Result res;
    res.err = best.err;
    res.role = 5 + 3 * bc7_rotations(P);
    bc7_write_mode6(res.code, pk.q_a, pk.q_b, best.idx0, best.idx1);
    return res;
}

// One call site in the chain phase: the kernel body around it allocates its registers as for a single callee.
ITW_HD_NOINLINE Bc7Result bc7_chain(Bc7Warp& W, const Bc7Params& P, int lane, int slot, int u)
{
    if (u < 5) return bc7_chain_parts(W, P, lane, slot, u);
    const int nrot = bc7_rotations(P), k = u - 5;
    if (k < nrot)
        return bc7_chain_rotation(bc7_chain_block(W, slot), P.ch0 + k, (P.channels == 4) ? 1 : 0, P.refine[4], P.refine[5], P.rch,
                                  5 + 2 * k, 5 + 2 * nrot + k);
    return bc7_chain_mode6(W, P, lane, slot);
}

// =============================================================================================
// Warp program: per-lane phase functions.  A phase reads what earlier phases wrote to W and
// writes disjoint locations; the caller separates phases with a warp barrier.
// =============================================================================================
ITW_HD int bc7_group_count(const Bc7Warp& W, int g) { return mini(maxi(W.nvalid - kBc7Slots * g, 0), kBc7Slots); }   // valid blocks of group g

// texel k (RGBA8) of block `id` of a surface, blocks in row-major order
ITW_HD const uint8_t* bc7_texel_ptr(const SurfaceView& s, long long id, int k)
{
    const int bw = s.width >> 2;
    const int by = (int)(id / bw), bx = (int)(id - (long long)by * bw);
    return s.ptr + (size_t)(by * 4 + (k >> 2)) * (size_t)s.stride + (size_t)(bx * 4 + (k & 3)) * 4;
}
// texel k of block `id` of a surface into b.rgb[k] and b.tex[k]
ITW_HD void bc7_fetch_texel(Bc7Block& b, const SurfaceView& s, long long id, int k)
{
    const uint8_t* p = bc7_texel_ptr(s, id, k);
    const u32 rgb = (u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16);
    b.rgb[k] = rgb;
    b.tex[k] = rgb | ((u32)p[3] << 24);
}
// Loads half `half` (blocks 8*half .. 8*half+7 of the round's `ntotal`) into blk[].
ITW_HD void bc7_phase_load(int lane, Bc7Warp& W, const SurfaceView& s, long long first_block, int ntotal, int half)
{
    const int nvalid = mini(maxi(ntotal - kBc7Batch * half, 0), kBc7Batch);
    for (int t = lane; t < nvalid * 16; t += 32) {
        const int slot = t >> 4;
        bc7_fetch_texel(W.blk[slot], s, first_block + kBc7Batch * half + slot, t & 15);
    }
    if (lane == 0) { W.nvalid = nvalid; W.half = half; W.ntotal = ntotal; W.nparked = 0; }
    for (int t = lane; t < kBc7Batch * 5; t += 32) W.win_shape[kBc7Batch * half + t / 5][t % 5] = -1;
}
// After the shape phases of the second half: the first half is read again (texels and channel planes) for the chain phase.
// The plane words are read here too: a transpose after a barrier (bc7_phase_planes) would add a phase.
ITW_HD void bc7_phase_park(int lane, Bc7Warp& W, const SurfaceView& s, long long first_block, int ntotal)
{
    if (ntotal <= kBc7Batch) return;                       // single-half round: blk[] still holds it
    for (int t = lane; t < kBc7Batch * 16; t += 32) {
        const int slot = t >> 4, k = t & 15;
        const long long id = first_block + slot;
        bc7_fetch_texel(W.parked[slot], s, id, k);
        // plane word (c, i) = channel c of texels 4i..4i+3: here c = k & 3, i = k >> 2 (any bijection of 16 onto (c, i) does)
        const int c = k & 3, i = k >> 2;
        u32 v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) v |= (u32)bc7_texel_ptr(s, id, 4 * i + j)[c] << (8 * j);
        W.parked[slot].plane[c][i] = v;
    }
    if (lane == 0) W.nparked = kBc7Batch;
}
// channel planes from the packed texels (a 4x4 byte transpose per group of four texels)
ITW_HD void bc7_phase_planes(int lane, Bc7Warp& W)
{
    for (int t = lane; t < W.nvalid * 16; t += 32) {
        const int slot = t >> 4, c = (t >> 2) & 3, i = t & 3;
        const u32* x = &W.blk[slot].tex[4 * i];
        u32 v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) v |= ((x[j] >> (8 * c)) & 255u) << (8 * j);
        W.blk[slot].plane[c][i] = v;
    }
}
// One two-subset shape, both modes of a mode-slot pair (ma, mb) -- modes 1 and 3, or mode 7: fits once, quantises and searches
// per mode.  `slot` = position inside the group (scratch index), `blk` = the block.
ITW_HD_NOINLINE void bc7_eval_shape(Bc7Warp& W, int lane, int slot, const Bc7Block* blk, int shape, int n, int ma, bool do_a, int mb, bool do_b)
{
    const int mode_a = bc7_slot_mode(ma), mode_b = bc7_slot_mode(mb);
    const int pairs = 2;
    const int channels = (mode_a == 7) ? 4 : 3;
    const u32 chmask = (channels == 4) ? 0xFFFFFFFFu : 0x00FFFFFFu;
    u32 ends_a[6], ends_b[6];
#pragma unroll
    for (int i = 0; i < 6; i++) ends_a[i] = ends_b[i] = 0u;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        const Bc7Seg seg = bc7_fit(blk, 3, 1, (u32)shape_mask(shape, j), channels);
        if (do_a) {
            const Bc7Packed pk = bc7_quantise(seg, mode_a, channels);
            ends_a[2 * j] = pk.dec_a; ends_a[2 * j + 1] = pk.dec_b;
        }
        if (do_b) {
            const Bc7Packed pk = bc7_quantise(seg, mode_b, channels);
            ends_b[2 * j] = pk.dec_a; ends_b[2 * j + 1] = pk.dec_b;
        }
    }
    const u32 pattern = shape_pattern(shape);
    if (do_a)
        W.cand_err[slot][0][n] = bc7_assign(W.palette, lane, blk, 3, 1, bc7_mode_bits(mode_a) | kAssignThresholds, pairs, pattern, ends_a[0], ends_a[1], ends_a[2],
                                            ends_a[3], ends_a[4], ends_a[5], chmask).err;
    if (do_b)
        W.cand_err[slot][1][n] = bc7_assign(W.palette, lane, blk, 3, 1, bc7_mode_bits(mode_b) | kAssignThresholds, pairs, pattern, ends_b[0], ends_b[1], ends_b[2],
                                            ends_b[3], ends_b[4], ends_b[5], chmask).err;
}
// ---- three-subset shapes (modes 0 and 2) -------------------------------------------------------------------
// The 64 shapes x 3 subsets use only 140 distinct texel masks, and the PCA fit, the endpoint quantisation and the index-search
// error of a subset depend on its mask alone (the reference refits per shape and per mode with identical results,
// K:1279-1297).  So, for the four blocks of group g: phase A fits and quantises every distinct mask once and searches it for
// mode 2, two masks of one block per lane (lane <-> (block, lane pair of itw_masks3.cuh): bc7_fit_masks2 and
// bc7_masks_error2 run two independent chains each); phase B adds up the mode-2 errors of every shape's three masks and
// runs the mode-0 search of shapes 0..15 from the stored endpoints (lane <-> (block, shape)).  Same values as evaluating
// shape by shape: 25 % fewer fits and quantisations, 27 % fewer mode-2 texels searched.  Mode 0 stays per shape: its 36
// masks per block take several passes of short, divergent subset loops where its 16 shapes per block fill a dense pass, and
// that measured slower on the profiles that skip mode 2 (basic).
ITW_HD void bc7_phase_masks3(int lane, Bc7Warp& W, const Bc7Params& P, int g)
{
    const int ca = bc7_slot_count(P, 0), cb = bc7_slot_count(P, 1);
    const int npairs = ((cb > 0) ? ITW_MASK3_COUNT : ITW_MASK3_FIRST) / 2;
    const int nv = bc7_group_count(W, g);
    for (int t = lane; t < nv * npairs; t += 32) {
        // the blocks alternate, so that a step holds eight lane pairs of similar popcount
        const int slot = t % nv, u = 2 * (t / nv);
        const Bc7Block* blk = &W.blk[kBc7Slots * g + slot];
        const u32 mask_a = ITW_TABLE(mask3_unique)[u], mask_b = ITW_TABLE(mask3_unique)[u + 1];
        const Bc7Segs2 f = bc7_fit_masks2(blk, mask_a, mask_b);
        // every quantisation before the search, so that the two fits are dead across it
        if (ca > 0 && u < ITW_MASK3_FIRST) {                       // ITW_MASK3_FIRST is even: both masks or neither
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const Bc7Packed pk = bc7_quantise_m<0, 3>(f.seg[j]);
                W.masks3.ends0[slot][u + j][0] = pk.dec_a;
                W.masks3.ends0[slot][u + j][1] = pk.dec_b;
            }
        }
        if (cb > 0) {
            const Bc7Packed pa = bc7_quantise_m<2, 3>(f.seg[0]), pb = bc7_quantise_m<2, 3>(f.seg[1]);
            const Bc7Err2 e = bc7_masks_error2(blk, mask_a, mask_b, pa.dec_a, pa.dec_b, pb.dec_a, pb.dec_b);
            W.masks3.err2[slot][u] = e.a;
            W.masks3.err2[slot][u + 1] = e.b;
        }
    }
}
// Tasks [0, nv * ca) are block-major (slot, shape n < ca): the mode-0 searches fill whole steps; the tasks after them only add
// up the mode-2 errors of shapes [ca, cb).
ITW_HD void bc7_phase_shapes3(int lane, Bc7Warp& W, const Bc7Params& P, int g)
{
    const int ca = bc7_slot_count(P, 0), cb = bc7_slot_count(P, 1);
    const int nv = bc7_group_count(W, g);
    const int nfirst = nv * ca, rest = maxi(cb - ca, 0);
    for (int t = lane; t < nfirst + nv * rest; t += 32) {
        int slot, n;
        if (t < nfirst) { slot = t / ca; n = t - slot * ca; }
        else { const int u = t - nfirst; slot = u / rest; n = ca + (u - slot * rest); }
        const int u0 = ITW_TABLE(shape3_mask_id)[3 * n], u1 = ITW_TABLE(shape3_mask_id)[3 * n + 1], u2 = ITW_TABLE(shape3_mask_id)[3 * n + 2];
        if (n < ca) {
            const u32 (&e)[ITW_MASK3_FIRST][2] = W.masks3.ends0[slot];
            W.cand_err[slot][0][n] = bc7_assign(W.palette, lane, &W.blk[kBc7Slots * g + slot], 3, 1, 3, 3, shape_pattern(64 + n), e[u0][0],
                                                e[u0][1], e[u1][0], e[u1][1], e[u2][0], e[u2][1], 0x00FFFFFFu).err;
        }
        if (n < cb) W.cand_err[slot][1][n] = W.masks3.err2[slot][u0] + W.masks3.err2[slot][u1] + W.masks3.err2[slot][u2];
    }
}

// shapes of a pair of mode slots that walk the same list, for group g: (2,3) ranked two-subset, (4,4) mode 7
ITW_HD void bc7_phase_shapes(int lane, Bc7Warp& W, const Bc7Params& P, int g, int ma, int mb)
{
    const int ca = bc7_slot_count(P, ma), cb = (mb != ma) ? bc7_slot_count(P, mb) : 0;
    const int both = mini(ca, cb), count = maxi(ca, cb);
    // list positions [0, both) run both modes, [both, count) only the longer list's mode; tasks are ordered
    // so that the "both" positions of all blocks come first and a warp never mixes the two kinds
    const int nv = bc7_group_count(W, g);
    const int nboth = nv * both, nall = nv * count;
    for (int t = lane; t < nall; t += 32) {
        int slot, n;
        if (t < nboth) { slot = t / both; n = t - slot * both; }
        else { const int u = t - nboth, rest = count - both; slot = u / rest; n = both + (u - slot * rest); }
        bc7_eval_shape(W, lane, slot, &W.blk[kBc7Slots * g + slot], bc7_slot_shape(W, P, slot, ma, n), n, ma, n < ca, mb, n < cb);
    }
}
// split-bound keys of the 64 two-subset shapes; set 0 = RGB (modes 1,3), set 1 = profile channels (mode 7)
ITW_HD bool bc7_needs_keys(const Bc7Params& P, int set)
{
    if (!P.sel[1]) return false;
    return set == 0 ? !(P.t1 == 0 && P.t3 == 0) : (P.t7 != 0);
}
ITW_HD void bc7_phase_keys(int lane, Bc7Warp& W, const Bc7Params& P, int g, int set)
{
    const int channels = (set == 0) ? 3 : P.channels;
    for (int t = lane; t < bc7_group_count(W, g) * 64; t += 32) {
        const int slot = t >> 6, shape = t & 63;
        W.two.keys[slot][shape] = bc7_split_key(&W.blk[kBc7Slots * g + slot], shape, channels);
    }
}
// ---- full two-subset lists (modes 1 and 3) ----------------------------------------------------------------------------
// When the longer list holds all 64 shapes (max(t1, t3) = 64: the slow profiles), every shape is fitted and searched anyway
// and the ranking only decides ties (the winner is the first minimum in ranked order).  Then lane <-> (block, shape) over the
// whole group: one pair fit (whose first four power iterations give both split bounds, hence the key), quantisation of both
// subsets for modes 1 and 3 (bc7_quantise13: one call per subset, constants folded), and one walk over each subset's texels
// for both modes' errors.  Shorter lists (basic: 12 and 8 shapes)
// rank first and then evaluate only the top t shapes (bc7_phase_keys, bc7_phase_shapes), far fewer fits than all 64.
ITW_HD bool bc7_full_two(const Bc7Params& P) { return P.sel[1] && maxi(P.t1, P.t3) == 64; }
ITW_HD void bc7_phase_two_full(int lane, Bc7Warp& W, const Bc7Params& P, int g)
{
    const int nv = bc7_group_count(W, g);
    for (int t = lane; t < nv * 64; t += 32) {
        // the blocks alternate and the shapes come in popcount order, so that a step holds 8 shapes of similar popcount and
        // the lanes' subset walks are of similar length; results stay keyed by shape id
        const int slot = t % nv, shape = ITW_TABLE(shape2_order)[t / nv];
        const Bc7Block* blk = &W.blk[kBc7Slots * g + slot];
        const u32 mask0 = (u32)shape_mask(shape, 0);
        const Bc7Pair f = bc7_fit_pair(blk, mask0, 3);
        // both modes are always quantised and scored; a list the profile leaves empty is not stored
        const Bc7Packed13 q0 = bc7_quantise13(f.seg[0]), q1 = bc7_quantise13(f.seg[1]);
        const Bc7PairErr e = bc7_pair_error(blk, mask0, q0.m1.dec_a, q0.m1.dec_b, q1.m1.dec_a, q1.m1.dec_b, q0.m3.dec_a,
                                            q0.m3.dec_b, q1.m3.dec_a, q1.m3.dec_b);
        if (P.t1 > 0) W.cand_err[slot][0][shape] = e.mode1;
        if (P.t3 > 0) W.cand_err[slot][1][shape] = e.mode3;
        W.two.keys[slot][shape] = bc7_key_of(shape, f.bound[0], f.bound[1]);
    }
}
// The ranking decides which shapes a list of 0 < t < 64 entries holds; a list of all 64 is walked in shape order instead.
ITW_HD bool bc7_needs_rank(const Bc7Params& P, int set)
{
    for (int m = set ? 4 : 2; m <= (set ? 4 : 3); m++)
        if (bc7_slot_count(P, m) > 0 && bc7_slot_count(P, m) < 64) return true;
    return false;
}
ITW_HD void bc7_phase_rank(int lane, Bc7Warp& W, int g, int set)
{
    for (int t = lane; t < bc7_group_count(W, g) * 64; t += 32) {
        const int slot = t >> 6, i = t & 63;
        W.order[slot][set][rank_of(W.two.keys[slot], 64, i)] = (uint8_t)(W.two.keys[slot][i] & 63);
    }
}
// Winners of lists that hold all 64 two-subset shapes (and of a short list evaluated next to such a list), for mode slots
// (ma, mb) of group g: the first minimum in list order; K:1320
// (strict <, so an error of kErrNone never wins and an empty list gives -1).  That is the minimum of (error, tie), where the tie
// is the list position, or the ranking key for a list in shape order (bc7_shape_order; keys compare as signed ints, as in
// rank_of).  by_shape: the errors are stored by shape id, not by list position (bc7_phase_two_full).
// Two phases: bc7_phase_strips, lane <-> (block, list, strip of 16 entries), then bc7_phase_winners, lane <-> (block, list),
// which combines the four strips.  The strip routine is not inlined (inlined into the kernel, it made bc7_chain spill 72 bytes
// instead of 4, -Xptxas -v) and takes the list lengths by value (a Bc7Params by reference would be read from local memory).
ITW_HD_NOINLINE void bc7_strips(int lane, Bc7Warp& W, int g, int nm, int ca, int cb, bool two, bool by_shape)
{
    for (int t = lane; t < bc7_group_count(W, g) * nm * kBc7Strips; t += 32) {
        const int strip = t % kBc7Strips, list = t / kBc7Strips, slot = list / nm, which = list - slot * nm;
        const int count = which ? cb : ca;
        const bool keyed = two && count == 64;                        // bc7_shape_order
        const bool ranked = by_shape && !keyed;                       // errors by shape id, entries in ranked order
        const int* err = W.cand_err[slot][which];
        int best = -1, best_err = kErrNone, best_tie = 0;
        // the lanes of a strip parity start at 16 different entries: entry n of (slot, which, strip) lies in bank
        // (16 strip + n) % 32 of cand_err and of the keys, so reading the strips in step was a 16-way bank conflict.  The
        // comparison is on (error, tie), so the order of the walk does not matter.
        const int rot = (t >> 1) & 15;
#pragma unroll 1
        for (int i = 0; i < 16; i++) {
            const int n = 16 * strip + ((i + rot) & 15);
            if (n < count) {
                const int e = err[ranked ? (W.order[slot][0][n] & 63) : n];
                const int tie = keyed ? W.two.keys[slot][n] : n;
                if (e < best_err || (e == best_err && best >= 0 && tie < best_tie)) { best_err = e; best = n; best_tie = tie; }
            }
        }
        W.strip.err[strip][slot][which] = best_err;
        W.strip.pos[strip][slot][which] = best;
    }
}
ITW_HD void bc7_phase_strips(int lane, Bc7Warp& W, const Bc7Params& P, int g, int ma, int mb, bool by_shape)
{
    bc7_strips(lane, W, g, (mb != ma) ? 2 : 1, bc7_slot_count(P, ma), (mb != ma) ? bc7_slot_count(P, mb) : 0, ma >= 2, by_shape);
}
ITW_HD void bc7_phase_winners(int lane, Bc7Warp& W, const Bc7Params& P, int g, int ma, int mb)
{
    const int nm = (mb != ma) ? 2 : 1;
    for (int t = lane; t < bc7_group_count(W, g) * nm; t += 32) {
        const int slot = t / nm, which = t - slot * nm;
        const int m = which ? mb : ma;
        const bool keyed = bc7_shape_order(P, m);
        int best = -1, best_err = kErrNone, best_tie = 0;
        for (int s = 0; s < kBc7Strips; s++) {
            const int e = W.strip.err[s][slot][which], n = W.strip.pos[s][slot][which];
            if (n < 0) continue;
            const int tie = keyed ? W.two.keys[slot][n] : n;
            if (e < best_err || (e == best_err && best >= 0 && tie < best_tie)) { best_err = e; best = n; best_tie = tie; }
        }
        W.win_shape[kBc7Batch * W.half + kBc7Slots * g + slot][m] = (best < 0) ? -1 : bc7_slot_shape(W, P, slot, m, best);
    }
}
// Lists in list order (modes 0 / 2, ranked lists) keep one phase: lane <-> (block, list) walks the list.  Through the strip
// phases they measured slower on basic (+0.5 %, H100): their lists are at most 16 entries long except mode 2's.
ITW_HD void bc7_phase_first_min(int lane, Bc7Warp& W, const Bc7Params& P, int g, int ma, int mb)
{
    const int nm = (mb != ma) ? 2 : 1;
    for (int t = lane; t < bc7_group_count(W, g) * nm; t += 32) {
        const int slot = t / nm, which = t - slot * nm;
        const int m = which ? mb : ma;
        const int count = bc7_slot_count(P, m);
        int best = -1, best_err = kErrNone;
        for (int n = 0; n < count; n++) {
            const int e = W.cand_err[slot][which][n];
            if (e < best_err) { best_err = e; best = n; }
        }
        W.win_shape[kBc7Batch * W.half + kBc7Slots * g + slot][m] = (best < 0) ? -1 : bc7_slot_shape(W, P, slot, m, best);
    }
}
#if defined(__CUDACC__) && defined(ITW_BC7_PHASE_CLOCKS)
// Per-phase cycle attribution (tools/bc7_phase_clocks.py; not in the product build): thread 0 of every CTA reads clock64()
// after every barrier and adds the cycles since its previous reading to the phase site it just left.  Sites are numbered in
// the order the program macros expand them.  In the chain phase of a full round it also times each of its passes as lane 0
// sees them: divergent lanes are not guaranteed to have reconverged when lane 0 reads the clock, and the atomics sit inside
// the timed loop, so a pass time is an estimate of the pass, good for comparing passes and builds.
constexpr int kBc7ClockSites = 40;
struct Bc7Clocks {
    unsigned long long site[kBc7ClockSites];     // cycles summed over the CTAs
    char name[kBc7ClockSites][48];               // the phase call of each site
    unsigned long long full_sum, full_count;     // cycles of the full rounds (summed) and their number, over the CTAs
    unsigned long long last_sum, last_max, last_ctas;   // the partial last round: summed, longest CTA, CTAs that ran it
    unsigned long long pass_sum[kBc7MaxRoles], pass_count[kBc7MaxRoles];   // chain passes of the full rounds
    int pass_unit[kBc7MaxRoles][2];              // the two units of each such pass (-1: none)
};
__device__ Bc7Clocks g_bc7_clocks;
#endif
// Chain phase over the whole round.  With nb = per_warp blocks (a power of two, 1..16), lane L works for block L % nb in every
// pass and runs the active units L / nb, L / nb + 32 / nb, ...: a pass holds 32 / nb consecutive units for all blocks, so its
// lanes run the same KIND of unit (partitioned / rotation / mode 6) almost everywhere, and a lane keeps the best candidate of
// ITS block in registers.  Sixteen blocks make a pass two units wide: (mode 0, mode 2), (mode 1, mode 3), (rotation,
// rotation), ... are equally long, where four-wide passes pair three-subset with two-subset chains and leave the last pass
// half empty.  Fewer blocks (the last round of a launch) run wider passes: with one block, all its units run in one pass.
// The units run in bc7_active_unit's order, which is not the reference's, so a lane keeps the minimum of (error, role) and
// the store phase compares (error, role): the first strict minimum in role order (K:1358, :1638, :1650, :1684).
ITW_HD void bc7_phase_chains(int lane, Bc7Warp& W, const Bc7Params& P, int nb)
{
    const int nactive = bc7_active_units(P);
    const int slot = lane & (nb - 1);
    int best_err = kErrNone, best_role = 0;
    u32 code[4] = {0u, 0u, 0u, 0u};
#if defined(__CUDA_ARCH__) && defined(ITW_BC7_PHASE_CLOCKS)
    const bool timed = threadIdx.x == 0 && nb == kBc7Super;
    unsigned long long pass_start = clock64();
#endif
    if (slot < W.ntotal)
        for (int i = lane / nb; i < nactive; i += 32 / nb) {
            const int u = bc7_active_unit(P, i);
            const Bc7Result res = bc7_chain(W, P, lane, slot, u);
            if (res.err < best_err || (res.err == best_err && res.role < best_role)) {
                best_err = res.err; best_role = res.role;
#pragma unroll
                for (int j = 0; j < 4; j++) code[j] = res.code[j];
            }
#if defined(__CUDA_ARCH__) && defined(ITW_BC7_PHASE_CLOCKS)
            if (timed) {
                const unsigned long long now = clock64();
                const int p = i / 2;
                atomicAdd(&g_bc7_clocks.pass_sum[p], now - pass_start);
                atomicAdd(&g_bc7_clocks.pass_count[p], 1ull);
                g_bc7_clocks.pass_unit[p][0] = u;
                g_bc7_clocks.pass_unit[p][1] = (i + 1 < nactive) ? bc7_active_unit(P, i + 1) : -1;
                pass_start = clock64();
            }
#endif
        }
    W.fin.err[lane] = best_err;
    W.fin.role[lane] = best_role;
#pragma unroll
    for (int i = 0; i < 4; i++) W.fin.code[lane][i] = code[i];
}
// the block's winner among the lanes that worked for it, then the 16-byte store; K:2027
ITW_HD void bc7_phase_store(int lane, Bc7Warp& W, int nb, uint8_t* dst, long long first_block)
{
    for (int t = lane; t < W.ntotal; t += 32) {
        int best = t;
        for (int j = 1; j < 32 / nb; j++) {
            const int l = t + nb * j;
            if (W.fin.err[l] < W.fin.err[best] || (W.fin.err[l] == W.fin.err[best] && W.fin.role[l] < W.fin.role[best])) best = l;
        }
        u32* out = reinterpret_cast<u32*>(dst + (size_t)(first_block + t) * 16);
#pragma unroll
        for (int i = 0; i < 4; i++) out[i] = W.fin.code[best][i];
    }
}

// The program of one round (per_warp = 1, 2, 4, 8 or 16 blocks per warp: `nvalid` of them from `first_block` of `surf`,
// results to block `out_block` of `dst`), as a list of (phase, barrier) pairs.
#define ITW_BC7_GROUP_PROGRAM(PHASE, g)                                                \
    if (P.sel[0]) {                                                                    \
        PHASE(bc7_phase_masks3(lane, W, P, g));                                        \
        PHASE(bc7_phase_shapes3(lane, W, P, g));                                       \
        PHASE(bc7_phase_first_min(lane, W, P, g, 0, 1));                               \
    }                                                                                  \
    if (bc7_full_two(P)) {                                                             \
        PHASE(bc7_phase_two_full(lane, W, P, g));                                      \
        if (bc7_needs_rank(P, 0)) {                                                    \
            PHASE(bc7_phase_rank(lane, W, g, 0));                                      \
        }                                                                              \
        PHASE(bc7_phase_strips(lane, W, P, g, 2, 3, true));                            \
        PHASE(bc7_phase_winners(lane, W, P, g, 2, 3));                                 \
    } else if (bc7_needs_keys(P, 0)) {                                                 \
        PHASE(bc7_phase_keys(lane, W, P, g, 0));                                       \
        PHASE(bc7_phase_rank(lane, W, g, 0));                                          \
        PHASE(bc7_phase_shapes(lane, W, P, g, 2, 3));                                  \
        PHASE(bc7_phase_first_min(lane, W, P, g, 2, 3));                               \
    }                                                                                  \
    if (bc7_needs_keys(P, 1)) {                                                        \
        PHASE(bc7_phase_keys(lane, W, P, g, 1));                                       \
        if (bc7_needs_rank(P, 1)) {                                                    \
            PHASE(bc7_phase_rank(lane, W, g, 1));                                      \
            PHASE(bc7_phase_shapes(lane, W, P, g, 4, 4));                              \
            PHASE(bc7_phase_first_min(lane, W, P, g, 4, 4));                           \
        } else {                                                                       \
            PHASE(bc7_phase_shapes(lane, W, P, g, 4, 4));                              \
            PHASE(bc7_phase_strips(lane, W, P, g, 4, 4, false));                       \
            PHASE(bc7_phase_winners(lane, W, P, g, 4, 4));                             \
        }                                                                              \
    }
// The halves and the groups are LOOPS, not copies: four inlined copies of every shape phase made the kernel body 6.6 k
// instructions (105 KB) -- the phases of one copy are what the instruction cache should hold.  A round of at most four blocks
// per warp has one group.
#define ITW_BC7_SHAPE_PROGRAM(PHASE)                                                   \
    ITW_UNROLL(1)                                                                      \
    for (int half = 0; half < ((per_warp > kBc7Batch) ? 2 : 1); half++) {              \
        PHASE(bc7_phase_load(lane, W, surf, first_block, nvalid, half));               \
        PHASE(bc7_phase_planes(lane, W));                                              \
        ITW_UNROLL(1)                                                                  \
        for (int g = 0; g < ((per_warp > kBc7Slots) ? 2 : 1); g++) {                   \
            ITW_BC7_GROUP_PROGRAM(PHASE, g)                                            \
        }                                                                              \
    }                                                                                  \
    if (per_warp > kBc7Batch) {                                                        \
        PHASE(bc7_phase_park(lane, W, surf, first_block, nvalid));                     \
    }
#define ITW_BC7_CHAIN_PROGRAM(PHASE)                                                   \
    PHASE(bc7_phase_chains(lane, W, P, per_warp));                                     \
    PHASE(bc7_phase_store(lane, W, per_warp, dst, out_block));
#define ITW_BC7_PROGRAM(PHASE)                                                         \
    ITW_BC7_SHAPE_PROGRAM(PHASE)                                                       \
    ITW_BC7_CHAIN_PROGRAM(PHASE)

#if defined(__CUDACC__)
// All warps of a CTA walk the phases in lock step (block barrier between phases) and one CTA fills an
// SM: at any moment every warp of the SM is inside the same few hundred instructions, which is what
// the instruction cache needs -- the first version of this kernel lost 90 % of its issue slots to
// instruction fetch.  Work per phase is the same for every warp, so the
// barriers cost little.
constexpr int kBc7WarpsPerCta = 16;
constexpr size_t kBc7SmemBytes = sizeof(Bc7Warp) * kBc7WarpsPerCta;

// kTma: the consecutive blocks a CTA works on in one round (16 warps x per_warp blocks) are fetched by the TMA engine
// (cp.async.bulk, SASS UBLKCP) into a 4-row shared-memory tile, signalled through an mbarrier; the load phases read the tile
// from shared memory.  One tile buffer is enough: it is free again once the last load phase of a round is over, and the next
// tile then streams in behind the whole chain phase.  Needs 16-byte aligned surface rows; other surfaces use the plain
// global-load variant.
constexpr int kBc7TileBlocks = kBc7WarpsPerCta * kBc7Super;              // 256
constexpr int kBc7TileRowBytes = kBc7TileBlocks * 16;                     // 4096

#if defined(ITW_BC7_PHASE_CLOCKS)
__device__ void bc7_clock_tick(int site, const char* name, unsigned long long& last)
{
    const unsigned long long now = clock64();
    atomicAdd(&g_bc7_clocks.site[site], now - last);
    last = now;
    if (blockIdx.x == 0 && g_bc7_clocks.name[site][0] == 0)
        for (int i = 0; i < 47 && name[i]; i++) g_bc7_clocks.name[site][i] = name[i];
}
#define ITW_BC7_TICK(name) if (threadIdx.x == 0) bc7_clock_tick(__COUNTER__ - clock_site0, name, clock_last)
#else
#define ITW_BC7_TICK(name)
#endif

// Schedule.  A full round gives every warp of the grid kBc7Super blocks: wave = grid x 16 warps x 16 blocks.  The blocks left
// after the full rounds (fewer than a wave) are dealt over ALL warps of the grid as one last round of per_warp = 1, 2, 4, 8 or
// 16 blocks, the smallest that covers them, instead of a sixteen-block round of the first few CTAs while the other SMs idle.
// Warps stay CTA-major, so a CTA's share of a round is one contiguous run of blocks (one TMA tile).  Small surfaces are the
// same case with zero full rounds.
template <bool kTma>
__global__ void __launch_bounds__(kBc7WarpsPerCta * 32, 1)
bc7_kernel(SurfaceView gsurf, uint8_t* __restrict__ dst, Bc7Params P, long long nblocks)
{
    extern __shared__ __align__(16) unsigned char bc7_smem[];
    __shared__ __align__(128) unsigned char stage[kTma ? 4 * kBc7TileRowBytes : 16];
    __shared__ __align__(8) unsigned long long full;
    Bc7Warp& W = reinterpret_cast<Bc7Warp*>(bc7_smem)[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // The schedule lives in shared memory and is read again in every round: held in registers across the phases, it added 40
    // bytes to the kernel's spills at the 128-register cap (-Xptxas -v).  Round counters are ints (a round is at least 16 blocks).
    __shared__ int sched[2];                                              // full rounds; blocks per warp of the last one (0: none)
    if (threadIdx.x == 0) {
        const long long wave = (long long)gridDim.x * kBc7TileBlocks;
        const long long nfull = nblocks / wave, rem = nblocks - nfull * wave;
        int p = 0;
        if (rem > 0)
            for (p = 1; p < kBc7Super && (rem + p - 1) / p > (long long)gridDim.x * kBc7WarpsPerCta; p *= 2) {}
        sched[0] = (int)nfull;
        sched[1] = p;
    }
    auto round_per_warp = [&](int round) { return round < sched[0] ? kBc7Super : (round == sched[0] ? sched[1] : 0); };
    auto tile_first = [&](int round) {
        return round * ((long long)gridDim.x * kBc7TileBlocks) + (long long)blockIdx.x * kBc7WarpsPerCta * round_per_warp(round);
    };
    auto prefetch = [&](int round) {                                      // one thread feeds the TMA engine
        const long long fb = tile_first(round), tile_blocks = (long long)kBc7WarpsPerCta * round_per_warp(round);
        if (tile_blocks == 0 || fb >= nblocks) return;
        const long long left = nblocks - fb;
        tma_prefetch_tile(stage, kBc7TileRowBytes, &full, gsurf, fb, (int)(left < tile_blocks ? left : tile_blocks), 16);
    };
#if defined(ITW_BC7_PHASE_CLOCKS)
    const int clock_site0 = __COUNTER__;
    unsigned long long clock_last = clock64();
#endif
    if (kTma && threadIdx.x == 0) mbar_init(&full, 1);
    __syncthreads();
    if (kTma && threadIdx.x == 0) prefetch(0);
    for (int round = 0;; round++) {
        const int per_warp = round_per_warp(round);
        const long long cta_first = tile_first(round);
        if (per_warp == 0 || cta_first >= nblocks) break;               // all done, or nothing for this CTA in the last round
#if defined(ITW_BC7_PHASE_CLOCKS)
        const unsigned long long round_start = clock_last;
#endif
        const long long out_block = cta_first + (long long)warp * per_warp;
        const long long left = nblocks - out_block;
        const int nvalid = (int)(left <= 0 ? 0 : (left < per_warp ? left : per_warp));
        SurfaceView surf = gsurf;
        long long first_block = out_block;
        if (kTma) {
            mbar_wait(&full, (unsigned)(round & 1));
            surf = SurfaceView{stage, kBc7TileBlocks * 4, 4, kBc7TileRowBytes};
            first_block = (long long)warp * per_warp;                    // block index inside the staged tile
        }
        ITW_BC7_TICK("round start (TMA wait)");
#define ITW_PHASE_DEVICE(call) call; __syncthreads(); ITW_BC7_TICK(#call)
        ITW_BC7_SHAPE_PROGRAM(ITW_PHASE_DEVICE)
        if (kTma && threadIdx.x == 0) prefetch(round + 1);               // every load phase of this round is behind a barrier
        ITW_BC7_CHAIN_PROGRAM(ITW_PHASE_DEVICE)
#undef ITW_PHASE_DEVICE
#if defined(ITW_BC7_PHASE_CLOCKS)
        if (threadIdx.x == 0) {
            const unsigned long long cycles = clock_last - round_start;
            if (per_warp == kBc7Super && round < sched[0]) {
                atomicAdd(&g_bc7_clocks.full_sum, cycles);
                atomicAdd(&g_bc7_clocks.full_count, 1ull);
            } else {
                atomicAdd(&g_bc7_clocks.last_sum, cycles);
                atomicMax(&g_bc7_clocks.last_max, cycles);
                atomicAdd(&g_bc7_clocks.last_ctas, 1ull);
            }
        }
#endif
    }
}
#undef ITW_BC7_TICK
#endif

}  // namespace itw
