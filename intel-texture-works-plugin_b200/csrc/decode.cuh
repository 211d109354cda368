// decode.cuh -- BCn DECODERS (SURVEY.md 8f-3): the step after the hot path in the plug-in's preview
// (IntelPlugin.cpp:1051-1066 -> DirectX::Decompress -> D3DXDecodeBC*, DirectXTex/DirectXTexCompress.cpp:358-468).
//
// One thread decodes one 4x4 block and writes its 16 texels (4 x 128-bit row stores for RGBA8; a warp covers 32
// adjacent blocks, so every row store is a contiguous 512-byte request).  Bandwidth-bound: 8/16 B in, 64/128 B out.
//
// Contract.  BC7 and BC6H are integer-exact by the format definition (interpolation ((64-w)a + wb + 32) >> 6,
// BC6H un-quantisation and the final (x*31)>>6 to half bits; DirectXTex/BC6HBC7.cpp:1077-1236, :1937-2144), so the
// result is THE decode.  DirectXTex decodes BC1-BC5 to FLOAT texels (BC.cpp:322-370, :897-936, BC4BC5.cpp:42-95) and the
// preview stores them as UNORM8 through DirectXMath.  Here: BC1 / BC3 colours evaluate DirectXTex's float expressions and
// round to nearest; the 8-value alpha / BC4 / BC5 ramps use integer formulas that equal round-to-nearest of DirectXTex's
// float ramps for EVERY endpoint pair and index (tests/test_bc45_vs_directxtex.py, tests/test_decode.py, both against the
// reference's own decoder bodies).  What stays outside the tree is only the rounding mode of that final store.
// The numpy restatement of exactly these rules is tests/bcn_decode.py.
#pragma once
#include "bc6h.cuh"

namespace itw {

// LSB-first reader over one 128-bit block
// The block is kept in four 32-bit registers and CONSUMED: every read returns the low n bits and funnel-shifts the whole
// 128-bit value right by n (n < 32), four SHF instructions, no position bookkeeping and no branches.
ITW_HD u32 funnel_r(u32 lo, u32 hi, int n)     // low word of (hi:lo) >> n, 0 <= n < 32
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, n);
#else
    return (u32)((((unsigned long long)hi << 32) | lo) >> n);
#endif
}
struct BitReader {
    u32 w0, w1, w2, w3;
    ITW_HD void init(const u32 (&w)[4]) { w0 = w[0]; w1 = w[1]; w2 = w[2]; w3 = w[3]; }
    ITW_HD void skip(int n)                   // 0 <= n < 32
    {
        w0 = funnel_r(w0, w1, n);
        w1 = funnel_r(w1, w2, n);
        w2 = funnel_r(w2, w3, n);
        w3 >>= n;
    }
    ITW_HD u32 get(int n)                     // 0 <= n <= 16
    {
        const u32 v = w0 & ((1u << n) - 1u);
        skip(n);
        return v;
    }
};

// ---- BC1 colour block -> packed RGBA (alpha 255, or 0 for the transparent code of 3-colour mode) ----
// DirectXTex's DecodeBC1 (BC.cpp:322-370) in its own float operations -- endpoint = n * (1/31) or n * (1/63), interpolants
// (c1 - c0) * t + c0 with t = 1/3, 2/3 or 1/2 (XMVectorLerp: a multiply, then an add) -- followed by the UNORM8 store as
// x * 255 + 0.5 truncated.  The float part is checked against the reference's own body (tests/test_decode.py); the store is
// DirectXMath (outside the tree), round-to-nearest is the assumption.  Note that this is NOT bit replication of the 5/6-bit
// endpoints: 7/31 decodes to 58, not 57.
ITW_HD u32 unorm8_of(float x) { return (u32)(int)(x * 255.0f + 0.5f); }
struct Unorm8Store { ITW_HD static u32 of(float x) { return unorm8_of(x); } };
// Store::of(float) -> byte is the store applied to DirectXTex's float endpoints / interpolants (display.cuh adds the sRGB ones)
template <class Store>
ITW_HD void decode_bc1_colour_as(u32 (&px)[16], u32 w0, u32 w1, bool force4)
{
    const u32 c0 = w0 & 0xFFFFu, c1 = w0 >> 16;
    const bool four = (c0 > c1) || force4;
    u32 p0 = 0xFF000000u, p1 = 0xFF000000u, p2 = 0xFF000000u, p3 = four ? 0xFF000000u : 0u;
#pragma unroll
    for (int c = 0; c < 3; c++) {                               // c = 0: red (bits 11..15), 1: green (5..10), 2: blue (0..4)
        const int shift = (c == 0) ? 11 : ((c == 1) ? 5 : 0);
        const u32 mask = (c == 1) ? 63u : 31u;
        const float scale = (c == 1) ? (1.0f / 63.0f) : (1.0f / 31.0f);
        const float f0 = (float)((c0 >> shift) & mask) * scale, f1 = (float)((c1 >> shift) & mask) * scale;
        const float len = f1 - f0;
        const float f2 = four ? (len * (1.0f / 3.0f) + f0) : (len * 0.5f + f0);
        const float f3 = len * (2.0f / 3.0f) + f0;
        p0 |= Store::of(f0) << (8 * c);
        p1 |= Store::of(f1) << (8 * c);
        p2 |= Store::of(f2) << (8 * c);
        if (four) p3 |= Store::of(f3) << (8 * c);
    }
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const u32 q = (w1 >> (2 * k)) & 3u;
        px[k] = (q == 0) ? p0 : ((q == 1) ? p1 : ((q == 2) ? p2 : p3));
    }
}
ITW_HD void decode_bc1_colour(u32 (&px)[16], u32 w0, u32 w1, bool force4) { decode_bc1_colour_as<Unorm8Store>(px, w0, w1, force4); }
// ---- BC3 alpha / BC4 / BC5 channel block -> 16 values ----
ITW_HD void decode_alpha(u32 (&val)[16], u32 w0, u32 w1)
{
    const u32 a0 = w0 & 255u, a1 = (w0 >> 8) & 255u;
    const unsigned long long idx = ((unsigned long long)w1 << 16) | (w0 >> 16);
    const bool eight = a0 > a1;
    // the eight palette entries packed one per byte, then a 64-bit shift per texel instead of a select chain
    unsigned long long pal = (unsigned long long)a0 | ((unsigned long long)a1 << 8);
#pragma unroll
    for (u32 q = 2; q < 8; q++) {
        u32 v;
        if (eight) v = ((8u - q) * a0 + (q - 1u) * a1 + 3u) / 7u;
        else if (q == 6) v = 0u;
        else if (q == 7) v = 255u;
        else v = ((6u - q) * a0 + (q - 1u) * a1 + 2u) / 5u;
        pal |= (unsigned long long)v << (8 * q);
    }
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const u32 q = (u32)(idx >> (3 * k)) & 7u;
        val[k] = (u32)(pal >> (8 * q)) & 255u;
    }
}

// ---- BC7; format definition as implemented by DirectXTex/BC6HBC7.cpp:1937-2144 ----
// subsets, partition bits, rotation bits, index-selection bits, colour bits, alpha bits, endpoint p-bits,
// shared p-bits, index bits, second index bits
struct Bc7ModeDesc { int ns, pb, rb, isb, cb, ab, epb, spb, ib, ib2; };
ITW_HD Bc7ModeDesc bc7_mode_desc(int m)
{
    switch (m) {
        case 0: return Bc7ModeDesc{3, 4, 0, 0, 4, 0, 1, 0, 3, 0};
        case 1: return Bc7ModeDesc{2, 6, 0, 0, 6, 0, 0, 1, 3, 0};
        case 2: return Bc7ModeDesc{3, 6, 0, 0, 5, 0, 0, 0, 2, 0};
        case 3: return Bc7ModeDesc{2, 6, 0, 0, 7, 0, 1, 0, 2, 0};
        case 4: return Bc7ModeDesc{1, 0, 2, 1, 5, 6, 0, 0, 2, 3};
        case 5: return Bc7ModeDesc{1, 0, 2, 0, 7, 8, 0, 0, 2, 2};
        case 6: return Bc7ModeDesc{1, 0, 0, 0, 7, 7, 1, 0, 4, 0};
        default: return Bc7ModeDesc{2, 6, 0, 0, 5, 5, 1, 0, 2, 0};
    }
}
ITW_HD int lowest_set_bit(u32 v)              // v != 0
{
#if defined(__CUDA_ARCH__)
    return __ffs((int)v) - 1;
#else
    return __builtin_ctz(v);
#endif
}
ITW_HD u32 widen8(u32 v, int bits) { return ((v << (8 - bits)) | (v >> (2 * bits - 8))) & 255u; }

// Returns false for the reserved mode (mode byte 0): the block decodes to transparent black, as in DirectXTex
// (BC6HBC7.cpp:2135-2143).  All endpoint arrays are indexed by fully unrolled loops so that they live in registers.
ITW_HD bool decode_bc7(u32 (&px)[16], const u32 (&w)[4])
{
    if ((w[0] & 255u) == 0u) {
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = 0u;
        return false;
    }
    BitReader b;
    b.init(w);
    const int mode = lowest_set_bit(w[0] & 255u);
    b.skip(mode + 1);
    const Bc7ModeDesc d = bc7_mode_desc(mode);
    const int shape = (int)b.get(d.pb), rot = (int)b.get(d.rb), isel = (int)b.get(d.isb);
    const int ne = 2 * d.ns;
    u32 ep[6][4];
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int e = 0; e < 6; e++) ep[e][c] = (e < ne) ? b.get(d.cb) : 0u;
#pragma unroll
    for (int e = 0; e < 6; e++) ep[e][3] = (d.ab && e < ne) ? b.get(d.ab) : 255u;
    int cbits = d.cb, abits = d.ab;
    if (d.epb) {
#pragma unroll
        for (int e = 0; e < 6; e++) {
            if (e < ne) {
                const u32 p = b.get(1);
#pragma unroll
                for (int c = 0; c < 3; c++) ep[e][c] = (ep[e][c] << 1) | p;
                if (d.ab) ep[e][3] = (ep[e][3] << 1) | p;
            }
        }
        cbits++;
        if (d.ab) abits++;
    }
    if (d.spb) {
#pragma unroll
        for (int s = 0; s < 2; s++) {            // mode 1 only: two subsets
            const u32 p = b.get(1);
#pragma unroll
            for (int c = 0; c < 3; c++) {
                ep[2 * s][c] = (ep[2 * s][c] << 1) | p;
                ep[2 * s + 1][c] = (ep[2 * s + 1][c] << 1) | p;
            }
        }
        cbits++;
    }
    u32 pk[6];                                   // packed r | g<<8 | b<<16 | a<<24
#pragma unroll
    for (int e = 0; e < 6; e++) {
        const u32 a = d.ab ? widen8(ep[e][3], abits) : 255u;
        pk[e] = widen8(ep[e][0], cbits) | (widen8(ep[e][1], cbits) << 8) | (widen8(ep[e][2], cbits) << 16) | (a << 24);
    }
    const u32 pattern = (d.ns == 1) ? 0u : shape_pattern(d.ns == 2 ? shape : 64 + shape);
    const int anchor1 = (d.ns == 1) ? -1 : shape_anchor(d.ns == 2 ? shape : 64 + shape, 1);
    const int anchor2 = (d.ns == 3) ? shape_anchor(64 + shape, 2) : -1;
    unsigned long long i1 = 0, i2 = 0;           // 4 bits per texel
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const bool anchor = (k == 0) || (k == anchor1) || (k == anchor2);
        i1 |= (unsigned long long)b.get(anchor ? d.ib - 1 : d.ib) << (4 * k);
    }
    if (d.ib2) {
#pragma unroll
        for (int k = 0; k < 16; k++) i2 |= (unsigned long long)b.get(k == 0 ? d.ib2 - 1 : d.ib2) << (4 * k);
    }
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const u32 s = (pattern >> (2 * k)) & 3u;
        const u32 e0 = (s == 0) ? pk[0] : ((s == 1) ? pk[2] : pk[4]);
        const u32 e1 = (s == 0) ? pk[1] : ((s == 1) ? pk[3] : pk[5]);
        const int q1 = (int)((i1 >> (4 * k)) & 15ull), q2 = (int)((i2 >> (4 * k)) & 15ull);
        u32 cw, aw;
        if (!d.ib2) cw = aw = (u32)bc7_weight(d.ib, q1);
        else if (!isel) { cw = (u32)bc7_weight(d.ib, q1); aw = (u32)bc7_weight(d.ib2, q2); }
        else { cw = (u32)bc7_weight(d.ib2, q2); aw = (u32)bc7_weight(d.ib, q1); }
        // two 16-bit lanes per word: every lane is at most 64*255 + 32 < 2^16
        const u32 rb = (((64u - cw) * (e0 & 0x00FF00FFu) + cw * (e1 & 0x00FF00FFu) + 0x00200020u) >> 6) & 0x00FF00FFu;
        const u32 g = (((64u - cw) * ((e0 >> 8) & 255u) + cw * ((e1 >> 8) & 255u) + 32u) >> 6);
        const u32 a = (((64u - aw) * (e0 >> 24) + aw * (e1 >> 24) + 32u) >> 6);
        u32 v = rb | (g << 8) | (a << 24);
        if (rot) {                               // swap alpha with channel rot-1
            const int sh = 8 * (rot - 1);
            const u32 ch = (v >> sh) & 255u;
            v = (v & ~((255u << sh) | 0xFF000000u)) | (a << sh) | (ch << 24);
        }
        px[k] = v;
    }
    return true;
}

// ---- BC6H, unsigned; format definition as implemented by DirectXTex/BC6HBC7.cpp:1077-1236 ----
ITW_HD int bc6_mode_epb(int mode)
{
    // {10,7,11,11,11,9,8,8,8,6,10,11,12,16} packed 5 bits each
    const unsigned long long t = 10ull | (7ull << 5) | (11ull << 10) | (11ull << 15) | (11ull << 20) | (9ull << 25) | (8ull << 30) |
                                 (8ull << 35) | (8ull << 40) | (6ull << 45) | (10ull << 50) | (11ull << 55);
    if (mode < 12) return (int)((t >> (5 * mode)) & 31ull);
    return (mode == 12) ? 12 : 16;
}
// delta bits of endpoints 1..3 per channel (r | g << 4 | b << 8); modes 9 and 10 store plain values
ITW_HD u32 bc6_mode_delta_bits(int mode)
{
    switch (mode) {
        case 0: case 5: return 0x555u;
        case 1: return 0x666u;
        case 2: return 0x445u;       // r 5, g 4, b 4
        case 3: return 0x454u;       // r 4, g 5, b 4
        case 4: return 0x544u;       // r 4, g 4, b 5
        case 6: return 0x556u;       // r 6, g 5, b 5
        case 7: return 0x565u;       // r 5, g 6, b 5
        case 8: return 0x655u;       // r 5, g 5, b 6
        case 11: return 0x999u;
        case 12: return 0x888u;
        case 13: return 0x444u;
        default: return 0u;
    }
}
// out[k][0] = r | g << 16, out[k][1] = b | 0x3C00 << 16 (half bit patterns, alpha = 1.0).  Returns false for the
// reserved mode fields (decoded as opaque black, BC6HBC7.cpp:1088-1106).  The twelve endpoint fields are gathered
// into three 64-bit registers (per channel: endpoints 0..3, 16 bits each) -- no per-thread arrays, hence no local
// memory (the array version spilled to DRAM).
//
// kSigned = BC6H_SF16 (D3DXDecodeBC6HS = D3DX_BC6H::Decode(true, ...), what DirectX::Decompress runs for DXGI_FORMAT_BC6H_SF16,
// DirectXTexCompress.cpp:414): every endpoint is sign-extended at the mode's endpoint width (BC6HBC7.cpp:1141-1157, :582-594),
// un-quantised symmetrically (:1318-1336), the interpolated value is scaled by 31/32 on its magnitude (:1351-1354) and leaves
// as sign | magnitude half bits (BC.h INT2F16).
ITW_HD int bc6_dequant_signed(int v, int bits)                         // BC6HBC7.cpp:1318-1336
{
    if (bits >= 16) return v;
    const bool neg = v < 0;
    if (neg) v = -v;
    int unq;
    if (v == 0) unq = 0;
    else if (v >= ((1 << (bits - 1)) - 1)) unq = 0x7FFF;
    else unq = ((v << 15) + 0x4000) >> (bits - 1);
    return neg ? -unq : unq;
}
template <bool kSigned>
ITW_HD bool decode_bc6h(u32 (&px)[16][2], const u32 (&w)[4])
{
    const u32 m2 = w[0] & 3u;
    const u32 field = (m2 < 2u) ? m2 : (w[0] & 31u);
    int mode = -1;
    for (int m = 0; m < 14; m++)
        if ((u32)bc6_prefix(m) == field) mode = m;
    if (mode < 0) {
#pragma unroll
        for (int k = 0; k < 16; k++) { px[k][0] = 0u; px[k][1] = 0x3C000000u; }
        return false;
    }
    BitReader b;
    b.init(w);
#if defined(__CUDA_ARCH__)
    const Bc6Step* steps = d_bc6_layout[mode];
#else
    const Bc6Step* steps = h_bc6_layout[mode];
#endif
    unsigned long long ch0 = 0ull, ch1 = 0ull, ch2 = 0ull;
    for (int i = 0; i < kBc6MaxSteps; i++) {
        const int f = steps[i].f, bit = steps[i].b, n = steps[i].n;
        if (n == 0) break;
        u32 v;                                               // the field's bits, already at their positions
        if (n > 0) v = b.get(n) << bit;
        else {
            v = 0u;
            for (int j = 0; j < -n; j++) v |= b.get(1) << (bit - j);
        }
        if (f == 0) continue;                                // mode prefix
        const int e = (f - 1) / 3, c = (f - 1) % 3;
        const unsigned long long add = (unsigned long long)v << (16 * e);
        if (c == 0) ch0 |= add; else if (c == 1) ch1 |= add; else ch2 |= add;
    }
    const int regions = (mode < 10) ? 2 : 1;
    const int epb = bc6_mode_epb(mode);
    const u32 dbits = bc6_mode_delta_bits(mode);
    const u32 mask = (1u << epb) - 1u;
    int lo[2][3], hi[2][3];                                  // decoded endpoints A, B per subset and channel
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const unsigned long long chv = (c == 0) ? ch0 : ((c == 1) ? ch1 : ch2);
        const u32 base = (u32)chv & 0xFFFFu;
        const int nb = (int)((dbits >> (4 * c)) & 15u);
        int ep[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            u32 v = (u32)(chv >> (16 * i)) & 0xFFFFu;
            if (i > 0 && nb > 0) {
                if (v & (1u << (nb - 1))) v -= 1u << nb;     // sign-extend the delta (wraps, masked below)
                v = (base + v) & mask;
            }
            if (kSigned) {
                int sv = (int)v;
                if (epb < 32 && (v & (1u << (epb - 1)))) sv -= 1 << epb;      // SIGN_EXTEND at the endpoint width
                ep[i] = bc6_dequant_signed(sv, epb);
            } else ep[i] = bc6_dequant((int)v, epb);
        }
        lo[0][c] = ep[0]; hi[0][c] = ep[1]; lo[1][c] = ep[2]; hi[1][c] = ep[3];
    }
    const int shape = (regions == 2) ? (int)b.get(5) : 0;
    const u32 pattern = (regions == 2) ? shape_pattern(shape) : 0u;
    const int anchor1 = (regions == 2) ? shape_anchor(shape, 1) : -1;
    const int ib = (regions == 2) ? 3 : 4;
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const bool second = ((pattern >> (2 * k)) & 3u) != 0u;
        const bool anchor = (k == 0) || (k == anchor1);
        const int q = (int)b.get(anchor ? ib - 1 : ib);
        const int wt = bc7_weight(ib, q);
        u32 h[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const int a = second ? lo[1][c] : lo[0][c], bb = second ? hi[1][c] : hi[0][c];
            const int v = ((64 - wt) * a + wt * bb + 32) >> 6;           // arithmetic shift of a possibly negative value, as in C++ on x86
            if (kSigned) {
                const int m = (v < 0) ? -(((-v) * 31) >> 5) : ((v * 31) >> 5);
                h[c] = (m < 0) ? (0x8000u | (u32)(-m)) : (u32)m;
            } else h[c] = (u32)((v * 31) >> 6);
        }
        px[k][0] = h[0] | (h[1] << 16);
        px[k][1] = h[2] | 0x3C000000u;
    }
    return true;
}

// ---- one block of any format -> 16 packed texels (RGBA8: one word, RGBA16F: two words) ----
// kFormat: ITW_FORMAT_* ids (DXGI numbers 71/77/80/83/95/98)
template <int kFormat>
ITW_HD void decode_block_rgba8(u32 (&px)[16], const u32 (&w)[4])
{
    if (kFormat == 71) decode_bc1_colour(px, w[0], w[1], false);
    else if (kFormat == 77) {
        u32 a[16];
        decode_bc1_colour(px, w[2], w[3], true);
        decode_alpha(a, w[0], w[1]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = (px[k] & 0x00FFFFFFu) | (a[k] << 24);
    } else if (kFormat == 80) {
        u32 r[16];
        decode_alpha(r, w[0], w[1]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = r[k] | 0xFF000000u;
    } else if (kFormat == 83) {
        u32 r[16], g[16];
        decode_alpha(r, w[0], w[1]);
        decode_alpha(g, w[2], w[3]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = r[k] | (g[k] << 8) | 0xFF000000u;
    } else decode_bc7(px, w);
}

#if defined(__CUDACC__)
// dst rows: `stride` bytes apart, texel (x, y) at dst + y*stride + x*texel_bytes
template <int kFormat, bool kVec16>
__global__ void __launch_bounds__(128) decode_kernel(const uint8_t* __restrict__ blocks, uint8_t* __restrict__ dst, int width,
                                                     int height, long long stride)
{
    const int bw = width >> 2, bh = height >> 2;
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= (long long)bw * bh) return;
    const int by = (int)(id / bw), bx = (int)(id - (long long)by * bw);
    u32 w[4];
    if (kFormat == 71 || kFormat == 80) {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(blocks) + id);
        w[0] = v.x; w[1] = v.y; w[2] = w[3] = 0u;
    } else {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(blocks) + id);
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
    }
    if (kFormat == 95 || kFormat == 96) {
        u32 px[16][2];
        decode_bc6h<kFormat == 96>(px, w);
        uint8_t* row = dst + (long long)(4 * by) * stride + (long long)bx * 32;
#pragma unroll
        for (int y = 0; y < 4; y++, row += stride) {
            if (kVec16) {
                reinterpret_cast<uint4*>(row)[0] = make_uint4(px[4 * y][0], px[4 * y][1], px[4 * y + 1][0], px[4 * y + 1][1]);
                reinterpret_cast<uint4*>(row)[1] = make_uint4(px[4 * y + 2][0], px[4 * y + 2][1], px[4 * y + 3][0], px[4 * y + 3][1]);
            } else {
#pragma unroll
                for (int x = 0; x < 4; x++) {
                    reinterpret_cast<u32*>(row)[2 * x] = px[4 * y + x][0];
                    reinterpret_cast<u32*>(row)[2 * x + 1] = px[4 * y + x][1];
                }
            }
        }
    } else {
        u32 px[16];
        decode_block_rgba8<kFormat>(px, w);
        uint8_t* row = dst + (long long)(4 * by) * stride + (long long)bx * 16;
#pragma unroll
        for (int y = 0; y < 4; y++, row += stride) {
            if (kVec16) *reinterpret_cast<uint4*>(row) = make_uint4(px[4 * y], px[4 * y + 1], px[4 * y + 2], px[4 * y + 3]);
            else {
#pragma unroll
                for (int x = 0; x < 4; x++) reinterpret_cast<u32*>(row)[x] = px[4 * y + x];
            }
        }
    }
}
#endif

}  // namespace itw
