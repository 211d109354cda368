// frontend.cuh -- pixel-format front end (SURVEY.md 8f-4): Photoshop's interleaved 8/16/32-bit planes -> the
// RGBA8 / RGBA16F surface the encoders read, in ONE pass per destination texel.  Restates, per texel,
//   IntelPlugin.h:41-96          FloatToByte, ConvertTo8Bit x3, ConvertTo16Bit x3                     (cited IPh:line)
//   IntelPlugin.cpp:291-433, :741-810   ConvertToBC{,4or5,6}From{8,16,32}Bit                          (cited IP:line)
//   IntelPlugin.cpp:1504-1546    FlipXYChannelNormalMap
//   IntelPlugin.cpp:1551-1612    NormalizeNormalMapChain
//   IntelPlugin.cpp:892-928      DoPaddingToMultiplesOf4 -- here a coordinate clamp (replicated edge texels)
// The reference runs these as four whole-image passes on the host; every one of them is per-texel, so the order
// convert -> flip -> normalise -> pad collapses into a single bandwidth-bound kernel.
//
// Half conversion: the plug-in calls DirectXMath's XMConvertFloatToHalf / XMConvertHalfToFloat (IPh:31-39), which
// is Windows SDK code and not in the reference tree.  front_half_from_float / front_float_from_half restate the
// published DirectXMath 3.06 scalar algorithm (the SDK generation of the reference's toolset): RNE on the rebiased
// pattern, |x| > 0x47FFEFFF -> 0x7FFF, truncating denormal shift, exponent 31 decoded as an ordinary binade.
// Outside the normal-half range other DirectXMath versions differ: unpinned there (DESIGN.md section 2).
#pragma once
#include "itw_device.cuh"
#include "gamma_table.cuh"
#include "display_tables.cuh"

namespace itw {

ITW_TABLE_DECL(uint32_t, gamma_threshold, 255)
// byte b -> the stored byte of XMColorSRGBToRGB(b * (1/255)) (tools/gen_display_tables.py); shared with display.cuh
ITW_TABLE_DECL(uint32_t, srgb_in_byte, 64)
ITW_HD u32 byte_table(const uint32_t* T, u32 b) { return (T[b >> 2] >> (8 * (b & 3u))) & 255u; }

struct FrontParams {
    const uint8_t* data;
    int width, height;        // source texels
    int planes, depth;        // 1..4; 8 / 16 / 32
    long long row_bytes;
    int family;               // 0 colour (BC1/3/7), 1 BC4/BC5 (missing planes copy plane 0), 2 HDR (BC6H -> RGBA16F)
    u32 flags;                // ITW_FRONT_*
};
constexpr u32 kFrontAlpha = 1, kFrontGamma = 2, kFrontFlipX = 4, kFrontFlipY = 8, kFrontNormalize = 16;

ITW_HD u32 front_half_from_float(float value)
{
    u32 bits = float_bits(value);
    const u32 sign = (bits & 0x80000000u) >> 16;
    bits &= 0x7FFFFFFFu;
    if (bits > 0x47FFEFFFu) return 0x7FFFu | sign;
    if (bits < 0x38800000u) {
        const u32 shift = 113u - (bits >> 23);
        bits = (shift < 32u) ? ((0x800000u | (bits & 0x7FFFFFu)) >> shift) : 0u;
    } else bits += 0xC8000000u;
    return (((bits + 0x0FFFu + ((bits >> 13) & 1u)) >> 13) & 0x7FFFu) | sign;
}
ITW_HD float front_float_from_half(u32 h)
{
    u32 mant = h & 0x3FFu, exp;
    if (h & 0x7C00u) exp = (h >> 10) & 31u;
    else if (mant) {
        exp = 1u;
        do { exp--; mant <<= 1; } while (!(mant & 0x400u));
        mant &= 0x3FFu;
    } else exp = (u32)-112;
    return bits_float(((h & 0x8000u) << 16) | ((exp + 112u) << 23) | (mant << 13));
}
// FloatToByte, IPh:41-48; the (unsigned char) of an out-of-range double is x86's cvttsd2si low byte: NaN -> 0
ITW_HD u32 front_byte(double v)
{
    if (v > 1.0) return 255u;
    if (v < 0.0) return 0u;
    if (!(v == v)) return 0u;
    return (u32)(int)(v * 255.0) & 255u;
}
// ConvertTo8Bit(double, gammaCorrect): (unsigned char)(pow((double)v, 1/2.2) * 255) with FloatToByte's clamps; IPh:41-48, :67-76.
// On [0, 1] this is a monotone step function of the float v, so it is evaluated WITHOUT pow as the number of thresholds
// T[k] <= v in the generated table (tools/gen_gamma_table.py: bisection on the oracle's own conversion); non-negative floats
// order like their bit patterns.  Outside [0, 1]: v > 1 -> 255; pow of a negative number is NaN -> 0, except
// pow(-inf, y) = +inf -> 255; pow(-0) = +0 -> 0; NaN -> 0.  The double-precision pow this replaces ran at 0.11 of the HBM
// roofline (FP64 rate).
ITW_HD u32 front_gamma_byte(float v)
{
    if (!(v == v)) return 0u;
    if (v > 1.0f) return 255u;
    if (v < 0.0f) return (float_bits(v) == 0xFF800000u) ? 255u : 0u;
    const u32 b = float_bits(v) & 0x7FFFFFFFu;                  // -0 counts as +0
    // start from a cheap single-precision estimate (any value would do: the two loops below make the count exact) and
    // walk to the entry whose thresholds bracket v -- two table reads in the common case instead of a binary search's eight
#if defined(__CUDA_ARCH__)
    const float est = __powf(v, 0.45454545f) * 255.0f;
#else
    const float est = powf(v, 0.45454545f) * 255.0f;
#endif
    int k = (int)est;
    k = (k < 0) ? 0 : ((k > 255) ? 255 : k);
    while (k > 0 && ITW_TABLE(gamma_threshold)[k - 1] > b) k--;
    while (k < 255 && ITW_TABLE(gamma_threshold)[k] <= b) k++;
    return (u32)k;
}
// one source element (raw bits: the 8/16-bit integer, or the float's bit pattern) -> byte; IPh:56-76.
// 16-bit: FloatToByte(v / 32768.0) = floor(v * 255 / 32768) exactly
ITW_HD u32 front_ldr_value(u32 raw, int depth, bool gamma)
{
    if (depth == 8) return raw;
    if (depth == 16) return (raw > 32768u) ? 255u : ((raw * 255u) >> 15);
    if (gamma) return front_gamma_byte(bits_float(raw));
    return front_byte((double)bits_float(raw));
}
// one source element -> half bits; IPh:79-96
ITW_HD u32 front_hdr_value(u32 raw, int depth)
{
    if (depth == 8) return front_half_from_float((float)raw / 255.0f);
    if (depth == 16) return front_half_from_float((float)((double)raw / 32768.0));
    return front_half_from_float(bits_float(raw));
}
ITW_HD u32 front_load_raw(const uint8_t* p, int depth)
{
    if (depth == 8) return *p;
    if (depth == 16) return *reinterpret_cast<const uint16_t*>(p);
    return *reinterpret_cast<const u32*>(p);
}

// NormalizeNormalMapChain on one texel; IP:1565-1584 (bytes around 128) and :1586-1607 (halves, unit length)
ITW_HD void front_normalize_ldr(u32& r, u32& g, u32& b)
{
    const float fr = (float)((int)r - 128), fg = (float)((int)g - 128), fb = (float)((int)b - 128);
    float m = sqrtf(fr * fr + fg * fg + fb * fb);
    if (m > 0.0f) {
        m = 127.0f / m;
        r = (u32)(int)(fr * m + 128.0f) & 255u;
        g = (u32)(int)(fg * m + 128.0f) & 255u;
        b = (u32)(int)(fb * m + 128.0f) & 255u;
    } else { r = 128u; g = 128u; b = 255u; }
}
ITW_HD void front_normalize_hdr(u32& r, u32& g, u32& b)
{
    const float fr = front_float_from_half(r), fg = front_float_from_half(g), fb = front_float_from_half(b);
    float m = sqrtf(fr * fr + fg * fg + fb * fb);
    if (m > 0.0f) {
        m = 1.0f / m;
        r = front_half_from_float(fr * m);
        g = front_half_from_float(fg * m);
        b = front_half_from_float(fb * m);
    } else { r = 0u; g = 0u; b = 0x3C00u; }
}
// the same on one stored RGBA8 texel: r, g and b normalised, alpha kept (normalize_kernel and none_store_kernel)
ITW_HD u32 front_normalize_rgba8(u32 v)
{
    u32 r = v & 255u, g = (v >> 8) & 255u, b = (v >> 16) & 255u;
    front_normalize_ldr(r, g, b);
    return r | (g << 8) | (b << 16) | (v & 0xFF000000u);
}

// FlipXYChannelNormalMap on one texel: IP:1519-1527 (bytes) and IP:1531-1542 (halves)
ITW_HD void front_flip_ldr(u32& r, u32& g, u32 flags)
{
    if (flags & kFrontFlipX) r = 255u - r;
    if (flags & kFrontFlipY) g = 255u - g;
}
ITW_HD void front_flip_hdr(u32& r, u32& g, u32 flags)
{
    if (flags & (kFrontFlipX | kFrontFlipY)) {
        const float fr = front_float_from_half(r), fg = front_float_from_half(g);
        if (flags & kFrontFlipX) r = front_half_from_float(1.0f - fr);
        if (flags & kFrontFlipY) g = front_half_from_float(1.0f - fg);
    }
}

// raw[c] = element of plane c (valid for c < planes) -> out[0] (RGBA8) or out[0..1] (RGBA16F: r | g << 16, b | a << 16)
ITW_HD void front_compose(u32 (&out)[2], const FrontParams& P, const u32 (&raw)[4])
{
    const bool alpha = (P.flags & kFrontAlpha) != 0;
    if (P.family == 2) {
        // IP:291-366.  The 32-bit variant reads alpha from plane 2 (IP:361) -- reference behaviour, kept.
        u32 r = front_hdr_value(raw[0], P.depth);
        u32 g = (P.planes > 1) ? front_hdr_value(raw[1], P.depth) : 0u;
        u32 b = (P.planes > 2) ? front_hdr_value(raw[2], P.depth) : 0u;
        const u32 a = alpha ? front_hdr_value((P.depth == 32) ? raw[2] : raw[3], P.depth) : 0x3C00u;
        front_flip_hdr(r, g, P.flags);
        if (P.flags & kFrontNormalize) front_normalize_hdr(r, g, b);
        out[0] = r | (g << 16);
        out[1] = b | (a << 16);
        return;
    }
    // IP:741-810 (colour: missing planes are 0) and IP:368-433 (BC4/BC5: missing planes copy plane 0)
    const bool gamma = (P.flags & kFrontGamma) != 0;
    u32 r = front_ldr_value(raw[0], P.depth, gamma);
    const u32 missing = (P.family == 1) ? r : 0u;
    u32 g = (P.planes > 1) ? front_ldr_value(raw[1], P.depth, gamma) : missing;
    u32 b = (P.planes > 2) ? front_ldr_value(raw[2], P.depth, gamma) : missing;
    const u32 a = alpha ? front_ldr_value(raw[3], P.depth, gamma) : 255u;
    front_flip_ldr(r, g, P.flags);
    if (P.flags & kFrontNormalize) front_normalize_ldr(r, g, b);
    out[0] = r | (g << 8) | (b << 16) | (a << 24);
    out[1] = 0u;
}
// Destination texel (x, y): clamp into the source (IP:892-928), load its planes, compose
ITW_HD void front_texel(u32 (&out)[2], const FrontParams& P, int x, int y)
{
    const int sx = (x < P.width) ? x : P.width - 1, sy = (y < P.height) ? y : P.height - 1;
    const int esize = P.depth >> 3;
    const uint8_t* px = P.data + (long long)sy * P.row_bytes + (long long)sx * P.planes * esize;
    u32 raw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int c = 0; c < 4; c++)                               // constant indices: raw stays in registers
        if (c < P.planes) raw[c] = front_load_raw(px + c * esize, P.depth);
    front_compose(out, P, raw);
}

// ---- mip levels from document layers (IP:1694-1850: CopyLayersIntoMipMaps, CopyFromLayerChannelIntoImage, FillLayerDataToWhite) ----
// One level as the kernel writes it: the lw x lh top-left rectangle of one layer, staged as planar, tightly packed planes.
constexpr int kLayerMaxLevels = 16;
struct LayerLevel {
    const uint8_t* plane[4];  // colour planes 0..channels-1; plane[3] = alpha, null = FillLayerDataToWhite
    uint8_t* dst;             // the level's RGBA8 / RGBA16F surface
    long long dst_stride;
    long long first;          // first thread of this level in the launch
    int lw, lh;               // texels read from the layer
    int pw, ph;               // texels written (>= lw x lh: the edge is replicated, DoPaddingToMultiplesOf4)
    int channels;             // 1..3
};
struct LayerLaunch {
    LayerLevel lv[kLayerMaxLevels];
    int count;
    int depth;                // the document's: 8, 16 or 32
    int hdr;                  // 1 = RGBA16F (BC6H), 0 = RGBA8
    u32 flip;                 // kFrontFlipX / kFrontFlipY: level 0 only, applied after the copy (IP:2100-2105)
};
// FillLayerDataToWhite (IP:1664-1689) as the raw element the converters then read.  At depth 16 it stores
// ConvertTo16Bit((unsigned8)255), the half 1.0 = 15360, which the 16-bit converters read as 15360 / 32768.
ITW_HD u32 layer_white_raw(int depth)
{
    return depth == 8 ? 255u : (depth == 16 ? 15360u : 0x3F800000u);
}
// Texel (x, y) of one level: `px` holds the texel before the copy (RGBA8 in px[0]; RGBA16F as front_compose packs it) and
// receives it after.  Planes c < channels and alpha are overwritten from the layer at the clamped position; the other planes
// keep what they held.  RGBA8 targets at depth 32 always take the gamma step: the call binds ConvertTo8Bit(double, true).
ITW_HD void layer_texel(u32 (&px)[2], const LayerLevel& L, int depth, bool hdr, u32 flip, int x, int y)
{
    const int sx = (x < L.lw) ? x : L.lw - 1, sy = (y < L.lh) ? y : L.lh - 1;
    const int esize = depth >> 3;
    const long long at = ((long long)sy * L.lw + sx) * esize;
    u32 v[4];
    if (hdr) { v[0] = px[0] & 0xFFFFu; v[1] = px[0] >> 16; v[2] = px[1] & 0xFFFFu; v[3] = px[1] >> 16; }
    else { v[0] = px[0] & 255u; v[1] = (px[0] >> 8) & 255u; v[2] = (px[0] >> 16) & 255u; v[3] = px[0] >> 24; }
    for (int c = 0; c < 4; c++) {
        if (c < 3 && c >= L.channels) continue;
        const u32 raw = (c < 3 || L.plane[3]) ? front_load_raw(L.plane[c] + at, depth) : layer_white_raw(depth);
        v[c] = hdr ? front_hdr_value(raw, depth) : front_ldr_value(raw, depth, true);
    }
    if (hdr) {
        front_flip_hdr(v[0], v[1], flip);
        px[0] = v[0] | (v[1] << 16);
        px[1] = v[2] | (v[3] << 16);
    } else {
        front_flip_ldr(v[0], v[1], flip);
        px[0] = v[0] | (v[1] << 8) | (v[2] << 16) | (v[3] << 24);
    }
}

// ---- cube maps from a cross document (IP:1200-1265: ConvertToCubeMapFromCross) ----
// Cells (column, row) of +X,-X,+Y,-Y,+Z,-Z: the horizontal 4x3 cross (IP:1211) and the vertical 3x4 one, where -Z moves to (1, 3)
// and is copied unrotated (IP:1225-1226).  Host side: the launch carries the six texel origins.
constexpr int kCubeCells[2][6][2] = {{{2, 1}, {0, 1}, {1, 0}, {1, 2}, {1, 1}, {3, 1}}, {{2, 1}, {0, 1}, {1, 0}, {1, 2}, {1, 1}, {1, 3}}};
struct CubeCross {
    FrontParams P;            // the whole document (flags: alpha, gamma)
    uint8_t* dst;             // level 0 of face 0; face f at dst + f * face_bytes, w x h texels, rows `stride` apart
    long long face_bytes, stride;
    int w, h;                 // face size
    int origin[6][2];         // texel origin of each face's cell in the document
    int linear;               // RGBA8 only: the cells are linearised (XMColorSRGBToRGB on r, g, b; alpha passes)
};
// Texel (x, y) of face `face`: the front end at the cell's texel, then -- for an _SRGB encoding with mip maps, whose document scratch is
// R8G8B8A8_UNORM_SRGB while the cube scratch is R8G8B8A8_UNORM (IP:152-154, :1240-1246) -- CopyRectangle's conversion (DirectXTexMisc.cpp:
// 174-274: _LoadScanline, _ConvertScanline with TEX_FILTER_SRGB_IN, the UNORM8 store), which is a byte -> byte map per colour channel.
ITW_HD void cube_texel(u32 (&out)[2], const CubeCross& C, int face, int x, int y)
{
    int ox = 0, oy = 0;
#pragma unroll
    for (int f = 0; f < 6; f++)                               // constant indices: the table stays in the parameter space, no stack copy
        if (f == face) { ox = C.origin[f][0]; oy = C.origin[f][1]; }
    front_texel(out, C.P, ox + x, oy + y);
    if (C.linear) {
        const u32 v = out[0];
        out[0] = byte_table(ITW_TABLE(srgb_in_byte), v & 255u) | (byte_table(ITW_TABLE(srgb_in_byte), (v >> 8) & 255u) << 8) |
                 (byte_table(ITW_TABLE(srgb_in_byte), (v >> 16) & 255u) << 16) | (v & 0xFF000000u);
    }
}

#if defined(__CUDACC__)
// One thread per destination texel: a warp writes 128 (RGBA8) or 256 (RGBA16F) contiguous bytes and reads
// 32 * planes * depth/8 contiguous source bytes.  Algorithmic traffic per texel: planes*depth/8 B in, 4 / 8 B out.
// General path (any alignment, any width).
__global__ void __launch_bounds__(256) front_kernel(FrontParams P, uint8_t* __restrict__ dst, int dst_w, int dst_h, long long dst_stride)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= dst_w || y >= dst_h) return;
    u32 out[2];
    front_texel(out, P, x, y);
    uint8_t* row = dst + (long long)y * dst_stride;
    if (P.family == 2) *reinterpret_cast<uint2*>(row + (long long)x * 8) = make_uint2(out[0], out[1]);
    else *reinterpret_cast<u32*>(row + (long long)x * 4) = out[0];
}
// NormalizeNormalMapChain over one stored (padded) level, in place: the plug-in normalises every level AFTER the mip
// chain exists (IP:2149-2152); per-texel, so it commutes with the edge replication of the padding.
__global__ void __launch_bounds__(256) normalize_kernel(uint8_t* __restrict__ ptr, int w, int h, long long stride, int hdr)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w || y >= h) return;
    if (hdr) {
        u32* p = reinterpret_cast<u32*>(ptr + (long long)y * stride + (long long)x * 8);
        u32 r = p[0] & 0xFFFFu, g = p[0] >> 16, b = p[1] & 0xFFFFu;
        const u32 a = p[1] >> 16;
        front_normalize_hdr(r, g, b);
        p[0] = r | (g << 16);
        p[1] = b | (a << 16);
    } else {
        u32* p = reinterpret_cast<u32*>(ptr + (long long)y * stride + (long long)x * 4);
        *p = front_normalize_rgba8(*p);
    }
}
// Layers into mip levels: every level of `P` in ONE launch, one thread per written texel, the levels back to back in the
// thread index (the small levels would otherwise be all launch overhead).  In place: a thread reads its own texel only when
// planes survive the copy, and the generated levels' padding already replicates their edge, so no thread reads another's.
__global__ void __launch_bounds__(256) layer_kernel(const __grid_constant__ LayerLaunch P)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int k = 0;
    while (k + 1 < P.count && i >= P.lv[k + 1].first) k++;
    const LayerLevel& L = P.lv[k];
    const long long j = i - L.first;
    if (j >= (long long)L.pw * L.ph) return;
    const int y = (int)(j / L.pw), x = (int)(j - (long long)y * L.pw);
    uint8_t* p = L.dst + (long long)y * L.dst_stride + (long long)x * (P.hdr ? 8 : 4);
    const bool keep = L.channels < 3;                       // alpha is always written
    u32 px[2] = {0u, 0u};
    if (P.hdr) {
        if (keep) { const uint2 t = *reinterpret_cast<const uint2*>(p); px[0] = t.x; px[1] = t.y; }
        layer_texel(px, L, P.depth, true, P.flip, x, y);
        *reinterpret_cast<uint2*>(p) = make_uint2(px[0], px[1]);
    } else {
        if (keep) px[0] = *reinterpret_cast<const u32*>(p);
        layer_texel(px, L, P.depth, false, P.flip, x, y);
        *reinterpret_cast<u32*>(p) = px[0];
    }
}
// Level 0 of all six faces of a cross document in ONE launch: blockIdx.z = face, blockIdx.y = row, one thread per texel.  Per texel
// planes*depth/8 B in, 4 / 8 B out; the document is read once in total (the cells do not overlap).
__global__ void __launch_bounds__(256) cube_faces_kernel(const __grid_constant__ CubeCross C)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, face = blockIdx.z;
    if (x >= C.w || y >= C.h) return;
    u32 out[2];
    cube_texel(out, C, face, x, y);
    uint8_t* row = C.dst + face * C.face_bytes + (long long)y * C.stride;
    if (C.P.family == 2) *reinterpret_cast<uint2*>(row + (long long)x * 8) = make_uint2(out[0], out[1]);
    else *reinterpret_cast<u32*>(row + (long long)x * 4) = out[0];
}
// Fast path: one thread per TWO quads of four destination texels -> 128-bit stores; the 4 * planes * depth/8 source
// bytes of a quad are contiguous and 4-byte aligned, and are fetched as 32-bit words into registers (all indices are
// compile-time constants; both quads' loads are issued before any conversion so that two requests per thread are in
// flight).  Needs dst_w % 4 == 0, 16-byte aligned dst rows and 4-byte aligned source rows; quads that touch the
// replicated edge fall back to the per-texel routine.
template <int kDepth, int kPlanes>
__global__ void __launch_bounds__(256) front_kernel_x4(FrontParams P, uint8_t* __restrict__ dst, int dst_w, int dst_h, long long dst_stride)
{
    constexpr int kWords = kPlanes * kDepth / 8;              // 32-bit words per quad
    constexpr int kQuads = 2;
    const int xbase = (blockIdx.x * blockDim.x + threadIdx.x) * 4 * kQuads, y = blockIdx.y;
    if (xbase >= dst_w || y >= dst_h) return;
    FrontParams Q = P;                                        // compile-time depth / planes for the conversion code
    Q.depth = kDepth;
    Q.planes = kPlanes;
    const bool vec = (kWords % 4 == 0) && ((reinterpret_cast<uintptr_t>(P.data) | (uintptr_t)P.row_bytes) & 15u) == 0;
    u32 wv[kQuads][kWords];
    bool inside[kQuads], live[kQuads];
#pragma unroll
    for (int q = 0; q < kQuads; q++) {
        const int x0 = xbase + 4 * q;
        live[q] = x0 < dst_w;
        inside[q] = live[q] && (x0 + 3 < P.width) && (y < P.height);
        if (inside[q]) {
            const u32* src = reinterpret_cast<const u32*>(P.data + (long long)y * P.row_bytes) + (long long)(x0 >> 2) * kWords;
            if (vec) {
#pragma unroll
                for (int i = 0; i < kWords / 4; i++) {
                    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src) + i);
                    wv[q][4 * i] = v.x; wv[q][4 * i + 1] = v.y; wv[q][4 * i + 2] = v.z; wv[q][4 * i + 3] = v.w;
                }
            } else {
#pragma unroll
                for (int i = 0; i < kWords; i++) wv[q][i] = __ldg(src + i);
            }
        }
    }
    uint8_t* row = dst + (long long)y * dst_stride;
#pragma unroll
    for (int q = 0; q < kQuads; q++) {
        if (!live[q]) continue;
        const int x0 = xbase + 4 * q;
        u32 out[4][2];
        if (inside[q]) {
#pragma unroll
            for (int t = 0; t < 4; t++) {
                u32 raw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int c = 0; c < kPlanes; c++) {
                    const int e = t * kPlanes + c;            // element index inside the quad
                    if (kDepth == 8) raw[c] = (wv[q][e >> 2] >> (8 * (e & 3))) & 255u;
                    else if (kDepth == 16) raw[c] = (wv[q][e >> 1] >> (16 * (e & 1))) & 0xFFFFu;
                    else raw[c] = wv[q][e];
                }
                front_compose(out[t], Q, raw);
            }
        } else {
#pragma unroll
            for (int t = 0; t < 4; t++) front_texel(out[t], Q, x0 + t, y);
        }
        if (P.family == 2) {
            uint4* o = reinterpret_cast<uint4*>(row + (long long)x0 * 8);
            o[0] = make_uint4(out[0][0], out[0][1], out[1][0], out[1][1]);
            o[1] = make_uint4(out[2][0], out[2][1], out[3][0], out[3][1]);
        } else {
            *reinterpret_cast<uint4*>(row + (long long)x0 * 4) = make_uint4(out[0][0], out[1][0], out[2][0], out[3][0]);
        }
    }
}
#endif

}  // namespace itw
