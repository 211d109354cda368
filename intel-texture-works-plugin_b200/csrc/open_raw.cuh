// open_raw.cuh -- THE OPEN PATH FOR UNCOMPRESSED FILES: what the plug-in's DoReadStart / DoReadContinue (IntelPlugin.cpp:2419-2742)
// do with a DDS file whose loaded format is already the read target (R8G8B8A8_UNORM, R8G8B8A8_UNORM_SRGB, R16G16B16A16_UNORM,
// R32G32B32A32_FLOAT), so that neither Decompress nor Convert runs (:2547-2553).
//
//   the loaded texel   LoadFromDDSMemory's _CopyImage (DirectXTexDDS.cpp:1024-1250): a plain row copy; for X8B8G8R8 _CopyScanline
//                      with TEXP_SCANLINE_SETALPHA (alpha 255); for the 24-bit R8G8B8 header _LegacyExpandScanline, which reads the
//                      three bytes as B, G, R ("24bpp Direct3D 9 files are actually BGR") and adds alpha 255.
//   alpha scan         ScratchImage::IsAlphaAllOpaque's non-compressed branch (DirectXTexImage.cpp:760-793): every texel of every
//                      image through _LoadScanline, "not opaque" when alpha < 0.99f.  Exact integer / float tests:
//                        UNORM8   XMLoadUByteN4 = byte * (1/255): 252/255 = 0.98824 < 0.99f < 253/255 = 0.99216  -> byte <= 252
//                        UNORM16  XMLoadUShortN4 = v * (1/65535): 64879 -> 0.989990, 64880 -> 0.990005         -> v <= 64879
//                        FLOAT    the stored float itself: a < 0.99f (so a NaN alpha counts as opaque)
//                      The margins (> 5e-6) are far above float rounding; tests/test_dds_open_uncompressed.py checks every byte,
//                      every ushort and the float edges against the cut branch.  The images of a DDS payload lie back to back with
//                      tight rows, so the payload is nothing but texels and the scan is one pass over its bytes.
//   layer store        one DoReadContinue (:2646-2727): channels 0..planes-1 of the loaded texel into the top-left corner of a zeroed
//                      layer of the top-level size; for a cube map with alpha the last plane is forced to 255 (depth 8), 1.0f
//                      (depth 32) or ConvertTo16Bit((unsigned8)255) = F32toF16(1.0f) = 0x3C00 (depth 16: a half-float bit pattern
//                      in a UNORM16 plane, IntelPlugin.h:77-80).  16-bit layers get the file's 0..65535 values unscaled, although
//                      Photoshop's 16-bit range is 0..32768 (IntelPlugin.h:62-63).  Both are the plug-in's behaviour, reproduced.
#pragma once
#include <cstring>
#include "open.cuh"

namespace itw {

// The loaded texel's source form: what the payload holds and how LoadFromDDSMemory turns it into the loaded format.
enum RawSource : int {
    kRawRgba8 = 0,      // R8G8B8A8_UNORM / _SRGB, copied
    kRawRgbx8 = 1,      // X8B8G8R8: R8G8B8A8_UNORM with alpha set to 255
    kRawBgr8 = 2,       // R8G8B8 (24 bpp): B, G, R bytes expanded to R8G8B8A8_UNORM with alpha 255
    kRawRgba16 = 3,     // R16G16B16A16_UNORM, copied
    kRawRgba32f = 4,    // R32G32B32A32_FLOAT, copied
    // The converted forms (itw_open_conv.inc): the loaded format, put through DirectX::Convert's _Convert into the target
    kConvRgba16f = 5,   // R16G16B16A16_FLOAT (10)        -> R16G16B16A16_UNORM
    kConvR16f = 6,      // R16_FLOAT (54)                 -> R16G16B16A16_UNORM
    kConvRg16f = 7,     // R16G16_FLOAT (34)              -> R16G16B16A16_UNORM
    kConvRgba16s = 8,   // R16G16B16A16_SNORM (13)        -> R16G16B16A16_UNORM
    kConvRg16 = 9,      // R16G16_UNORM (35)              -> R16G16B16A16_UNORM
    kConvRg16s = 10,    // R16G16_SNORM (37)              -> R16G16B16A16_UNORM
    kConvR16s = 11,     // R16_SNORM (58)                 -> R16G16B16A16_UNORM
    kConvR11g11b10f = 12,   // R11G11B10_FLOAT (26)       -> R16G16B16A16_UNORM
    kConvR9g9b9e5 = 13, // R9G9B9E5_SHAREDEXP (67)        -> R16G16B16A16_UNORM
    kConvRg8 = 14,      // R8G8_UNORM (49)                -> R8G8B8A8_UNORM
    kConvRg8s = 15,     // R8G8_SNORM (51)                -> R8G8B8A8_UNORM
    kConvRgba8s = 16,   // R8G8B8A8_SNORM (31)            -> R8G8B8A8_UNORM
    kConvR8s = 17,      // R8_SNORM (63)                  -> R8G8B8A8_UNORM
    kConvA8 = 18,       // A8_UNORM (65)                  -> R8G8B8A8_UNORM
    kConvBgra4 = 19,    // B4G4R4A4_UNORM (115)           -> R8G8B8A8_UNORM
    kConvBgrx4 = 20,    // X4R4G4B4: B4G4R4A4_UNORM with the alpha nibble set to 0xF on load (_CopyScanline, TEXP_SCANLINE_SETALPHA)
    kConvRg32f = 21,    // R32G32_FLOAT (16)              -> R32G32B32A32_FLOAT
    // The expanded forms (itw_open_exp.inc): LoadFromDDSMemory's _LegacyExpandScanline (DirectXTexDDS.cpp:726-1018) on load
    kExpA4l4 = 22,      // A4L4 (8 bpp): the 4:4 expansion into B4G4R4A4_UNORM (115), then kConvBgra4's _Convert -> R8G8B8A8_UNORM
    kExpA8r3g3b2 = 23,  // A8R3G3B2 (16 bpp): 3:3:2 bit replication into R8G8B8A8_UNORM, alpha the high byte
    kExpP8 = 24,        // P8 (8 bpp): the palette entry of the index, as R8G8B8A8_UNORM
    kExpA8p8 = 25       // A8P8 (16 bpp): the palette entry of the low byte, the high byte OR'd into its alpha
};
ITW_HD constexpr int raw_src_bytes(int src)
{
    return src == kRawBgr8 ? 3
         : src == kRawRgba16 || src == kConvRgba16f || src == kConvRgba16s || src == kConvRg32f ? 8
         : src == kRawRgba32f ? 16
         : src == kConvR16f || src == kConvR16s || src == kConvRg8 || src == kConvRg8s || src == kConvBgra4 || src == kConvBgrx4 ||
           src == kExpA8r3g3b2 || src == kExpA8p8 ? 2
         : src == kConvR8s || src == kConvA8 || src == kExpA4l4 || src == kExpP8 ? 1
         : 4;
}
// bytes of one plane of the target (the layer's depth / 8)
ITW_HD constexpr int raw_plane_bytes(int src)
{
    return src == kRawRgba32f || src == kConvRg32f ? 4 : src == kRawRgba16 || (src >= kConvRgba16f && src <= kConvR9g9b9e5) ? 2 : 1;
}
// The converted form of a loaded DXGI format, -1 for a format this path does not convert (X4R4G4B4 is chosen by its header).
ITW_HD constexpr int conv_kind_of(unsigned dxgi)
{
    return dxgi == 10 ? kConvRgba16f : dxgi == 54 ? kConvR16f : dxgi == 34 ? kConvRg16f : dxgi == 13 ? kConvRgba16s
         : dxgi == 35 ? kConvRg16 : dxgi == 37 ? kConvRg16s : dxgi == 58 ? kConvR16s : dxgi == 26 ? kConvR11g11b10f
         : dxgi == 67 ? kConvR9g9b9e5 : dxgi == 49 ? kConvRg8 : dxgi == 51 ? kConvRg8s : dxgi == 31 ? kConvRgba8s
         : dxgi == 63 ? kConvR8s : dxgi == 65 ? kConvA8 : dxgi == 115 ? kConvBgra4 : dxgi == 16 ? kConvRg32f : -1;
}
// DoReadStart's target of a converted form (:2534-2544): BitsPerColor > 16 -> 2, > 8 -> 11, else 28 (none of the forms is _SRGB); the
// layer depth is its plane width.
ITW_HD constexpr int conv_target_of(int src) { return raw_plane_bytes(src) == 4 ? 2 : raw_plane_bytes(src) == 2 ? 11 : 28; }
// HasAlpha(loaded format) (DirectXTexUtil.cpp): IsAlphaAllOpaque returns early without it (DirectXTexImage.cpp:749-750)
ITW_HD constexpr bool conv_has_alpha(int src)
{
    return src == kConvRgba16f || src == kConvRgba16s || src == kConvRgba8s || src == kConvA8 || src == kConvBgra4 || src == kConvBgrx4;
}

// The expanded header forms (ITW_EXP_P8, _A8P8, _A8R3G3B2, _A4L4 = 0..3 of itw_bcn.h section 16): the format LoadFromDDSMemory loads
// (g_LegacyDDSMap, DirectXTexDDS.cpp:84-125) and the texel form.  DoReadStart's target is 28 and the depth 8 for all four: A4L4's
// 115 goes through the non-WIC _Convert (as A4R4G4B4 does in section 14), the others are loaded as the target.
ITW_HD constexpr unsigned exp_loaded_of(int form) { return form == 3 ? 115u : 28u; }
ITW_HD constexpr int exp_kind_of(int form) { return form == 0 ? kExpP8 : form == 1 ? kExpA8p8 : form == 2 ? kExpA8r3g3b2 : kExpA4l4; }
ITW_HD constexpr bool exp_has_palette(int form) { return form == 0 || form == 1; }

// The alpha decision of one loaded texel from the word that holds its alpha (the texel's last 32 bits): true when alpha < 0.99f.
// Converted forms (the loaders of _LoadScanline, restated below; exact tests on the stored bits where the margins allow):
//   R16G16B16A16_FLOAT  XMConvertHalfToFloat(a) < 0.99f, compared as a float (exponent 31 is a large finite value, never NaN)
//   R16G16B16A16_SNORM  XMLoadShortN4 = max(-1, s * (1/32767)): 32439 -> 0.989990, 32440 -> 0.990020       -> s <= 32439
//   R8G8B8A8_SNORM      XMLoadByteN4 = max(-1, c * (1/127)): 125 -> 0.984252, 126 -> 0.992126              -> c <= 125
//   A8_UNORM            byte / 255.f (the hand-written loop): 252 -> 0.988235, 253 -> 0.992157           -> byte <= 252
//   B4G4R4A4_UNORM      nibble * (1/15) (XMLoadUNibble4 * s_Scale): 14 -> 0.933333, 15 -> 1.0               -> nibble <= 14
// A word holds one alpha (texels of 4 bytes or more), two (4444: the top nibble of each ushort) or four (A8: every byte).
template <int kSrc>
ITW_HD bool raw_alpha_below(u32 word)
{
    if constexpr (kSrc == kRawRgba16) return (word >> 16) <= 64879u;
    else if constexpr (kSrc == kRawRgba32f) {
        float a;
        memcpy(&a, &word, 4);
        return a < 0.99f;
    } else if constexpr (kSrc == kConvRgba16f) {
        return front_float_from_half(word >> 16) < 0.99f;
    } else if constexpr (kSrc == kConvRgba16s) {
        return (int)(short)(word >> 16) <= 32439;
    } else if constexpr (kSrc == kConvRgba8s) {
        return (int)(signed char)(word >> 24) <= 125;
    } else if constexpr (kSrc == kConvA8) {
        return (word & 0xFFu) <= 252u || ((word >> 8) & 0xFFu) <= 252u || ((word >> 16) & 0xFFu) <= 252u || (word >> 24) <= 252u;
    } else if constexpr (kSrc == kConvBgra4) {
        return ((word >> 12) & 0xFu) <= 14u || (word >> 28) <= 14u;
    } else if constexpr (kSrc == kExpA8r3g3b2) {          // the loaded alpha is the high byte of each ushort
        return ((word >> 8) & 0xFFu) <= 252u || (word >> 24) <= 252u;
    } else if constexpr (kSrc == kExpA4l4) {              // the loaded 4444 alpha is the high nibble of each byte
        return ((word >> 4) & 0xFu) <= 14u || ((word >> 12) & 0xFu) <= 14u || ((word >> 20) & 0xFu) <= 14u || (word >> 28) <= 14u;
    } else {
        return (word >> 24) <= 252u;
    }
}
// The same for the palettised forms, whose loaded alpha is the palette entry's fourth byte (D3D9's peFlags; P8), OR'd with the
// texel's high byte (A8P8): UNORM8 `<= 252`.  `alpha` holds the 256 entries' alpha bytes; the first `n` texels of the word are tested
// (a payload's last word may be partial, and an index no texel holds never counts).
template <int kSrc>
ITW_HD bool pal_alpha_below(const uint8_t* alpha, u32 word, int n)
{
    bool below = false;
    if constexpr (kSrc == kExpP8) {
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (k < n) below |= alpha[(word >> (8 * k)) & 0xFFu] <= 252u;
    } else {
#pragma unroll
        for (int k = 0; k < 2; k++)
            if (k < n) below |= ((u32)alpha[(word >> (16 * k)) & 0xFFu] | ((word >> (16 * k + 8)) & 0xFFu)) <= 252u;
    }
    return below;
}

// mul_rn / add_rn / div_rn, conv_saturate and the target stores conv_unorm16 / conv_unorm8 are open.cuh's.
// XMLoadShortN* / XMLoadByteN* (DirectXMath 3.06): the integer times the rounded reciprocal, clamped at -1 (-32768 and -128)
ITW_HD float conv_snorm16(u32 bits) { const float v = mul_rn((float)(int)(short)bits, 1.0f / 32767.0f); return v > -1.0f ? v : -1.0f; }
ITW_HD float conv_snorm8(u32 bits) { const float v = mul_rn((float)(int)(signed char)bits, 1.0f / 127.0f); return v > -1.0f ? v : -1.0f; }
// One channel of XMLoadFloat3PK (DirectXMath 3.06): an unsigned float of a 5-bit exponent and an m-bit mantissa, exactly; exponent 31
// is Inf / NaN.
template <int kMant>
ITW_HD float conv_packed_float(u32 f)
{
    u32 mant = f & ((1u << kMant) - 1u), exp = f >> kMant;
    if (exp == 31u) return bits_float(0x7F800000u | (mant << (23 - kMant)));
    if (exp == 0u) {
        if (mant) {
            exp = 1u;
            do { exp--; mant <<= 1; } while (!(mant & (1u << kMant)));
            mant &= (1u << kMant) - 1u;
        } else {
            exp = (u32)-112;
        }
    }
    return bits_float(((exp + 112u) << 23) | (mant << (23 - kMant)));
}

// _LegacyExpandScanline's rows of the expanded forms (DirectXTexDDS.cpp:807-916), per texel, without TEXP_SCANLINE_SETALPHA (none of
// the four entries has CONV_FLAGS_NOALPHA).  A4L4 -> B4G4R4A4_UNORM: the luminance nibble into blue, green and red, alpha on top.
ITW_HD u32 exp_a4l4_word(u32 t) { const u32 l = t & 0x0Fu; return l | (l << 4) | (l << 8) | ((t & 0xF0u) << 8); }
// The R8G8B8A8_UNORM word of the texel at `p`: A8R3G3B2 by bit replication, P8 / A8P8 through `pal` (the file's 256 palette words).
template <int kSrc>
ITW_HD u32 exp_rgba8_word(const uint8_t* p, const u32* pal)
{
    if constexpr (kSrc == kExpP8) {
        return pal[p[0]];
    } else {
        const u32 t = (u32)p[0] | ((u32)p[1] << 8);
        if constexpr (kSrc == kExpA8p8) return pal[t & 0xFFu] | ((t & 0xFF00u) << 16);
        else return (t & 0xE0u) | ((t & 0xE0u) >> 3) | ((t & 0xC0u) >> 6)
                  | ((t & 0x1Cu) << 11) | ((t & 0x1Cu) << 8) | ((t & 0x18u) << 5)
                  | ((t & 0x03u) << 22) | ((t & 0x03u) << 20) | ((t & 0x03u) << 18) | ((t & 0x03u) << 16) | ((t & 0xFF00u) << 16);
    }
}

// The converted texel at `p` (4-byte aligned when its texel has 4 bytes or more) as the target's planes: DirectX::Convert's _Convert
// with filter 0 (DirectXTexConvert.cpp:4321-4400) for one texel.  _LoadScanline's case of the loaded format gives (r, g, b, a) floats
// (absent channels 0, alpha 1); _ConvertScanline(target, loaded, 0) then applies, for these pairs, SNORM -> UNORM v * 0.5 + 0.5 on all
// four channels, FLOAT -> UNORM saturate, or nothing (UNORM, the shared exponent, FLOAT -> FLOAT), followed by the R -> RGB splat of
// the one-channel formats; _StoreScanline rounds into the target.  Every product and sum rounds on its own, as in the reference.
template <int kSrc>
ITW_HD void conv_texel(const uint8_t* p, u32 (&o)[4])
{
    float c[4] = {0.0f, 0.0f, 0.0f, 1.0f};
    if constexpr (kSrc == kConvRg32f) {                  // XMLoadFloat2 and XMStoreFloat4: bit copies, (r, g, 0, 1)
        o[0] = reinterpret_cast<const u32*>(p)[0];
        o[1] = reinterpret_cast<const u32*>(p)[1];
        o[2] = 0u;
        o[3] = 0x3F800000u;
        return;
    } else if constexpr (kSrc == kConvRgba16f || kSrc == kConvRgba16s) {
        const u32 lo = reinterpret_cast<const u32*>(p)[0], hi = reinterpret_cast<const u32*>(p)[1];
        const u32 h[4] = {lo & 0xFFFFu, lo >> 16, hi & 0xFFFFu, hi >> 16};
#pragma unroll
        for (int k = 0; k < 4; k++) c[k] = kSrc == kConvRgba16f ? front_float_from_half(h[k]) : conv_snorm16(h[k]);
    } else if constexpr (kSrc == kConvRg16f || kSrc == kConvRg16 || kSrc == kConvRg16s) {
        const u32 w = *reinterpret_cast<const u32*>(p);
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const u32 h = (w >> (16 * k)) & 0xFFFFu;
            c[k] = kSrc == kConvRg16f ? front_float_from_half(h) : kSrc == kConvRg16s ? conv_snorm16(h) : mul_rn((float)h, 1.0f / 65535.0f);
        }
    } else if constexpr (kSrc == kConvR16f) {
        c[0] = front_float_from_half((u32)p[0] | ((u32)p[1] << 8));
    } else if constexpr (kSrc == kConvR16s) {            // the hand-written loop: a true division, no clamp
        c[0] = div_rn((float)(int)(short)((u32)p[0] | ((u32)p[1] << 8)), 32767.0f);
    } else if constexpr (kSrc == kConvR11g11b10f) {
        const u32 w = *reinterpret_cast<const u32*>(p);
        c[0] = conv_packed_float<6>(w & 0x7FFu);
        c[1] = conv_packed_float<6>((w >> 11) & 0x7FFu);
        c[2] = conv_packed_float<5>(w >> 22);
    } else if constexpr (kSrc == kConvR9g9b9e5) {        // XMLoadFloat3SE: 2^(e - 24) times each 9-bit mantissa, exactly
        const u32 w = *reinterpret_cast<const u32*>(p);
        const float scale = bits_float(0x33800000u + ((w >> 27) << 23));
#pragma unroll
        for (int k = 0; k < 3; k++) c[k] = mul_rn(scale, (float)((w >> (9 * k)) & 0x1FFu));
    } else if constexpr (kSrc == kConvRg8) {
        c[0] = mul_rn((float)p[0], 1.0f / 255.0f);
        c[1] = mul_rn((float)p[1], 1.0f / 255.0f);
    } else if constexpr (kSrc == kConvRg8s) {
        c[0] = conv_snorm8(p[0]);
        c[1] = conv_snorm8(p[1]);
    } else if constexpr (kSrc == kConvRgba8s) {
        const u32 w = *reinterpret_cast<const u32*>(p);
#pragma unroll
        for (int k = 0; k < 4; k++) c[k] = conv_snorm8(w >> (8 * k));
    } else if constexpr (kSrc == kConvR8s) {             // the hand-written loop: a true division, no clamp
        c[0] = div_rn((float)(int)(signed char)p[0], 127.0f);
    } else if constexpr (kSrc == kConvA8) {              // (0, 0, 0, byte / 255.f)
        c[3] = div_rn((float)p[0], 255.0f);
    } else if constexpr (kSrc == kConvBgra4 || kSrc == kConvBgrx4 || kSrc == kExpA4l4) {   // XMLoadUNibble4 * (1/15), swizzled <2, 1, 0, 3>
        const u32 w = kSrc == kExpA4l4 ? exp_a4l4_word(p[0]) : (u32)p[0] | ((u32)p[1] << 8) | (kSrc == kConvBgrx4 ? 0xF000u : 0u);
#pragma unroll
        for (int k = 0; k < 4; k++) c[k] = mul_rn((float)((w >> (4 * (k == 3 ? 3 : 2 - k))) & 0xFu), 1.0f / 15.0f);
    }
    constexpr bool kSnorm = kSrc == kConvRgba16s || kSrc == kConvRg16s || kSrc == kConvR16s || kSrc == kConvRg8s || kSrc == kConvRgba8s ||
                            kSrc == kConvR8s;
    constexpr bool kFloat = kSrc == kConvRgba16f || kSrc == kConvR16f || kSrc == kConvRg16f || kSrc == kConvR11g11b10f;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (kSnorm) c[k] = add_rn(mul_rn(c[k], 0.5f), 0.5f);      // XMVectorMultiplyAdd(v, g_XMOneHalf, g_XMOneHalf)
        if (kFloat) c[k] = conv_saturate(c[k]);
    }
    if (kSrc == kConvR16f || kSrc == kConvR16s || kSrc == kConvR8s) c[1] = c[2] = c[0];   // R format -> RGB format
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = raw_plane_bytes(kSrc) == 2 ? conv_unorm16(c[k]) : conv_unorm8(c[k]);
}

// The loaded texel at `p` (4-byte aligned unless kRawBgr8 or a form of fewer than 4 bytes) as four plane values of the target: bytes,
// ushorts or float bit patterns.  `pal`: the palette of kExpP8 / kExpA8p8.
template <int kSrc>
ITW_HD void raw_load_texel(const uint8_t* p, u32 (&v)[4], const u32* pal = nullptr)
{
    if constexpr (kSrc >= kExpA8r3g3b2) {
        const u32 w = exp_rgba8_word<kSrc>(p, pal);
#pragma unroll
        for (int c = 0; c < 4; c++) v[c] = (w >> (8 * c)) & 0xFFu;
    } else if constexpr (kSrc >= kConvRgba16f) {
        conv_texel<kSrc>(p, v);
    } else if constexpr (kSrc == kRawBgr8) {
        v[0] = p[2]; v[1] = p[1]; v[2] = p[0]; v[3] = 255u;
    } else if constexpr (kSrc == kRawRgba8 || kSrc == kRawRgbx8) {
        const u32 w = *reinterpret_cast<const u32*>(p);
#pragma unroll
        for (int c = 0; c < 4; c++) v[c] = (w >> (8 * c)) & 0xFFu;
        if (kSrc == kRawRgbx8) v[3] = 255u;
    } else if constexpr (kSrc == kRawRgba16) {
        const u32 lo = reinterpret_cast<const u32*>(p)[0], hi = reinterpret_cast<const u32*>(p)[1];
        v[0] = lo & 0xFFFFu; v[1] = lo >> 16; v[2] = hi & 0xFFFFu; v[3] = hi >> 16;
    } else {
#pragma unroll
        for (int c = 0; c < 4; c++) v[c] = reinterpret_cast<const u32*>(p)[c];
    }
}

// DoReadContinue's per-texel rule: the loaded texel's planes, with the last of kPlanes forced for a cube map with alpha.
template <int kSrc, int kPlanes>
ITW_HD void raw_layer_texel(const u32 (&v)[4], bool force_alpha, u32 (&o)[4])
{
    constexpr u32 kForced = raw_plane_bytes(kSrc) == 2 ? 0x3C00u : raw_plane_bytes(kSrc) == 4 ? 0x3F800000u : 255u;
#pragma unroll
    for (int c = 0; c < 4; c++) o[c] = c < kPlanes ? v[c] : 0u;
    if (force_alpha) o[kPlanes - 1] = kForced;
}

#if defined(__CUDACC__)
// The scan of `bytes` payload bytes of kSrc texels (kRawRgba8, kRawRgba16, kRawRgba32f, a converted form with alpha or an expanded form) at a 4-byte
// aligned `payload`: *flag becomes 1 if any texel is not opaque.  The bytes up to the first 16-byte boundary and after the last one are
// read as words by the first threads; the body goes in 16-byte loads, grid-stride, four loads in flight per thread.  Word j of the
// payload holds an alpha when j % (texel words) is the texel's last word; texels of one or two bytes put alphas in every word, and
// their payload may end in a partial word, which one more thread reads byte by byte (its missing bytes padded with opaque ones).
// below(word, n): whether a texel among the first n bytes of the word is not opaque.
template <int kSrc, class Below>
__device__ __forceinline__ void raw_alpha_scan(const uint8_t* __restrict__ payload, long long bytes, int* __restrict__ flag,
                                               const Below& below_of)
{
    constexpr int kTexelWords = raw_src_bytes(kSrc) >= 4 ? raw_src_bytes(kSrc) / 4 : 1;
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x, threads = (long long)gridDim.x * blockDim.x;
    const long long to16 = (long long)((16u - (unsigned)(reinterpret_cast<uintptr_t>(payload) & 15u)) & 15u);
    const long long head = to16 < bytes ? to16 : bytes;
    const long long n16 = (bytes - head) >> 4, tail = head + (n16 << 4);
    const u32* words = reinterpret_cast<const u32*>(payload);
    bool below = false;
    // the words outside the 16-byte body: `head / 4` before it, the rest after it
    const long long edge = head / 4 + (bytes - tail) / 4;
    if (id < edge) {
        const long long j = id < head / 4 ? id : tail / 4 + (id - head / 4);
        if (j % kTexelWords == kTexelWords - 1) below = below_of(__ldg(words + j), 4);
    }
    if constexpr (raw_src_bytes(kSrc) < 4) {
        if (id == edge && (bytes & 3)) {
            u32 w = 0xFFFFFFFFu;
            for (long long b = bytes & ~3LL; b < bytes; b++) w = (w & ~(0xFFu << (8 * (b & 3)))) | ((u32)payload[b] << (8 * (b & 3)));
            below = below_of(w, (int)(bytes & 3));
        }
    }
    // which of a body vector's four words hold an alpha (the body starts at word head / 4)
    u32 lanes = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
        if ((head / 4 + k) % kTexelWords == kTexelWords - 1) lanes |= 1u << k;
    const uint4* body = reinterpret_cast<const uint4*>(payload + head);
    for (long long i = id; i < n16; i += 4 * threads) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = i + u * threads < n16 ? __ldg(body + i + u * threads) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (i + u * threads >= n16) break;
            const u32 w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
            for (int k = 0; k < 4; k++)
                if ((lanes >> k) & 1u) below |= below_of(w[k], 4);
        }
    }
    if (__any_sync(0xFFFFFFFFu, below) && (threadIdx.x & 31) == 0) *flag = 1;
}
template <int kSrc>
__global__ void __launch_bounds__(256) open_raw_alpha_kernel(const uint8_t* __restrict__ payload, long long bytes, int* __restrict__ flag)
{
    raw_alpha_scan<kSrc>(payload, bytes, flag, [](u32 w, int) { return raw_alpha_below<kSrc>(w); });
}

// A P8 / A8P8 file's palette, passed to the kernels by value (1 KB of kernel parameters) and copied to shared memory at CTA start, so
// that every CTA holds it and a layer call stages only the image it reads.
struct RawPalette {
    u32 e[256];
};
// The scan of the palettised forms: open_raw_alpha_kernel's pass with the palette's alpha bytes in shared memory.  256 threads.
template <int kSrc>
__global__ void __launch_bounds__(256) open_pal_alpha_kernel(const uint8_t* __restrict__ payload, long long bytes, int* __restrict__ flag,
                                                             const __grid_constant__ RawPalette pal)
{
    __shared__ uint8_t alpha[256];
    alpha[threadIdx.x] = (uint8_t)(pal.e[threadIdx.x] >> 24);
    __syncthreads();
    raw_alpha_scan<kSrc>(payload, bytes, flag, [&](u32 w, int n) { return pal_alpha_below<kSrc>(alpha, w, n / raw_src_bytes(kSrc)); });
}

// One layer: `dst` holds `height` rows of `width` texels of kPlanes planes of raw_plane_bytes(kSrc) bytes, rows `row_bytes` apart;
// dst and row_bytes are 16-byte aligned.  The image (iw x ih texels of raw_src_bytes(kSrc) bytes, tight rows at `src`, 4-byte aligned
// unless kRawBgr8) lands in the top-left corner, zeros elsewhere.  A warp covers 128 texels of one layer row: each lane builds four
// texels and store_staged_row writes the row with 16-byte stores.  force_alpha: the last plane of every image texel is forced.
// `pal`: the palette of kExpP8 / kExpA8p8.
template <int kSrc, int kPlanes>
__device__ __forceinline__ void raw_layer_rows(const uint8_t* __restrict__ src, int iw, int ih, uint8_t* __restrict__ dst, int width,
                                               int height, long long row_bytes, bool force_alpha, const u32* pal)
{
    constexpr int kPlaneBytes = raw_plane_bytes(kSrc), kSrcBytes = raw_src_bytes(kSrc);
    constexpr int kTexel = kPlanes * kPlaneBytes;              // bytes per layer texel: 3, 4, 6, 8, 12 or 16
    constexpr int kTileRow = 4 * kTexel;                       // bytes of one lane's four texels
    __shared__ uint4 stage[8][staged_row_slots(kTileRow)];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunks = (width + 127) >> 7;
    const long long g = (long long)blockIdx.x * 8 + warp;      // warp-uniform: (layer row, chunk of 128 texels)
    if (g >= (long long)height * chunks) return;
    const int Y = (int)(g / chunks), chunk = (int)(g - (long long)Y * chunks), x0 = 128 * chunk + 4 * lane;
    const uint8_t* srow = src + ((long long)Y * iw + x0) * kSrcBytes;
    u32 t[kTileRow / 4];
#pragma unroll
    for (int i = 0; i < kTileRow / 4; i++) t[i] = 0u;
#pragma unroll
    for (int x = 0; x < 4; x++) {
        if (Y >= ih || x0 + x >= iw) break;
        u32 v[4], o[4];
        raw_load_texel<kSrc>(srow + x * kSrcBytes, v, pal);
        raw_layer_texel<kSrc, kPlanes>(v, force_alpha, o);
#pragma unroll
        for (int c = 0; c < kPlanes; c++) {
            const int b = (x * kPlanes + c) * kPlaneBytes;     // byte offset in the lane's piece; a plane never straddles a word
            t[b >> 2] |= o[c] << (8 * (b & 3));
        }
    }
    const int span = min(128, width - 128 * chunk) * kTexel;
    store_staged_row<kTileRow>(stage[warp], lane, x0 < width, t, span, dst + (long long)Y * row_bytes + (long long)chunk * 128 * kTexel);
}
template <int kSrc, int kPlanes>
__global__ void __launch_bounds__(256) open_raw_layer_kernel(const uint8_t* __restrict__ src, int iw, int ih, uint8_t* __restrict__ dst,
                                                             int width, int height, long long row_bytes, bool force_alpha)
{
    raw_layer_rows<kSrc, kPlanes>(src, iw, ih, dst, width, height, row_bytes, force_alpha, nullptr);
}
// The layer of an expanded form: for P8 / A8P8 the palette in shared memory first, then open_raw_layer_kernel's rows.  256 threads.
// At least four CTAs per SM: ptxas's default budget for these rows (40 registers) spills the store's byte tail around its copy loop.
template <int kSrc, int kPlanes>
__global__ void __launch_bounds__(256, 4) open_exp_layer_kernel(const uint8_t* __restrict__ src, int iw, int ih, uint8_t* __restrict__ dst,
                                                                int width, int height, long long row_bytes, bool force_alpha,
                                                                const __grid_constant__ RawPalette pal)
{
    __shared__ u32 spal[kSrc == kExpP8 || kSrc == kExpA8p8 ? 256 : 1];
    if constexpr (kSrc == kExpP8 || kSrc == kExpA8p8) {
        spal[threadIdx.x] = pal.e[threadIdx.x];
        __syncthreads();
    }
    raw_layer_rows<kSrc, kPlanes>(src, iw, ih, dst, width, height, row_bytes, force_alpha, spal);
}
#endif

}  // namespace itw
