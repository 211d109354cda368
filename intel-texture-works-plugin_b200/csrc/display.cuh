// display.cuh -- DECOMPRESS FOR DISPLAY: one BC block -> 16 texels of a TARGET format, the rules of DirectX::Decompress
// (DirectXTexCompress.cpp:358-468: _DecompressBC -> _ConvertScanline(temp, 16, target, source, 0) -> _StoreScanline), which the
// plug-in's preview runs after every encode (IntelPlugin.cpp:1024-1059).
//
//   source                    target                      rule
//   BC1/3/5/7 UNORM           R8G8B8A8_UNORM (28)         kDisplayPlain: the bytes of decode_kernel
//   BC4 UNORM                 28                          kDisplayPlain, red copied into green and blue (r, r, r, 255): BC4 is an
//                                                         R format and the target an RGB one, so _ConvertScanline's channel-mask
//                                                         branch "R format -> RGB format" splats red (DirectXTexConvert.cpp:3445-3457)
//   BC1/3/7 _SRGB             28                          kDisplaySrgbIn: XMColorSRGBToRGB on r, g, b, then the UNORM8 store
//   BC1/3/7 _SRGB             R8G8B8A8_UNORM_SRGB (29)    kDisplayPlain: SRGB in and SRGB out cancel (DirectXTexConvert.cpp:3042-3045)
//   BC1/3/4/5/7 UNORM         29                          kDisplaySrgbOut: XMColorRGBToSRGB on r, g, b, then the UNORM8 store
//                                                         (BC4: the red splat first, so (s, s, s, 255))
// No other branch of _ConvertScanline's special cases (:3060-3557) changes these pairs: BC1/3/7 and BC6H are RGBA like the targets,
// BC5 is RG (no channel branch matches RG -> RGB).
//   BC6H UF16 / SF16          28                          kDisplayHdrUnorm: half -> float -> saturate (FLOAT -> UNORM, :3340-3350) -> store
//   BC6H UF16 / SF16          R32G32B32A32_FLOAT (2)      kDisplayHdrFloat: half -> float exactly, alpha 1.0
//
// Which float each decoder hands to _ConvertScanline (that is what the sRGB curves see):
//   BC1, BC3 colour   DecodeBC1's own float endpoints n*(1/31), n*(1/63) and interpolants (f1-f0)*t+f0 (BC.cpp:322-370).  The stored
//                     byte is a monotone step function of that float: 255 thresholds (srgb_in_threshold for SRGB in, srgb_tables.cuh's
//                     linear_threshold for SRGB out), counted by an 8-step search -- no pow on the GPU.
//   BC3 alpha         never converted (the sRGB curves leave alpha alone, :2771), so the integer ramp of decode_alpha stands.
//   BC4, BC5          BC4_UNORM::DecodeFromIndex (BC4BC5.cpp:50-70): r0/255.0f, r1/255.0f and (f0*(7-i) + f1*i)/7.0f, (.../5.0f),
//                     0.0f, 1.0f -- re-evaluated here for the SRGB-out rule (bc4_float) and counted against linear_threshold.
//   BC7               byte * (1/255) (HDRColorA from LDRColorA, BC.h:152-155): a byte -> byte table per direction.
//   BC6H              the half bit patterns of decode_bc6h, widened by XMConvertHalfToFloat (front_float_from_half, DirectXMath 3.06).
// Tables: display_tables.cuh, generated from the oracle's own sRGB functions by tools/gen_display_tables.py.
//
// One thread per block, as decode_kernel: 8/16 B in, 64 B (RGBA8) or 256 B (RGBA32F) out.  Texels outside width x height are not
// written (_DecompressBC's ragged edge blocks, :424-465); whole blocks of an aligned surface leave through 128-bit row stores.
#pragma once
#include "decode.cuh"
#include "mips_f16.cuh"
#include "display_tables.cuh"

namespace itw {

ITW_TABLE_DECL(uint32_t, srgb_in_threshold, 255)
ITW_TABLE_DECL(uint32_t, srgb_out_byte, 64)      // srgb_in_byte and byte_table: frontend.cuh

enum DisplayRule { kDisplayPlain = 0, kDisplaySrgbIn = 1, kDisplaySrgbOut = 2, kDisplayHdrUnorm = 3, kDisplayHdrFloat = 4 };

// Number of entries of a sorted 255-entry threshold table that are <= f: the stored byte.  Signed compare of the bit patterns, so
// every negative float (and -0) counts 0; the thresholds are positive.
ITW_HD u32 threshold_count(const uint32_t* T, float f)
{
    const int b = (int)float_bits(f);
    int k = 0;
#pragma unroll
    for (int s = 128; s; s >>= 1)
        if ((int)T[k + s - 1] <= b) k += s;
    return (u32)k;
}

struct SrgbInStore { ITW_HD static u32 of(float x) { return threshold_count(ITW_TABLE(srgb_in_threshold), x); } };
struct SrgbOutStore { ITW_HD static u32 of(float x) { return threshold_count(ITW_TABLE(linear_threshold), x); } };

// BC4_UNORM::DecodeFromIndex (BC4BC5.cpp:50-70) in its own float operations
ITW_HD float bc4_float(u32 a0, u32 a1, u32 q)
{
    const float f0 = (float)a0 / 255.0f, f1 = (float)a1 / 255.0f;
    if (q == 0u) return f0;
    if (q == 1u) return f1;
    if (a0 > a1) {
        q -= 1u;
        return (f0 * (float)(7u - q) + f1 * (float)q) / 7.0f;
    }
    if (q == 6u) return 0.0f;
    if (q == 7u) return 1.0f;
    q -= 1u;
    return (f0 * (float)(5u - q) + f1 * (float)q) / 5.0f;
}
// one BC4 channel block -> 16 sRGB-encoded bytes (the eight palette floats are converted once)
ITW_HD void display_bc4_srgb_out(u32 (&val)[16], u32 w0, u32 w1)
{
    const u32 a0 = w0 & 255u, a1 = (w0 >> 8) & 255u;
    const unsigned long long idx = ((unsigned long long)w1 << 16) | (w0 >> 16);
    unsigned long long pal = 0ull;
#pragma unroll
    for (u32 q = 0; q < 8; q++) pal |= (unsigned long long)SrgbOutStore::of(bc4_float(a0, a1, q)) << (8 * q);
#pragma unroll
    for (int k = 0; k < 16; k++) val[k] = (u32)(pal >> (8 * ((u32)(idx >> (3 * k)) & 7u))) & 255u;
}

// kDisplayHdrUnorm's element: half -> float (XMLoadHalf4), FLOAT -> UNORM saturate (_ConvertScanline, :3340-3350), UNORM8 store.
// Also the whole of the non-WIC _Convert(R16G16B16A16_FLOAT -> R8G8B8A8_UNORM) of the HDR original pane, channel by channel.
ITW_HD u32 display_hdr_unorm8(u32 half) { return mip_unorm8_store(front_float_from_half(half)); }

// ---- one block -> 16 RGBA8 texels (targets 28 / 29); kFormat is the decoder (71/77/80/83/98), kRule a DisplayRule ----
template <int kFormat, int kRule>
ITW_HD void display_block_rgba8(u32 (&px)[16], const u32 (&w)[4])
{
    if (kFormat == 95 || kFormat == 96) {                         // BC6H -> R8G8B8A8_UNORM: FLOAT -> UNORM saturates, then the store
        u32 h[16][2];
        decode_bc6h<kFormat == 96>(h, w);
#pragma unroll
        for (int k = 0; k < 16; k++)
            px[k] = display_hdr_unorm8(h[k][0] & 0xFFFFu) | (display_hdr_unorm8(h[k][0] >> 16) << 8) | (display_hdr_unorm8(h[k][1] & 0xFFFFu) << 16) |
                    0xFF000000u;
        return;
    }
    if (kFormat == 80) {                                          // R format -> RGB format (:3445-3457): red copied into green and blue
        u32 r[16];
        if (kRule == kDisplayPlain) decode_alpha(r, w[0], w[1]);
        else display_bc4_srgb_out(r, w[0], w[1]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = r[k] * 0x010101u | 0xFF000000u;
        return;
    }
    if (kRule == kDisplayPlain) {
        decode_block_rgba8<kFormat>(px, w);
        return;
    }
    if (kFormat == 71 || kFormat == 77) {
        const u32 c0 = (kFormat == 71) ? w[0] : w[2], c1 = (kFormat == 71) ? w[1] : w[3];
        if (kRule == kDisplaySrgbIn) decode_bc1_colour_as<SrgbInStore>(px, c0, c1, kFormat == 77);
        else decode_bc1_colour_as<SrgbOutStore>(px, c0, c1, kFormat == 77);
        if (kFormat == 77) {
            u32 a[16];
            decode_alpha(a, w[0], w[1]);
#pragma unroll
            for (int k = 0; k < 16; k++) px[k] = (px[k] & 0x00FFFFFFu) | (a[k] << 24);
        }
    } else if (kFormat == 83) {                                   // UNORM only, so kDisplaySrgbOut; b = 0 stays 0, alpha 1.0
        u32 r[16], g[16];
        display_bc4_srgb_out(r, w[0], w[1]);
        display_bc4_srgb_out(g, w[2], w[3]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = r[k] | (g[k] << 8) | 0xFF000000u;
    } else {
        decode_bc7(px, w);
        const uint32_t* T = (kRule == kDisplaySrgbIn) ? ITW_TABLE(srgb_in_byte) : ITW_TABLE(srgb_out_byte);
#pragma unroll
        for (int k = 0; k < 16; k++)
            px[k] = byte_table(T, px[k] & 255u) | (byte_table(T, (px[k] >> 8) & 255u) << 8) | (byte_table(T, (px[k] >> 16) & 255u) << 16) |
                    (px[k] & 0xFF000000u);
    }
}
// ---- BC6H -> R32G32B32A32_FLOAT: 16 texels x 4 float bit patterns ----
template <int kFormat>
ITW_HD void display_block_f32(u32 (&px)[16][4], const u32 (&w)[4])
{
    u32 h[16][2];
    decode_bc6h<kFormat == 96>(h, w);
#pragma unroll
    for (int k = 0; k < 16; k++) {
        px[k][0] = float_bits(front_float_from_half(h[k][0] & 0xFFFFu));
        px[k][1] = float_bits(front_float_from_half(h[k][0] >> 16));
        px[k][2] = float_bits(front_float_from_half(h[k][1] & 0xFFFFu));
        px[k][3] = 0x3F800000u;
    }
}

#if defined(__CUDACC__)
// dst rows `stride` bytes apart; texel (x, y) at dst + y*stride + x*texel (4 B, or 16 B for kDisplayHdrFloat).  kVec16: dst and
// stride are 16-byte aligned (otherwise 4-byte aligned).
template <int kFormat, int kRule, bool kVec16>
__global__ void __launch_bounds__(128) display_kernel(const uint8_t* __restrict__ blocks, uint8_t* __restrict__ dst, int width, int height,
                                                      long long stride)
{
    const int bw = (width + 3) >> 2, bh = (height + 3) >> 2;
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
    const int cols = min(4, width - 4 * bx), rows = min(4, height - 4 * by);
    if (kRule == kDisplayHdrFloat) {
        u32 px[16][4];
        display_block_f32<kFormat>(px, w);
        uint8_t* row = dst + (long long)(4 * by) * stride + (long long)bx * 64;
#pragma unroll
        for (int y = 0; y < 4; y++, row += stride) {
            if (y >= rows) break;
#pragma unroll
            for (int x = 0; x < 4; x++) {
                if (x >= cols) break;
                const u32* t = px[4 * y + x];
                if (kVec16) reinterpret_cast<uint4*>(row)[x] = make_uint4(t[0], t[1], t[2], t[3]);
                else {
#pragma unroll
                    for (int c = 0; c < 4; c++) reinterpret_cast<u32*>(row)[4 * x + c] = t[c];
                }
            }
        }
    } else {
        u32 px[16];
        display_block_rgba8<kFormat, kRule>(px, w);
        uint8_t* row = dst + (long long)(4 * by) * stride + (long long)bx * 16;
#pragma unroll
        for (int y = 0; y < 4; y++, row += stride) {
            if (y >= rows) break;
            if (kVec16 && cols == 4) *reinterpret_cast<uint4*>(row) = make_uint4(px[4 * y], px[4 * y + 1], px[4 * y + 2], px[4 * y + 3]);
            else {
#pragma unroll
                for (int x = 0; x < 4; x++)
                    if (x < cols) reinterpret_cast<u32*>(row)[x] = px[4 * y + x];
            }
        }
    }
}
// The HDR original pane (itw_preview_uncompressed_hdr): DirectX::Convert(R16G16B16A16_FLOAT -> R8G8B8A8_UNORM, TEX_FILTER_DEFAULT)
// of a w x h RGBA16F scratch, which takes the non-WIC _Convert (DirectXTexConvert.cpp:4321-): all four channels through
// display_hdr_unorm8, alpha included.  Grid (ceil(w / 256), h); 8 B read and 4 B written per texel.
__global__ void __launch_bounds__(256) hdr_unorm8_kernel(const uint8_t* __restrict__ src, long long sstride, int w, int h, uint8_t* __restrict__ dst,
                                                         long long dstride)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w || y >= h) return;
    const uint2 t = __ldg(reinterpret_cast<const uint2*>(src + (long long)y * sstride) + x);
    reinterpret_cast<u32*>(dst + (long long)y * dstride)[x] = display_hdr_unorm8(t.x & 0xFFFFu) | (display_hdr_unorm8(t.x >> 16) << 8) |
                                                              (display_hdr_unorm8(t.y & 0xFFFFu) << 16) | (display_hdr_unorm8(t.y >> 16) << 24);
}
// Every texel of a w x h surface := one constant texel (1 word for RGBA8, 2 for RGBA16F).  The preview cross: cells without a face.
__global__ void __launch_bounds__(256) fill_texels_kernel(uint8_t* __restrict__ ptr, int w, int h, long long stride, int words, u32 lo, u32 hi)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w || y >= h) return;
    u32* p = reinterpret_cast<u32*>(ptr + (long long)y * stride) + (long long)x * words;
    p[0] = lo;
    if (words == 2) p[1] = hi;
}
#endif

}  // namespace itw
