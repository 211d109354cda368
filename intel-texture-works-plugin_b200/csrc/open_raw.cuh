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
    kRawRgba32f = 4     // R32G32B32A32_FLOAT, copied
};
ITW_HD constexpr int raw_src_bytes(int src) { return src == kRawBgr8 ? 3 : src == kRawRgba16 ? 8 : src == kRawRgba32f ? 16 : 4; }
ITW_HD constexpr int raw_plane_bytes(int src) { return src == kRawRgba16 ? 2 : src == kRawRgba32f ? 4 : 1; }

// The alpha decision of one loaded texel from the word that holds its alpha (the texel's last 32 bits): true when alpha < 0.99f.
template <int kSrc>
ITW_HD bool raw_alpha_below(u32 word)
{
    if constexpr (kSrc == kRawRgba16) return (word >> 16) <= 64879u;
    else if constexpr (kSrc == kRawRgba32f) {
        float a;
        memcpy(&a, &word, 4);
        return a < 0.99f;
    } else {
        return (word >> 24) <= 252u;
    }
}

// The loaded texel at `p` (4-byte aligned unless kRawBgr8) as four plane values: bytes, ushorts or float bit patterns.
template <int kSrc>
ITW_HD void raw_load_texel(const uint8_t* p, u32 (&v)[4])
{
    if constexpr (kSrc == kRawBgr8) {
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
    constexpr u32 kForced = kSrc == kRawRgba16 ? 0x3C00u : kSrc == kRawRgba32f ? 0x3F800000u : 255u;
#pragma unroll
    for (int c = 0; c < 4; c++) o[c] = c < kPlanes ? v[c] : 0u;
    if (force_alpha) o[kPlanes - 1] = kForced;
}

#if defined(__CUDACC__)
// The scan of `bytes` payload bytes of kSrc texels (kRawRgba8, kRawRgba16 or kRawRgba32f) at a 4-byte aligned `payload`: *flag becomes
// 1 if any texel is not opaque.  The bytes up to the first 16-byte boundary and after the last one are read as words by the first
// threads; the body goes in 16-byte loads, grid-stride, four loads in flight per thread.  Word j of the payload holds an alpha when
// j % (texel words) is the texel's last word.
template <int kSrc>
__global__ void __launch_bounds__(256) open_raw_alpha_kernel(const uint8_t* __restrict__ payload, long long bytes, int* __restrict__ flag)
{
    constexpr int kTexelWords = raw_src_bytes(kSrc) / 4;
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
        if (j % kTexelWords == kTexelWords - 1) below = raw_alpha_below<kSrc>(__ldg(words + j));
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
                if ((lanes >> k) & 1u) below |= raw_alpha_below<kSrc>(w[k]);
        }
    }
    if (__any_sync(0xFFFFFFFFu, below) && (threadIdx.x & 31) == 0) *flag = 1;
}

// One layer: `dst` holds `height` rows of `width` texels of kPlanes planes of raw_plane_bytes(kSrc) bytes, rows `row_bytes` apart;
// dst and row_bytes are 16-byte aligned.  The image (iw x ih texels of raw_src_bytes(kSrc) bytes, tight rows at `src`, 4-byte aligned
// unless kRawBgr8) lands in the top-left corner, zeros elsewhere.  A warp covers 128 texels of one layer row: each lane builds four
// texels and store_staged_row writes the row with 16-byte stores.  force_alpha: the last plane of every image texel is forced.
template <int kSrc, int kPlanes>
__global__ void __launch_bounds__(256) open_raw_layer_kernel(const uint8_t* __restrict__ src, int iw, int ih, uint8_t* __restrict__ dst,
                                                             int width, int height, long long row_bytes, bool force_alpha)
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
        raw_load_texel<kSrc>(srow + x * kSrcBytes, v);
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
#endif

}  // namespace itw
