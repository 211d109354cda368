// open.cuh -- THE OPEN PATH: what the plug-in's DoReadStart / DoReadContinue (IntelPlugin.cpp:2419-2742) do with a block-compressed
// DDS file, on the GPU.
//
//   alpha scan         ScratchImage::IsAlphaAllOpaque (DirectXTexImage.cpp:744-759): _IsAlphaAllOpaqueBC (DirectXTexCompress.cpp:
//                      472-554) over EVERY image of the file (every mip of every item).  A texel is not opaque when the decoder's
//                      float alpha is < 0.99f; texels of ragged edge blocks outside the image do not count.  Only BC3 / BC7 (and their
//                      _SRGB forms) reach it: BC4 / BC5 / BC6H have no alpha, and the plug-in ignores the answer for BC1 (:2469-2471).
//   layer store        one DoReadContinue: DirectX::Decompress of one image to R8G8B8A8_UNORM[_SRGB] / R32G32B32A32_FLOAT (:2558),
//                      then the copy of channels 0..planes-1 into the top-left corner of a zeroed, interleaved layer of the top-level
//                      size (:2646-2727), with the last plane forced to 255 / 1.0f for a cube map with alpha (:2696, :2724).
//
// The alpha decision is integer-exact.
//   BC7: the decoder's float is byte * (1/255) (BC.h:152-155); 252/255 < 0.99f < 253/255, so "not opaque" is byte <= 252.
//   BC3: D3DXDecodeBC3's alpha palette is a0/255, a1/255, the 7-step interpolants ((8-q)a0 + (q-1)a1) / (7*255), the 5-step ones
//        ((6-q)a0 + (q-1)a1) / (5*255), 0 and 1.  The interpolant closest to 0.99 below it is 1767/1785 (0.98992) and above it
//        1768/1785 (0.99048); for 5 steps 1262/1275 and 1263/1275.  Float rounding (a few ulp, ~1e-7) cannot cross 0.99, and
//        decode_alpha's byte ((N + 3) / 7, (N + 2) / 5) is <= 252 exactly when N <= 1767 (resp. 1262).  So the same byte test holds.
//   tests/test_dds_open.py checks both against the cut _IsAlphaAllOpaqueBC for every (a0, a1, index) of a BC3 alpha block and every
//   alpha byte of BC7 modes 5, 6 and 7.
//
// open_layer_kernel: a warp covers 32 adjacent 4x4 tiles of one tile row of the LAYER.  Tiles inside the image decode their block with
// the display decoders (display.cuh) unchanged; the rest of the layer is zeros, so every byte of the layer is written exactly once and
// no memset pass precedes it.  Each lane packs its tile's row of texels (12, 16, 48 or 64 bytes) into the warp's row in shared memory;
// the warp then stores that row with 16-byte stores (plus a byte tail at the layer's right edge), so three-plane rows leave as whole
// 128-byte lines rather than as 12-byte pieces (store_staged_row, which open_raw.cuh's layer kernel shares).
#pragma once
#include "display.cuh"

namespace itw {

// XMVectorSaturate (max with 0, then min with 1: a NaN becomes 0)
ITW_HD float conv_saturate(float x)
{
    x = x > 0.0f ? x : 0.0f;
    return x < 1.0f ? x : 1.0f;
}
// The target stores: XMStoreUShortN4 (R16G16B16A16_UNORM) and the bias + XMStoreUByteN4 of R8G8B8A8_UNORM, both ASSUMED round to
// nearest with the half added after the product (DESIGN section 2): trunc(saturate(x) * max + 0.5).
ITW_HD u32 conv_unorm16(float x) { return (u32)add_rn(mul_rn(conv_saturate(x), 65535.0f), 0.5f); }
ITW_HD u32 conv_unorm8(float x) { return (u32)add_rn(mul_rn(conv_saturate(x), 255.0f), 0.5f); }

// ---- itw_dds_open_other_bc (include/itw_bcn.h section 15): the block-compressed files section 9 does not open ----
// The loaded format's decoder instantiation of the kernels below, after _DecompressBC's promotion of the typeless formats
// (DirectXTexCompress.cpp:382-392): 70 -> 71 (BC1), 73 / 74 / 75 -> 74 (BC2), 76 / 77 (DXT4) -> 77, 79 -> 80, 81 (BC4_SNORM),
// 82 -> 83, 84 (BC5_SNORM), 94 -> 94 (BC6H_UF16 into 16-bit UNORM planes), 97 -> 98.  -1 for every other format.
ITW_HD constexpr int obc_decoder_of(unsigned f)
{
    return f == 70 ? 71 : (f >= 73 && f <= 75) ? 74 : (f == 76 || f == 77) ? 77 : f == 79 ? 80 : f == 81 ? 81 : f == 82 ? 83
         : f == 84 ? 84 : f == 94 ? 94 : f == 97 ? 98 : -1;
}
// DoReadStart's target (IntelPlugin.cpp:2534-2544): BitsPerColor is 16 for BC6H_TYPELESS, which the BC6H test names not, so
// R16G16B16A16_UNORM; IsSRGB holds for BC2_UNORM_SRGB alone; every other format has at most 8 bits per colour.
ITW_HD constexpr int obc_target_of(unsigned f) { return f == 94 ? 11 : f == 75 ? 29 : 28; }
ITW_HD constexpr int obc_depth_of(unsigned f) { return obc_target_of(f) == 11 ? 16 : 8; }      // BitsPerColor of the target (:2591)
// HasAlpha of the loaded format: the plug-in's BC1 exclusion (:2470-2471) names only 71 / 72, so BC1_TYPELESS counts
ITW_HD constexpr bool obc_has_alpha(unsigned f) { return f == 70 || (f >= 73 && f <= 77) || f == 97; }
ITW_HD constexpr int obc_block_bytes(unsigned f) { return f == 70 || f == 79 || f == 81 ? 8 : 16; }

// The first alpha byte that reads as opaque (see above).
constexpr u32 kOpaqueAlphaMin = 253u;

// BC2's explicit alpha as a byte: D3DXDecodeBC2 (BC.cpp:794-817) gives nibble * (1/15.f), which the byte store rounds to nibble * 17.
// The alpha scan reads the same byte: 14 -> 238, 15 -> 255, so "not opaque" (nibble * (1/15.f) < 0.99f) is byte <= 252 here too.
ITW_HD u32 bc2_alpha_byte(u32 w0, u32 w1, int k)
{
    return conv_unorm8(mul_rn((float)(((k < 8 ? w0 : w1) >> (4 * (k & 7))) & 15u), 1.0f / 15.0f));
}

// One block of an alpha-bearing format (71 BC1 for BC1_TYPELESS, 74 BC2, 77 BC3, 98 BC7; _SRGB forms decode alike): does a texel
// inside the image (the first `cols` columns and `rows` rows of the block) have alpha below 0.99?
template <int kFormat>
ITW_HD bool open_block_not_opaque(const u32 (&w)[4], int cols, int rows)
{
    u32 a[16];
    if (kFormat == 77) {
        decode_alpha(a, w[0], w[1]);
    } else if (kFormat == 74) {
#pragma unroll
        for (int k = 0; k < 16; k++) a[k] = bc2_alpha_byte(w[0], w[1], k);
    } else if (kFormat == 71) {            // three-colour blocks decode index 3 to alpha 0 (punch-through), every other texel to 255
        u32 px[16];
        decode_bc1_colour(px, w[0], w[1], false);
#pragma unroll
        for (int k = 0; k < 16; k++) a[k] = px[k] >> 24;
    } else {
        u32 px[16];
        decode_bc7(px, w);                 // the reserved mode decodes to alpha 0: not opaque, as in DirectXTex
#pragma unroll
        for (int k = 0; k < 16; k++) a[k] = px[k] >> 24;
    }
    bool below = false;
#pragma unroll
    for (int k = 0; k < 16; k++)
        if ((k & 3) < cols && (k >> 2) < rows && a[k] < kOpaqueAlphaMin) below = true;
    return below;
}

// One image of the alpha scan: its blocks are payload blocks [first, first + bw*bh) (images are stored back to back, item-major,
// mip-minor, so block index and byte offset agree for the whole payload).
struct OpenImage {
    long long first;
    int bw, width, height;
};

// BC4_SNORM::DecodeFromIndex (BC4BC5.cpp:106-131) in its own float operations.  The mode compares the RAW signed endpoints; the values
// read -128 as -127, so (-127, -128) runs the eight-value mode with two equal endpoints.
ITW_HD float bc4s_float(int r0, int r1, u32 q)
{
    const float f0 = div_rn((float)(r0 == -128 ? -127 : r0), 127.0f), f1 = div_rn((float)(r1 == -128 ? -127 : r1), 127.0f);
    if (q == 0u) return f0;
    if (q == 1u) return f1;
    if (r0 > r1) {
        q -= 1u;
        return div_rn(add_rn(mul_rn(f0, (float)(7u - q)), mul_rn(f1, (float)q)), 7.0f);
    }
    if (q == 6u) return -1.0f;
    if (q == 7u) return 1.0f;
    q -= 1u;
    return div_rn(add_rn(mul_rn(f0, (float)(5u - q)), mul_rn(f1, (float)q)), 5.0f);
}
// _ConvertScanline's SNORM -> UNORM (DirectXTexConvert.cpp:3331-3342: XMVectorMultiplyAdd(v, 0.5, 0.5), a product and a sum) and the
// R8G8B8A8_UNORM store
ITW_HD u32 snorm_unorm8(float v) { return conv_unorm8(add_rn(mul_rn(v, 0.5f), 0.5f)); }
// one BC4_SNORM channel block -> 16 bytes of the target (the eight palette bytes are computed once)
ITW_HD void bc4s_unorm8(u32 (&val)[16], u32 w0, u32 w1)
{
    const int r0 = (int)(signed char)(w0 & 255u), r1 = (int)(signed char)((w0 >> 8) & 255u);
    const unsigned long long idx = ((unsigned long long)w1 << 16) | (w0 >> 16);
    unsigned long long pal = 0ull;
#pragma unroll
    for (u32 q = 0; q < 8; q++) pal |= (unsigned long long)snorm_unorm8(bc4s_float(r0, r1, q)) << (8 * q);
#pragma unroll
    for (int k = 0; k < 16; k++) val[k] = (u32)(pal >> (8 * ((u32)(idx >> (3 * k)) & 7u))) & 255u;
}

// One block -> 16 RGBA8 texels of R8G8B8A8_UNORM[_SRGB]: what Decompress stores for the 8-bit decoders of the open paths.
//   74 BC2        D3DXDecodeBC2: the colour half in four-colour mode (DecodeBC1(..., false), as BC3's), the explicit alpha
//   81 BC4_SNORM  (r, 0, 0, 1) -> SNORM -> UNORM on all four channels -> the R -> RGB copy (:3445-3457): (r', r', r', 255)
//   84 BC5_SNORM  (r, g, 0, 1) -> SNORM -> UNORM: blue 0 becomes 0.5 (byte 128), alpha 1 stays 1
//   the rest      display.cuh's plain decode
template <int kFormat>
ITW_HD void open_block_rgba8(u32 (&px)[16], const u32 (&w)[4])
{
    if constexpr (kFormat == 74) {
        decode_bc1_colour(px, w[2], w[3], true);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = (px[k] & 0x00FFFFFFu) | (bc2_alpha_byte(w[0], w[1], k) << 24);
    } else if constexpr (kFormat == 81) {
        u32 r[16];
        bc4s_unorm8(r, w[0], w[1]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = r[k] * 0x010101u | (snorm_unorm8(1.0f) << 24);
    } else if constexpr (kFormat == 84) {
        u32 r[16], g[16];
        bc4s_unorm8(r, w[0], w[1]);
        bc4s_unorm8(g, w[2], w[3]);
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = r[k] | (g[k] << 8) | (snorm_unorm8(0.0f) << 16) | (snorm_unorm8(1.0f) << 24);
    } else {
        display_block_rgba8<kFormat, kDisplayPlain>(px, w);
    }
}
// BC6H_TYPELESS (decoder 94) -> R16G16B16A16_UNORM: D3DXDecodeBC6HU's floats (display_block_f32<95>), FLOAT -> UNORM saturate and the
// XMStoreUShortN4 store, per channel; px[k][c] is the 16-bit value.
ITW_HD void open_block_unorm16(u32 (&px)[16][4], const u32 (&w)[4])
{
    display_block_f32<95>(px, w);
#pragma unroll
    for (int k = 0; k < 16; k++)
#pragma unroll
        for (int c = 0; c < 4; c++) px[k][c] = conv_unorm16(bits_float(px[k][c]));
}

#if defined(__CUDACC__)
// The row-staged store shared by the open path's layer kernels.  A warp writes one stretch of a layer row: lane k supplies the k-th
// kTileRow-byte piece of it (four texels), the pieces meet in shared memory, and the warp stores the first `span` bytes with 16-byte
// stores plus a byte tail at the layer's right edge, so rows of 3-plane texels leave as whole 128-byte lines.  Pieces of 16, 32, 48
// and 64 bytes go in as 16-byte stores (lanes 16 and 48 bytes apart meet 8 distinct bank quads per quarter warp); for 64 bytes one
// spare 16-byte slot after every 128 bytes spreads the lanes of a quarter warp over all eight quads as well.  12- and 24-byte pieces
// go in as words.  `srow` holds staged_row_slots(kTileRow) slots; dst and the row are 16-byte aligned.
__host__ __device__ constexpr int staged_row_slots(int tile_row)
{
    return 2 * tile_row + (tile_row == 64 ? tile_row / 4 : 0);     // 32 pieces of 16-byte slots, plus the spare slots of 64-byte pieces
}
template <int kTileRow>
__device__ __forceinline__ void store_staged_row(uint4* srow, int lane, bool has_piece, const u32 (&t)[kTileRow / 4], int span,
                                                 uint8_t* grow)
{
    constexpr int kWords = kTileRow / 4;
    constexpr int kVecs = kWords % 4 == 0 ? kWords / 4 : 0;
    constexpr int kPad = kVecs == 4 ? 1 : 0;
    auto slot = [](int k) { return k + kPad * (k >> 3); };      // smem slot of the row's k-th 16-byte piece
    if (has_piece) {
        if constexpr (kVecs > 0) {
#pragma unroll
            for (int j = 0; j < kVecs; j++) srow[slot(kVecs * lane + j)] = make_uint4(t[4 * j], t[4 * j + 1], t[4 * j + 2], t[4 * j + 3]);
        } else {
            u32* words = reinterpret_cast<u32*>(srow) + lane * kWords;
#pragma unroll
            for (int i = 0; i < kWords; i++) words[i] = t[i];
        }
    }
    __syncwarp();
    const int body = span & ~15;
    for (int i = lane; i < body >> 4; i += 32) reinterpret_cast<uint4*>(grow)[i] = srow[slot(i)];
    if (lane < span - body)
        grow[body + lane] = reinterpret_cast<const uint8_t*>(srow + slot(body >> 4))[lane];
    __syncwarp();
}

// One thread per block of every image; `images` sorted by `first`.  *flag becomes 1 if any texel of any image is not opaque.
template <int kFormat>
__global__ void __launch_bounds__(256) open_alpha_kernel(const uint8_t* __restrict__ payload, long long nblocks,
                                                         const OpenImage* __restrict__ images, int nimages, int* __restrict__ flag)
{
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool below = false;
    if (id < nblocks) {
        int lo = 0, hi = nimages - 1;                           // the last image with first <= id
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (images[mid].first <= id) lo = mid;
            else hi = mid - 1;
        }
        const OpenImage im = images[lo];
        const int local = (int)(id - im.first), by = local / im.bw, bx = local - by * im.bw;
        u32 w[4];
        if (kFormat == 77 || kFormat == 74) {                   // the alpha half of a BC3 / BC2 block is its first 8 bytes
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(payload) + 2 * id);
            w[0] = v.x; w[1] = v.y; w[2] = w[3] = 0u;
        } else if (kFormat == 71) {                             // 8-byte BC1 blocks
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(payload) + id);
            w[0] = v.x; w[1] = v.y; w[2] = w[3] = 0u;
        } else {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(payload) + id);
            w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
        }
        below = open_block_not_opaque<kFormat>(w, min(4, im.width - 4 * bx), min(4, im.height - 4 * by));
    }
    if (__any_sync(0xFFFFFFFFu, below) && (threadIdx.x & 31) == 0) *flag = 1;
}

// One layer: `dst` holds `height` rows of `width` texels of kPlanes channels (bytes for the LDR decoders 71/74/77/80/81/83/84/98,
// floats for BC6H 95/96, ushorts for BC6H_TYPELESS 94), rows `row_bytes` apart; dst and row_bytes are 16-byte aligned.  The image
// (iw x ih texels, blocks in raster order in `blocks`) lands in the top-left corner.  force_alpha: the last plane of every image texel
// is 255 / 1.0f (0x3C00 at 16 bits, open_raw.cuh's rule; no 16-bit format here has alpha).
template <int kFormat, int kPlanes>
__global__ void __launch_bounds__(256, 2) open_layer_kernel(const uint8_t* __restrict__ blocks, int iw, int ih, uint8_t* __restrict__ dst,
                                                         int width, int height, long long row_bytes, bool force_alpha)
{
    constexpr bool kHdr = kFormat == 95 || kFormat == 96, k16 = kFormat == 94;
    constexpr int kTexel = kPlanes * (kHdr ? 4 : k16 ? 2 : 1);  // bytes per layer texel
    constexpr int kTileRow = 4 * kTexel;                        // bytes of one tile's row: 12, 16, 24, 32, 48 or 64
    constexpr int kWords = kTileRow / 4;
    __shared__ uint4 stage[8][staged_row_slots(kTileRow)];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tw = (width + 3) >> 2, chunks = (tw + 31) >> 5;
    const long long g = (long long)blockIdx.x * 8 + warp;       // warp-uniform: (tile row, chunk of 32 tiles)
    if (g >= (long long)((height + 3) >> 2) * chunks) return;
    const int ty = (int)(g / chunks), chunk = (int)(g - (long long)ty * chunks), tx = 32 * chunk + lane;
    const int ibw = (iw + 3) >> 2;
    const bool in_image = tx < ibw && ty < ((ih + 3) >> 2);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (in_image) {
        const long long id = (long long)ty * ibw + tx;
        if (kFormat == 71 || kFormat == 80 || kFormat == 81) {
            const uint2 h = __ldg(reinterpret_cast<const uint2*>(blocks) + id);
            v.x = h.x; v.y = h.y;
        } else {
            v = __ldg(reinterpret_cast<const uint4*>(blocks) + id);
        }
    }
    const u32 w[4] = {v.x, v.y, v.z, v.w};
    // the tile's texels: four float bit patterns (BC6H) or ushorts (BC6H_TYPELESS) per texel, or one RGBA8 word; warps wholly outside
    // the image skip the decode
    u32 pf[16][4], p8[16];
    if (__any_sync(0xFFFFFFFFu, in_image)) {
        if constexpr (kHdr) display_block_f32<kFormat>(pf, w);
        else if constexpr (k16) open_block_unorm16(pf, w);
        else open_block_rgba8<kFormat>(p8, w);
    }
    const int cols = in_image ? min(4, iw - 4 * tx) : 0;        // texels of this tile that belong to the image
    const int span = min(128, width - 128 * chunk) * kTexel;    // bytes of the warp's part of a layer row
    uint8_t* out = dst + (long long)chunk * 128 * kTexel;
    uint4* srow = stage[warp];
#pragma unroll
    for (int y = 0; y < 4; y++) {
        const int Y = 4 * ty + y;
        if (Y >= height) break;
        const bool row_in = in_image && Y < ih;
        u32 t[kWords];
        if constexpr (kHdr) {
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int c = 0; c < kPlanes; c++) {
                    u32 v = (row_in && x < cols) ? pf[4 * y + x][c] : 0u;
                    if (c == kPlanes - 1 && force_alpha && row_in && x < cols) v = 0x3F800000u;
                    t[kPlanes * x + c] = v;
                }
        } else if constexpr (k16) {                             // ushort j of the piece is plane j % kPlanes of texel j / kPlanes
#pragma unroll
            for (int i = 0; i < kWords; i++) t[i] = 0u;
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int c = 0; c < kPlanes; c++) {
                    u32 v = (row_in && x < cols) ? pf[4 * y + x][c] : 0u;
                    if (c == kPlanes - 1 && force_alpha && row_in && x < cols) v = 0x3C00u;
                    const int j = kPlanes * x + c;
                    t[j >> 1] |= v << (16 * (j & 1));
                }
        } else {
            u32 q[4];
#pragma unroll
            for (int x = 0; x < 4; x++) {
                q[x] = (row_in && x < cols) ? p8[4 * y + x] : 0u;
                if (force_alpha && row_in && x < cols) q[x] |= 255u << (8 * (kPlanes - 1));
            }
            if constexpr (kPlanes == 4) {
#pragma unroll
                for (int x = 0; x < 4; x++) t[x] = q[x];
            } else {                                            // r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
                t[0] = (q[0] & 0x00FFFFFFu) | (q[1] << 24);
                t[1] = ((q[1] >> 8) & 0xFFFFu) | (q[2] << 16);
                t[2] = ((q[2] >> 16) & 0xFFu) | (q[3] << 8);
            }
        }
        store_staged_row<kTileRow>(srow, lane, tx < tw, t, span, out + (long long)Y * row_bytes);
    }
}
#endif

}  // namespace itw
