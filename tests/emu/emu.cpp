// emu.cpp -- TEST-ONLY lane-by-lane CPU execution of the product's kernel logic.
//
// The CUDA kernels in intel-texture-works-plugin_b200/csrc/*.cuh are written as per-lane phase
// functions (__host__ __device__).  This file compiles the very same headers with g++ and drives
// every phase for lanes 0..31 in turn, with a warp barrier between phases, so the kernels' logic
// (everything except the GPU's own float instructions) can be checked against the oracle on a
// machine without a GPU.  It is built by tests/emu/build_emu.py into tests/emu/libitw_emu.so and
// is loaded only by tests.  The product library never contains or calls this code.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/bc4_bc5.cuh"
#include "../../intel-texture-works-plugin_b200/csrc/itw_params.h"
#include "../../intel-texture-works-plugin_b200/csrc/mips.cuh"
#include "../../intel-texture-works-plugin_b200/csrc/decode.cuh"
#include "../../intel-texture-works-plugin_b200/csrc/frontend.cuh"
#include "../../intel-texture-works-plugin_b200/csrc/mips_f16.cuh"

using namespace itw;

static SurfaceView view_of(const rgba_surface* s) { return SurfaceView{s->ptr, s->width, s->height, s->stride}; }

template <class F>
static void per_block(const rgba_surface* src, uint8_t* dst, int bpb, F f)
{
    SurfaceView s = view_of(src);
    const int bw = s.width / 4, bh = s.height / 4;
    for (int by = 0; by < bh; by++)
        for (int bx = 0; bx < bw; bx++) {
            u32 tex[16], out[4];
            fetch_rows_rgba8<false>(tex, s, bx, by);
            f(tex, out);
            memcpy(dst + ((size_t)by * bw + bx) * bpb, out, bpb);
        }
}

// block decoders (csrc/decode.cuh), block by block through the kernel's own per-block routines
template <int kFormat>
static void emu_decode_as(const uint8_t* blocks, uint8_t* dst, int w, int h, int stride, int bpb)
{
    const int bw = w / 4, bh = h / 4;
    for (int by = 0; by < bh; by++)
        for (int bx = 0; bx < bw; bx++) {
            u32 wd[4] = {0, 0, 0, 0};
            memcpy(wd, blocks + ((size_t)by * bw + bx) * bpb, bpb);
            if (kFormat == 95 || kFormat == 96) {
                u32 px[16][2];
                decode_bc6h<kFormat == 96>(px, wd);
                for (int k = 0; k < 16; k++) memcpy(dst + (size_t)(4 * by + k / 4) * stride + (size_t)(4 * bx + k % 4) * 8, px[k], 8);
            } else {
                u32 px[16];
                decode_block_rgba8<kFormat>(px, wd);
                for (int k = 0; k < 16; k++) memcpy(dst + (size_t)(4 * by + k / 4) * stride + (size_t)(4 * bx + k % 4) * 4, &px[k], 4);
            }
        }
}

extern "C" {
void emu_CompressBlocksBC1(const rgba_surface* src, uint8_t* dst)
{ per_block(src, dst, 8, [](const u32 (&t)[16], u32 (&o)[4]) { bc1_bc3_encode_block<false>(t, o); }); }
void emu_CompressBlocksBC3(const rgba_surface* src, uint8_t* dst)
{ per_block(src, dst, 16, [](const u32 (&t)[16], u32 (&o)[4]) { bc1_bc3_encode_block<true>(t, o); }); }
void emu_CompressBlocksBC4(const rgba_surface* src, uint8_t* dst)
{ per_block(src, dst, 8, [](const u32 (&t)[16], u32 (&o)[4]) { bc4_bc5_encode_block<false>(t, o); }); }
void emu_CompressBlocksBC5(const rgba_surface* src, uint8_t* dst)
{ per_block(src, dst, 16, [](const u32 (&t)[16], u32 (&o)[4]) { bc4_bc5_encode_block<true>(t, o); }); }

// Lanes of a phase run one after the other.  On the GPU they run concurrently, so a phase must not depend on the order: the
// order is selectable (ascending, descending, a fixed shuffle) and tests/test_emu_parity.py requires identical output for all.
static int g_lane_order = 0;
void emu_set_lane_order(int mode) { g_lane_order = mode; }
static inline int emu_lane(int i) { return g_lane_order == 0 ? i : (g_lane_order == 1 ? 31 - i : (int)((i * 13u + 7u) & 31u)); }
#define ITW_PHASE_EMU(call) for (int lane_i = 0; lane_i < 32; lane_i++) { const int lane = emu_lane(lane_i); call; }

// Blocks per warp and round: bc7_kernel runs 16 in a full round and 1, 2, 4, 8 or 16 in the last one; the emulation runs
// a whole surface in rounds of one such size.  Returns -1 (and keeps the setting) for any other count.
static int g_bc7_per_warp = kBc7Super;
int emu_set_bc7_per_warp(int n)
{
    if (n != 1 && n != 2 && n != 4 && n != 8 && n != 16) return -1;
    g_bc7_per_warp = n;
    return 0;
}
void emu_CompressBlocksBC7(const rgba_surface* src, uint8_t* dst, bc7_enc_settings* settings)
{
    SurfaceView surf = view_of(src);
    const Bc7Params P = bc7_params_from(*settings);
    const long long nblocks = (long long)(surf.width / 4) * (surf.height / 4);
    const int per_warp = g_bc7_per_warp;
    static thread_local Bc7Warp W;
    for (long long first_block = 0; first_block < nblocks; first_block += per_warp) {
        const int nvalid = (int)((nblocks - first_block < per_warp) ? (nblocks - first_block) : per_warp);
        const long long out_block = first_block;
        ITW_BC7_PROGRAM(ITW_PHASE_EMU)
    }
}
void emu_CompressBlocksBC6H(const rgba_surface* src, uint8_t* dst, bc6h_enc_settings* settings)
{
    SurfaceView surf = view_of(src);
    const Bc6Params P = bc6_params_from(*settings);
    const long long nblocks = (long long)(surf.width / 4) * (surf.height / 4);
    static thread_local Bc6Warp W;
    W.layout = &h_bc6_layout[0][0];
    for (long long first_block = 0; first_block < nblocks; first_block += kBc6Slots) {
        const int nvalid = (int)((nblocks - first_block < kBc6Slots) ? (nblocks - first_block) : kBc6Slots);
        ITW_BC6_PROGRAM(ITW_PHASE_EMU)
    }
}

// one padded mip level, texel by texel, through the kernel's own per-texel routine (csrc/mips.cuh)
void emu_mip_level(const uint8_t* src, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh, int pw, int ph)
{
    for (int y = 0; y < ph; y++)
        for (int x = 0; x < pw; x++) reinterpret_cast<u32*>(dst + (size_t)y * pw * 4)[x] = mip_texel(src, sw, sh, sstride, dw, dh, x, y);
}
int emu_itw_decode(int format, const uint8_t* blocks, const rgba_surface* dst)
{
    switch (format) {
        case 71: emu_decode_as<71>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 8); return 0;
        case 77: emu_decode_as<77>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 16); return 0;
        case 80: emu_decode_as<80>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 8); return 0;
        case 83: emu_decode_as<83>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 16); return 0;
        case 95: emu_decode_as<95>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 16); return 0;
        case 96: emu_decode_as<96>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 16); return 0;
        case 98: emu_decode_as<98>(blocks, dst->ptr, dst->width, dst->height, dst->stride, 16); return 0;
        default: return -1;
    }
}
// pixel-format front end (csrc/frontend.cuh), texel by texel through the kernel's own per-texel routine
int emu_itw_convert_pixels(int format, const itw_pixel_source* src, uint32_t flags, const rgba_surface* dst)
{
    const int family = (format == 95) ? 2 : ((format == 80 || format == 83) ? 1 : 0);
    const long long row_bytes = src->row_bytes ? src->row_bytes : (long long)src->width * src->planes * (src->depth / 8);
    const FrontParams P{static_cast<const uint8_t*>(src->data), src->width, src->height, src->planes, src->depth, row_bytes, family, flags};
    const int texel = (family == 2) ? 8 : 4;
    for (int y = 0; y < dst->height; y++)
        for (int x = 0; x < dst->width; x++) {
            u32 out[2];
            front_texel(out, P, x, y);
            memcpy(dst->ptr + (size_t)y * dst->stride + (size_t)x * texel, out, texel);
        }
    return 0;
}
// one padded RGBA16F mip level, texel by texel, through the kernel's own per-texel routine (csrc/mips_f16.cuh)
void emu_mip_level_f16(const uint8_t* src, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh, int pw, int ph, int box, const uint8_t* stale_row)
{
    for (int y = 0; y < ph; y++)
        for (int x = 0; x < pw; x++) {
            u32 out[2];
            mip_f16_texel(out, src, sw, sh, sstride, dw, dh, x, y, box != 0, stale_row);
            memcpy(dst + ((size_t)y * pw + x) * 8, out, 8);
        }
}
// one padded RGBA8 mip level through the float filter of csrc/mips_f16.cuh: codec 1 = UNORM, 2 = UNORM_SRGB
void emu_mip_level_rgba8(int codec, const uint8_t* src, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh, int pw, int ph, int box, const uint8_t* stale_row)
{
    for (int y = 0; y < ph; y++)
        for (int x = 0; x < pw; x++) {
            u32 out[2];
            if (codec == 2) mip_float_texel<2>(out, src, sw, sh, sstride, dw, dh, x, y, box != 0, stale_row);
            else mip_float_texel<1>(out, src, sw, sh, sstride, dw, dh, x, y, box != 0, stale_row);
            memcpy(dst + ((size_t)y * pw + x) * 4, out, 4);
        }
}
// the product's profile tables (csrc/itw_params.h), exported so the emulation is self-contained
#define EMU_BC7(name, row) void emu_GetProfile_##name(bc7_enc_settings* s) { bc7_fill_profile(s, row); }
EMU_BC7(ultrafast, 0) EMU_BC7(veryfast, 1) EMU_BC7(fast, 2) EMU_BC7(basic, 3) EMU_BC7(slow, 4)
EMU_BC7(alpha_ultrafast, 5) EMU_BC7(alpha_veryfast, 6) EMU_BC7(alpha_fast, 7) EMU_BC7(alpha_basic, 8) EMU_BC7(alpha_slow, 9)
#define EMU_BC6(name, row) void emu_GetProfile_bc6h_##name(bc6h_enc_settings* s) { bc6_fill_profile(s, row); }
EMU_BC6(veryfast, 0) EMU_BC6(fast, 1) EMU_BC6(basic, 2) EMU_BC6(slow, 3) EMU_BC6(veryslow, 4)
}
