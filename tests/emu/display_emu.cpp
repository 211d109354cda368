// display_emu.cpp -- TEST-ONLY CPU execution of the display decompressor's per-block logic (csrc/display.cuh): the same
// __host__ __device__ functions display_kernel runs, driven block by block, with the kernel's ragged-edge rule.  Built by
// __graft_entry__.build() into tests/emu/libitw_display_emu.so and loaded only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/display.cuh"

using namespace itw;

template <int kFormat, int kRule>
static void run(const uint8_t* blocks, int w, int h, uint8_t* dst)
{
    const int bw = (w + 3) / 4, bh = (h + 3) / 4, bpb = (kFormat == 71 || kFormat == 80) ? 8 : 16;
    const int texel = (kRule == kDisplayHdrFloat) ? 16 : 4;
    for (int by = 0; by < bh; by++)
        for (int bx = 0; bx < bw; bx++) {
            u32 wd[4] = {0u, 0u, 0u, 0u};
            memcpy(wd, blocks + ((size_t)by * bw + bx) * bpb, bpb);
            u32 px8[16], pxf[16][4];
            if (kRule == kDisplayHdrFloat) display_block_f32<kFormat>(pxf, wd);
            else display_block_rgba8<kFormat, kRule>(px8, wd);
            for (int y = 0; y < 4 && 4 * by + y < h; y++)
                for (int x = 0; x < 4 && 4 * bx + x < w; x++) {
                    uint8_t* t = dst + ((size_t)(4 * by + y) * w + 4 * bx + x) * texel;
                    if (kRule == kDisplayHdrFloat) memcpy(t, pxf[4 * y + x], 16);
                    else memcpy(t, &px8[4 * y + x], 4);
                }
        }
}

// decoder: 71/77/80/83/95/96/98; rule: DisplayRule.  dst: tight rows of w texels.  Returns -1 for a pair the product rejects.
extern "C" int emu_display(int decoder, int rule, const uint8_t* blocks, int w, int h, uint8_t* dst)
{
#define CASE(F, R) \
    case F * 8 + R: run<F, R>(blocks, w, h, dst); return 0;
    switch (decoder * 8 + rule) {
        CASE(71, 0) CASE(71, 1) CASE(71, 2) CASE(77, 0) CASE(77, 1) CASE(77, 2) CASE(80, 0) CASE(80, 2) CASE(83, 0) CASE(83, 2)
        CASE(98, 0) CASE(98, 1) CASE(98, 2) CASE(95, 3) CASE(95, 4) CASE(96, 3) CASE(96, 4)
        default: return -1;
    }
#undef CASE
}
// the two float -> byte sRGB stores of the BC1 / BC3 colour path
extern "C" int emu_srgb_in_store(float f) { return (int)SrgbInStore::of(f); }
extern "C" int emu_srgb_out_store(float f) { return (int)SrgbOutStore::of(f); }
