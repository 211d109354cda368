// layers_emu.cpp -- TEST-ONLY CPU execution of the layer-to-level copy (csrc/frontend.cuh): the same __host__ __device__ routine
// layer_texel that layer_kernel runs per texel.  Built by __graft_entry__.build() into tests/emu/libitw_layers_emu.so and loaded
// only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/frontend.cuh"

using namespace itw;

// One level: `level` = pw x ph tightly packed RGBA8 / RGBA16F texels, modified in place as the kernel does (texels beyond lw x lh
// replicate the edge).  `planes` = channels 0..channel_count-1 and [3] = alpha or null, each TIGHT lw x lh planes of `depth` bits
// (the rectangle the host stages).  `flip` = ITW_FRONT_FLIP_* bits (level 0).
extern "C" int emu_layer_level(int hdr, uint8_t* level, int lw, int lh, int pw, int ph, int depth, const void* const* planes,
                               int channel_count, unsigned flip)
{
    if (channel_count < 1 || channel_count > 3 || pw < lw || ph < lh) return -1;
    LayerLevel L{};
    for (int c = 0; c < 4; c++) L.plane[c] = static_cast<const uint8_t*>(planes[c]);
    L.lw = lw; L.lh = lh; L.pw = pw; L.ph = ph; L.channels = channel_count;
    const int texel = hdr ? 8 : 4;
    for (int y = 0; y < ph; y++)
        for (int x = 0; x < pw; x++) {
            uint8_t* p = level + ((size_t)y * pw + x) * texel;
            u32 px[2] = {0u, 0u};
            memcpy(px, p, texel);
            layer_texel(px, L, depth, hdr != 0, flip, x, y);
            memcpy(p, px, texel);
        }
    return 0;
}
