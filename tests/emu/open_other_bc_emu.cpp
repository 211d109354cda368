// open_other_bc_emu.cpp -- TEST-ONLY CPU execution of the per-block routines of itw_dds_open_other_bc (csrc/open.cuh): the same
// __host__ __device__ open_block_rgba8, open_block_unorm16 and open_block_not_opaque that open_layer_kernel and open_alpha_kernel run
// for these formats, and the scope decisions the host code takes from obc_decoder_of / obc_target_of / obc_has_alpha.  Built by
// __graft_entry__.build() into tests/emu/libitw_open_other_bc_emu.so and loaded only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/open.cuh"

using namespace itw;

namespace {
template <int kDecoder>
void blocks_rgba8(const uint8_t* blocks, long long n, uint8_t* out)
{
    constexpr int kBpb = kDecoder == 71 || kDecoder == 80 || kDecoder == 81 ? 8 : 16;
    for (long long i = 0; i < n; i++) {
        u32 w[4] = {0u, 0u, 0u, 0u}, px[16];
        memcpy(w, blocks + i * kBpb, kBpb);
        open_block_rgba8<kDecoder>(px, w);
        memcpy(out + 64 * i, px, 64);      // little-endian: R, G, B, A bytes per texel
    }
}
}  // namespace

// `n` blocks of the loaded format's decoder (obc_decoder_of) -> 16 texels each, in block order: 4 bytes per texel (RGBA8), or 4
// ushorts per texel for decoder 94
extern "C" int emu_obc_blocks(int decoder, const uint8_t* blocks, long long n, uint8_t* out)
{
    switch (decoder) {
        case 71: blocks_rgba8<71>(blocks, n, out); return 0;
        case 74: blocks_rgba8<74>(blocks, n, out); return 0;
        case 77: blocks_rgba8<77>(blocks, n, out); return 0;
        case 80: blocks_rgba8<80>(blocks, n, out); return 0;
        case 81: blocks_rgba8<81>(blocks, n, out); return 0;
        case 83: blocks_rgba8<83>(blocks, n, out); return 0;
        case 84: blocks_rgba8<84>(blocks, n, out); return 0;
        case 98: blocks_rgba8<98>(blocks, n, out); return 0;
        case 94:
            for (long long i = 0; i < n; i++) {
                u32 w[4], px[16][4];
                memcpy(w, blocks + 16 * i, 16);
                open_block_unorm16(px, w);
                for (int k = 0; k < 16; k++)
                    for (int c = 0; c < 4; c++) {
                        const uint16_t v = (uint16_t)px[k][c];
                        memcpy(out + 128 * i + 8 * k + 2 * c, &v, 2);
                    }
            }
            return 0;
        default: return -1;
    }
}
// scan decoder 71 / 74 / 77 / 98: out[i] = 1 if every texel of the first `cols` x `rows` of block i is opaque
extern "C" int emu_obc_blocks_opaque(int decoder, const uint8_t* blocks, long long n, int cols, int rows, uint8_t* out)
{
    const int bpb = decoder == 71 ? 8 : 16;
    for (long long i = 0; i < n; i++) {
        u32 w[4] = {0u, 0u, 0u, 0u};
        memcpy(w, blocks + bpb * i, bpb);
        bool below;
        switch (decoder) {
            case 71: below = open_block_not_opaque<71>(w, cols, rows); break;
            case 74: below = open_block_not_opaque<74>(w, cols, rows); break;
            case 77: below = open_block_not_opaque<77>(w, cols, rows); break;
            case 98: below = open_block_not_opaque<98>(w, cols, rows); break;
            default: return -1;
        }
        out[i] = below ? 0 : 1;
    }
    return 0;
}
// The product's scope decisions for a loaded DXGI format: out = {decoder (-1 if not served), target, depth, HasAlpha, block bytes}
extern "C" void emu_obc_scope(unsigned dxgi, int* out)
{
    out[0] = obc_decoder_of(dxgi);
    out[1] = obc_target_of(dxgi);
    out[2] = obc_depth_of(dxgi);
    out[3] = obc_has_alpha(dxgi);
    out[4] = obc_block_bytes(dxgi);
}
