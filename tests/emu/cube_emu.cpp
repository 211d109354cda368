// cube_emu.cpp -- TEST-ONLY CPU execution of the cross-to-faces pass (csrc/frontend.cuh): the same __host__ __device__ routine
// cube_texel that cube_faces_kernel runs per texel, with the cell origins the host computes from kCubeCells.  Built by
// __graft_entry__.build() into tests/emu/libitw_cube_emu.so and loaded only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/frontend.cuh"

using namespace itw;

// `doc` = doc_w x doc_h texels of `planes` interleaved elements of `depth` bits, tightly packed.  `family` as FrontParams (0 colour,
// 2 BC6H).  `out` receives the six faces back to back, each w x h tight RGBA8 / RGBA16F texels, where w x h is the face size of the
// cross (horizontal when doc_w >= doc_h).  Returns 0, or -1 when the document is smaller than one texel per face.
extern "C" int emu_cube_faces(int family, const void* doc, int doc_w, int doc_h, int planes, int depth, unsigned flags, int linear, uint8_t* out)
{
    const int vertical = doc_w < doc_h ? 1 : 0;
    CubeCross C{};
    C.w = vertical ? doc_w / 3 : doc_w / 4;
    C.h = vertical ? doc_h / 4 : doc_h / 3;
    if (C.w < 1 || C.h < 1) return -1;
    C.P = FrontParams{static_cast<const uint8_t*>(doc), doc_w, doc_h, planes, depth, (long long)doc_w * planes * (depth / 8), family, flags};
    C.linear = linear;
    for (int f = 0; f < 6; f++) {
        C.origin[f][0] = kCubeCells[vertical][f][0] * C.w;
        C.origin[f][1] = kCubeCells[vertical][f][1] * C.h;
    }
    const int texel = family == 2 ? 8 : 4;
    for (int f = 0; f < 6; f++)
        for (int y = 0; y < C.h; y++)
            for (int x = 0; x < C.w; x++) {
                u32 px[2];
                cube_texel(px, C, f, x, y);
                memcpy(out + (((size_t)f * C.h + y) * C.w + x) * texel, px, texel);
            }
    return 0;
}
