// view_emu.cpp -- TEST-ONLY CPU execution of the dialog view (csrc/view.cuh): the same __host__ __device__ routines view_channels and
// view_texel that itw_preview_view's host code and view_kernel run, with the zoom divided by 1 << mip_level as the host does.  Built
// by __graft_entry__.build() into tests/emu/libitw_view_emu.so and loaded only by tests.
#include "../../intel-texture-works-plugin_b200/csrc/view.cuh"

using namespace itw;

// `src` = src_w x src_h texels of `planes` interleaved elements of `depth` bits, rows `row_bytes` apart.  `dst` receives
// width * height packed RGB8 texels.
extern "C" void emu_view(const void* src, int src_w, int src_h, int planes, int depth, long long row_bytes, int width, int height, int x,
                         int y, double zoom, int mip_level, unsigned channels, unsigned matte, uint8_t* dst)
{
    ViewParams V{static_cast<const uint8_t*>(src), row_bytes, src_w, src_h, planes, depth, width, height, x, y,
                 zoom / (double)(1 << mip_level), {-1, -1, -1}, matte};
    view_channels(V.index, channels, planes);
    for (int yt = 0; yt < height; yt++)
        for (int xt = 0; xt < width; xt++) {
            const u32 rgb = view_texel(V, xt, yt);
            uint8_t* p = dst + ((size_t)yt * width + xt) * 3;
            p[0] = (uint8_t)rgb;
            p[1] = (uint8_t)(rgb >> 8);
            p[2] = (uint8_t)(rgb >> 16);
        }
}
