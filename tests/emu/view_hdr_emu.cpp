// view_hdr_emu.cpp -- TEST-ONLY CPU execution of the preview dialog's HDR routines: the exposed view (view_channels, view_exposure
// and view_texel<true> of csrc/view.cuh, as itw_preview_view_exposed's host code and view_kernel<true> run them, with the zoom divided
// by 1 << mip_level as the host does) and the element of hdr_unorm8_kernel (display_hdr_unorm8 of csrc/display.cuh).  Built by
// __graft_entry__.build() into tests/emu/libitw_view_hdr_emu.so and loaded only by tests.
#include "../../intel-texture-works-plugin_b200/csrc/display.cuh"
#include "../../intel-texture-works-plugin_b200/csrc/view.cuh"

using namespace itw;

// `src` = src_w x src_h texels of `planes` interleaved elements of `depth` bits, rows `row_bytes` apart.  `dst` receives
// width * height packed RGB8 texels.
extern "C" void emu_view_exposed(const void* src, int src_w, int src_h, int planes, int depth, long long row_bytes, int width, int height,
                                 int x, int y, double zoom, int mip_level, unsigned channels, unsigned matte, float exposure, uint8_t* dst)
{
    ViewParamsExposed V{{static_cast<const uint8_t*>(src), row_bytes, src_w, src_h, planes, depth, width, height, x, y,
                         zoom / (double)(1 << mip_level), {-1, -1, -1}, matte}, view_exposure(exposure, channels, planes)};
    view_channels(V.index, channels, planes);
    for (int yt = 0; yt < height; yt++)
        for (int xt = 0; xt < width; xt++) {
            const u32 rgb = view_texel<true>(V, xt, yt);
            uint8_t* p = dst + ((size_t)yt * width + xt) * 3;
            p[0] = (uint8_t)rgb;
            p[1] = (uint8_t)(rgb >> 8);
            p[2] = (uint8_t)(rgb >> 16);
        }
}
// The element rule of the HDR pane's conversion (display_hdr_unorm8): `n` halves -> `n` bytes
extern "C" void emu_hdr_unorm8(const uint16_t* halves, long long n, uint8_t* dst)
{
    for (long long i = 0; i < n; i++) dst[i] = (uint8_t)display_hdr_unorm8(halves[i]);
}
