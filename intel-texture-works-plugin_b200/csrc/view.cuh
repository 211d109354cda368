// view.cuh -- the options dialog's view of one pane: IntelPlugin::FetchPreviewRGB (IntelPlugin.cpp:487-739), which
// PreviewDialog::updatePreviewBuffer (PreviewDialog.cpp:260-274) calls for both panes on every repaint, pan, zoom or channel toggle.
// Per dialog texel (xt, yt): the source texel (int((xt + xo) * zoom), int((yt + yo) * zoom)) in double, truncated toward zero; the
// matte bytes outside the source; else three channels picked by the channel table (:585-624) and stored as bytes (:626-738):
//   depth 8 / R8G8B8A8_UNORM          the byte
//   depth 16 (Photoshop's 0..32768)   ConvertTo8Bit(unsigned16) = FloatToByte(v / 32768.0)
//   depth 32 / R32G32B32A32_FLOAT     ConvertTo8Bit(f * exposure, false) = FloatToByte((double)(f * exposure)), the product in float
// The exposure is the dialog's slider (PreviewDialog.cpp:868-887, 2^(pos / 100)); InitData resets it to 1 at every DoWriteStart.
// view_kernel<false> (itw_preview_view) shows exposure 1, view_kernel<true> (itw_preview_view_exposed) the one the host passes.
// These are the front end's element converters (frontend.cuh) without the gamma step.
#pragma once
#include <type_traits>
#include "frontend.cuh"

namespace itw {

constexpr u32 kViewRed = 0x4, kViewGreen = 0x8, kViewBlue = 0x10, kViewAlpha = 0x20, kViewMask = 0x3C;   // PREVIEW_CHANNEL_*

struct ViewParams {
    const uint8_t* data;      // the source: src_w x src_h texels of `planes` interleaved elements of `depth` bits
    long long row_bytes;
    int src_w, src_h, planes, depth;
    int width, height;        // the dialog buffer
    int x, y;                 // previewOffsetX / Y
    double zoom;              // already divided by 1 << mip_level (:503-504)
    int index[3];             // the channel shown in R, G, B; -1 = 0
    u32 matte;                // 0x00BBGGRR
};
// view_kernel<true>'s parameters: the view and the exposure after view_exposure.  A struct of its own, so that view_kernel<false>
// keeps its parameter block, and with it its code.
struct ViewParamsExposed : ViewParams {
    float exposure;
};
template <bool kExposed> using ViewArgs = typename std::conditional<kExposed, ViewParamsExposed, ViewParams>::type;

// The channel table (:585-624).  0 shows RGB (:491-492).  Pure R, G, B or A show grey; in a mixture alpha takes the blue slot.  A
// channel beyond `planes` shows 0.  channelIndex[3] changes nothing that is shown.
ITW_HD void view_channels(int (&index)[3], u32 channels, int planes)
{
    u32 m = channels & kViewMask;
    if (!m) m = kViewRed | kViewGreen | kViewBlue;
    index[0] = index[1] = index[2] = -1;
    if (m == kViewRed) index[0] = index[1] = index[2] = 0;
    else if (m == kViewGreen) index[0] = index[1] = index[2] = planes > 1 ? 1 : -1;
    else if (m == kViewBlue) index[0] = index[1] = index[2] = planes > 2 ? 2 : -1;
    else if (m == kViewAlpha) index[0] = index[1] = index[2] = planes > 3 ? 3 : -1;
    else {
        if ((m & kViewRed) && planes > 0) index[0] = 0;
        if ((m & kViewGreen) && planes > 1) index[1] = 1;
        if ((m & kViewBlue) && planes > 2) index[2] = 2;
        if ((m & kViewAlpha) && planes > 3) index[2] = 3;
    }
}
// The exposure the sampling loops use (:615-621): the pure-alpha view of a source with an alpha plane resets it to 1.  In a mixture
// alpha keeps it, so the alpha shown in the blue slot moves with the slider.
ITW_HD float view_exposure(float exposure, u32 channels, int planes)
{
    return ((channels & kViewMask) == kViewAlpha && planes > 3) ? 1.0f : exposure;
}

// The source coordinate of dialog coordinate t, or -1 outside [0, n).  int(c) truncates toward zero, so c in (-1, 0) lands on 0;
// a NaN or a c beyond the int range is outside, as x86's cvttsd2si (INT_MIN) makes it in the plug-in.
ITW_HD int view_coord(int t, int offset, double zoom, int n)
{
    const double c = (double)((long long)t + offset) * zoom;
    return (c > -1.0 && c < (double)n) ? (int)c : -1;
}

// Dialog texel (xt, yt) -> r | g << 8 | b << 16.  kExposed: depth-32 elements are multiplied by V.exposure first, a float product
// (pixelSrc[i] * exposure, both float) rounded once and then widened; depths 8 and 16 ignore it, as the plug-in does.
template <bool kExposed = false>
ITW_HD u32 view_texel(const ViewArgs<kExposed>& V, int xt, int yt)
{
    const int x = view_coord(xt, V.x, V.zoom, V.src_w), y = view_coord(yt, V.y, V.zoom, V.src_h);
    if (x < 0 || y < 0) return V.matte & 0xFFFFFFu;
    const int esize = V.depth >> 3;
    const uint8_t* px = V.data + (long long)y * V.row_bytes + (long long)x * V.planes * esize;
    u32 rgb = 0u;
    for (int k = 0; k < 3; k++)
        if (V.index[k] >= 0) {
            const u32 raw = front_load_raw(px + V.index[k] * esize, V.depth);
            u32 v;
            if constexpr (kExposed)
                v = (V.depth == 32) ? front_byte((double)mul_rn(bits_float(raw), V.exposure)) : front_ldr_value(raw, V.depth, false);
            else
                v = front_ldr_value(raw, V.depth, false);
            rgb |= v << (8 * k);
        }
    return rgb;
}

#if defined(__CUDACC__)
// One thread per dialog texel, the source read straight from global memory: a gather bounded by the dialog size (1200 x 900 texels
// is 3.2 MB out).  The three bytes of a texel are stored separately: the buffer is packed RGB.
template <bool kExposed>
__global__ void __launch_bounds__(256) view_kernel(const __grid_constant__ ViewArgs<kExposed> V, uint8_t* __restrict__ dst)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)V.width * V.height) return;
    const int yt = (int)(i / V.width), xt = (int)(i - (long long)yt * V.width);
    const u32 rgb = view_texel<kExposed>(V, xt, yt);
    uint8_t* p = dst + i * 3;
    p[0] = (uint8_t)rgb;
    p[1] = (uint8_t)(rgb >> 8);
    p[2] = (uint8_t)(rgb >> 16);
}
#endif

}  // namespace itw
