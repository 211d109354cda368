// open_conv_emu.cpp -- TEST-ONLY CPU execution of the converted open path's per-texel routines (csrc/open_raw.cuh): the same
// __host__ __device__ raw_alpha_below, conv_texel (through raw_load_texel) and raw_layer_texel that open_raw_alpha_kernel and
// open_raw_layer_kernel run for the converted forms.  Built by __graft_entry__.build() into tests/emu/libitw_open_conv_emu.so and
// loaded only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/open_raw.cuh"

using namespace itw;

namespace {
template <int kSrc, int kPlanes>
void texels(const uint8_t* src, long long n, int force, uint8_t* dst)
{
    constexpr int kIn = raw_src_bytes(kSrc), kOut = kPlanes * raw_plane_bytes(kSrc);
    for (long long i = 0; i < n; i++) {
        alignas(16) uint8_t in[16];
        memcpy(in, src + i * kIn, kIn);
        u32 v[4], o[4];
        raw_load_texel<kSrc>(in, v);
        raw_layer_texel<kSrc, kPlanes>(v, force != 0, o);
        uint8_t out[16];
        for (int c = 0; c < kPlanes; c++) memcpy(out + c * raw_plane_bytes(kSrc), &o[c], raw_plane_bytes(kSrc));   // little-endian
        memcpy(dst + i * kOut, out, kOut);
    }
}
// out[i] = 1 if texel i is NOT opaque: the texel's alpha word; a texel of one or two bytes sits in slot `slot` of its word (byte or
// ushort position), the word's other slots padded with opaque bits
template <int kSrc>
void alpha(const uint8_t* src, long long n, int slot, uint8_t* out)
{
    constexpr int kIn = raw_src_bytes(kSrc);
    for (long long i = 0; i < n; i++) {
        u32 w = 0xFFFFFFFFu;
        if (kIn >= 4) memcpy(&w, src + i * kIn + kIn - 4, 4);
        else memcpy(reinterpret_cast<uint8_t*>(&w) + slot * kIn, src + i * kIn, kIn);
        out[i] = raw_alpha_below<kSrc>(w);
    }
}
}  // namespace

// `n` source texels (raw_src_bytes(kind) bytes each) -> `n` layer texels of `planes` planes, as open_raw_layer_kernel writes them
extern "C" int emu_conv_texels(int kind, int planes, const uint8_t* src, long long n, int force, uint8_t* dst)
{
#define EMU_CASE(K)                                              \
    case K:                                                      \
        if (planes == 3) texels<K, 3>(src, n, force, dst);       \
        else texels<K, 4>(src, n, force, dst);                   \
        return 0;
    if (planes != 3 && planes != 4) return -1;
    switch (kind) {
        EMU_CASE(kConvRgba16f) EMU_CASE(kConvR16f) EMU_CASE(kConvRg16f) EMU_CASE(kConvRgba16s) EMU_CASE(kConvRg16) EMU_CASE(kConvRg16s)
        EMU_CASE(kConvR16s) EMU_CASE(kConvR11g11b10f) EMU_CASE(kConvR9g9b9e5) EMU_CASE(kConvRg8) EMU_CASE(kConvRg8s) EMU_CASE(kConvRgba8s)
        EMU_CASE(kConvR8s) EMU_CASE(kConvA8) EMU_CASE(kConvBgra4) EMU_CASE(kConvBgrx4) EMU_CASE(kConvRg32f)
        default: return -1;
    }
#undef EMU_CASE
}
// out[i] = 1 if source texel i of a converted form with alpha is NOT opaque, read through the word that holds its alpha at `slot`
// (0..3 for A8, 0..1 for 4444, 0 otherwise)
extern "C" int emu_conv_alpha_below(int kind, const uint8_t* src, long long n, int slot, uint8_t* out)
{
    const int b = raw_src_bytes(kind);
    if (slot < 0 || (b >= 4 ? slot != 0 : slot * b >= 4)) return -1;
    switch (kind) {
        case kConvRgba16f: alpha<kConvRgba16f>(src, n, slot, out); return 0;
        case kConvRgba16s: alpha<kConvRgba16s>(src, n, slot, out); return 0;
        case kConvRgba8s: alpha<kConvRgba8s>(src, n, slot, out); return 0;
        case kConvA8: alpha<kConvA8>(src, n, slot, out); return 0;
        case kConvBgra4: alpha<kConvBgra4>(src, n, slot, out); return 0;
        default: return -1;
    }
}
// The product's scope decisions for a loaded DXGI format: out = {texel form (conv_kind_of, -1 if not served), target, depth, HasAlpha}
extern "C" void emu_conv_scope(unsigned dxgi, int* out)
{
    const int kind = conv_kind_of(dxgi);
    out[0] = kind;
    out[1] = kind < 0 ? 0 : conv_target_of(kind);
    out[2] = kind < 0 ? 0 : 8 * raw_plane_bytes(kind);
    out[3] = kind < 0 ? 0 : conv_has_alpha(kind);
}
