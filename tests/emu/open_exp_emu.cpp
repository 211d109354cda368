// open_exp_emu.cpp -- TEST-ONLY CPU execution of the expanded open path's per-texel routines (csrc/open_raw.cuh): the same
// __host__ __device__ raw_load_texel (exp_rgba8_word, and conv_texel for A4L4), raw_layer_texel, raw_alpha_below and pal_alpha_below
// that open_exp_layer_kernel, open_raw_alpha_kernel and open_pal_alpha_kernel run.  Built by __graft_entry__.build() into
// tests/emu/libitw_open_exp_emu.so and loaded only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/open_raw.cuh"

using namespace itw;

namespace {
template <int kSrc, int kPlanes>
void texels(const uint8_t* src, long long n, const u32* pal, int force, uint8_t* dst)
{
    constexpr int kIn = raw_src_bytes(kSrc);
    for (long long i = 0; i < n; i++) {
        uint8_t in[4] = {};
        memcpy(in, src + i * kIn, kIn);
        u32 v[4], o[4];
        raw_load_texel<kSrc>(in, v, pal);
        raw_layer_texel<kSrc, kPlanes>(v, force != 0, o);
        for (int c = 0; c < kPlanes; c++) dst[i * kPlanes + c] = (uint8_t)o[c];
    }
}
// out[i] = 1 if texel i is NOT opaque, read from the scan's word with the texel in slot `slot` and `fill` in the word's other slots
template <int kSrc>
void alpha(const uint8_t* src, long long n, int slot, const u32* pal, u32 fill, uint8_t* out)
{
    constexpr int kIn = raw_src_bytes(kSrc);
    uint8_t a[256];
    for (int k = 0; k < 256; k++) a[k] = pal ? (uint8_t)(pal[k] >> 24) : 0;
    for (long long i = 0; i < n; i++) {
        uint8_t w8[4];
        for (int s = 0; s < 4 / kIn; s++) memcpy(w8 + s * kIn, s == slot ? src + i * kIn : reinterpret_cast<const uint8_t*>(&fill), kIn);
        u32 w;
        memcpy(&w, w8, 4);
        if constexpr (kSrc == kExpP8 || kSrc == kExpA8p8) out[i] = pal_alpha_below<kSrc>(a, w, 4 / kIn);
        else out[i] = raw_alpha_below<kSrc>(w);
    }
}
}  // namespace

// `n` source texels of texel form `kind` (kExp*) -> `n` layer texels of `planes` byte planes, as open_exp_layer_kernel writes them;
// `pal`: 256 palette words (P8 / A8P8)
extern "C" int emu_exp_texels(int kind, int planes, const uint8_t* src, long long n, const uint32_t* pal, int force, uint8_t* dst)
{
#define EMU_CASE(K)                                                \
    case K:                                                        \
        if (planes == 3) texels<K, 3>(src, n, pal, force, dst);    \
        else texels<K, 4>(src, n, pal, force, dst);                \
        return 0;
    if (planes != 3 && planes != 4) return -1;
    if ((kind == kExpP8 || kind == kExpA8p8) && !pal) return -1;
    switch (kind) {
        EMU_CASE(kExpA4l4) EMU_CASE(kExpA8r3g3b2) EMU_CASE(kExpP8) EMU_CASE(kExpA8p8)
        default: return -1;
    }
#undef EMU_CASE
}
// out[i] = 1 if source texel i is NOT opaque by the scan's predicate, the texel at `slot` of its word (a byte for A4L4 / P8, a ushort
// for A8R3G3B2 / A8P8) and `fill` (one texel's bytes) in the other slots
extern "C" int emu_exp_alpha_below(int kind, const uint8_t* src, long long n, int slot, const uint32_t* pal, uint32_t fill, uint8_t* out)
{
    if (slot < 0 || slot * raw_src_bytes(kind) >= 4) return -1;
    if ((kind == kExpP8 || kind == kExpA8p8) && !pal) return -1;
    switch (kind) {
        case kExpA4l4: alpha<kExpA4l4>(src, n, slot, pal, fill, out); return 0;
        case kExpA8r3g3b2: alpha<kExpA8r3g3b2>(src, n, slot, pal, fill, out); return 0;
        case kExpP8: alpha<kExpP8>(src, n, slot, pal, fill, out); return 0;
        case kExpA8p8: alpha<kExpA8p8>(src, n, slot, pal, fill, out); return 0;
        default: return -1;
    }
}
// The product's decisions for a header form (ITW_EXP_*): out = {texel form, loaded format, palette (0/1), source bytes per texel}
extern "C" void emu_exp_scope(int form, int* out)
{
    out[0] = exp_kind_of(form);
    out[1] = (int)exp_loaded_of(form);
    out[2] = exp_has_palette(form);
    out[3] = raw_src_bytes(exp_kind_of(form));
}
