// open_raw_emu.cpp -- TEST-ONLY CPU execution of the uncompressed open path's per-texel routines (csrc/open_raw.cuh): the same
// __host__ __device__ raw_alpha_below, raw_load_texel and raw_layer_texel that open_raw_alpha_kernel and open_raw_layer_kernel run.
// Built by __graft_entry__.build() into tests/emu/libitw_open_raw_emu.so and loaded only by tests.
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
}  // namespace

// `n` source texels (raw_src_bytes(kind) bytes each) -> `n` layer texels of `planes` planes, as open_raw_layer_kernel writes them
extern "C" int emu_raw_texels(int kind, int planes, const uint8_t* src, long long n, int force, uint8_t* dst)
{
#define EMU_CASE(K)                                              \
    case K:                                                      \
        if (planes == 3) texels<K, 3>(src, n, force, dst);       \
        else texels<K, 4>(src, n, force, dst);                   \
        return 0;
    if (planes != 3 && planes != 4) return -1;
    switch (kind) {
        EMU_CASE(kRawRgba8) EMU_CASE(kRawRgbx8) EMU_CASE(kRawBgr8) EMU_CASE(kRawRgba16) EMU_CASE(kRawRgba32f)
        default: return -1;
    }
#undef EMU_CASE
}
// out[i] = 1 if source texel i (kRawRgba8, kRawRgba16 or kRawRgba32f) is NOT opaque, read through the word that holds its alpha
extern "C" int emu_raw_alpha_below(int kind, const uint8_t* src, long long n, uint8_t* out)
{
    const int bytes = kind == kRawRgba16 ? 8 : kind == kRawRgba32f ? 16 : 4;
    for (long long i = 0; i < n; i++) {
        u32 w;
        memcpy(&w, src + i * bytes + bytes - 4, 4);
        out[i] = kind == kRawRgba16 ? raw_alpha_below<kRawRgba16>(w) : kind == kRawRgba32f ? raw_alpha_below<kRawRgba32f>(w)
                                                                                            : raw_alpha_below<kRawRgba8>(w);
    }
    return 0;
}
