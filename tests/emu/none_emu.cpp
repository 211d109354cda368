// none_emu.cpp -- TEST-ONLY CPU execution of the "none" store's per-texel routine (csrc/none.cuh): the same __host__ __device__
// none_texel that none_store_kernel runs on every texel it moves into the payload.  Built by __graft_entry__.build() into
// tests/emu/libitw_none_emu.so and loaded only by tests.
#include "../../intel-texture-works-plugin_b200/csrc/none.cuh"

using namespace itw;

// `n` RGBA8 texels (one 32-bit word each) of `src` -> `dst`, as the store writes them
extern "C" void emu_none_texels(const uint32_t* src, long long n, int normalize, uint32_t* dst)
{
    for (long long i = 0; i < n; i++) dst[i] = none_texel(src[i], normalize);
}
