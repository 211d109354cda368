// open_emu.cpp -- TEST-ONLY CPU execution of the open path's per-block alpha predicate (csrc/open.cuh): the same __host__ __device__
// function open_alpha_kernel runs.  Built by __graft_entry__.build() into tests/emu/libitw_open_emu.so and loaded only by tests.
#include <cstring>
#include "../../intel-texture-works-plugin_b200/csrc/open.cuh"

using namespace itw;

// format: 77/78 (BC3) or 98/99 (BC7).  out[i] = 1 if every texel of the first `cols` x `rows` of block i is opaque.
extern "C" int emu_blocks_alpha_opaque(int format, const uint8_t* blocks, long long n, int cols, int rows, uint8_t* out)
{
    const bool bc3 = format == 77 || format == 78;
    if (!bc3 && format != 98 && format != 99) return -1;
    for (long long i = 0; i < n; i++) {
        u32 w[4];
        memcpy(w, blocks + 16 * i, 16);
        out[i] = (bc3 ? open_block_not_opaque<77>(w, cols, rows) : open_block_not_opaque<98>(w, cols, rows)) ? 0 : 1;
    }
    return 0;
}
