// bc7_rounds.cpp -- TEST-ONLY: the BC7 warp program, lane by lane on the CPU, at a chosen number of blocks per warp and round.
//
// bc7_kernel runs 16 blocks per warp in a full round and 1, 2, 4, 8 or 16 in the last one; this driver runs a whole surface
// in rounds of one such size, with the lanes of every phase in a chosen order (0 ascending, 1 descending, 2 the fixed shuffle
// 13 i + 7 mod 32), compiled for the CPU like tests/emu/emu.cpp.  Built and loaded by tests/test_bc7_emu_per_warp.py only.
#include "../../intel-texture-works-plugin_b200/csrc/itw_params.h"

using namespace itw;

extern "C" int bc7_rounds_encode(const rgba_surface* src, uint8_t* dst, const bc7_enc_settings* settings, int per_warp, int order)
{
    if (per_warp != 1 && per_warp != 2 && per_warp != 4 && per_warp != 8 && per_warp != 16) return -1;
    const SurfaceView surf{src->ptr, src->width, src->height, src->stride};
    const Bc7Params P = bc7_params_from(*settings);
    const long long nblocks = (long long)(surf.width / 4) * (surf.height / 4);
    static thread_local Bc7Warp W;
    for (long long first_block = 0; first_block < nblocks; first_block += per_warp) {
        const int nvalid = (int)((nblocks - first_block < per_warp) ? (nblocks - first_block) : per_warp);
        const long long out_block = first_block;
#define ITW_PHASE_ORDERED(call)                                                                                    \
    for (int lane_i = 0; lane_i < 32; lane_i++) {                                                                  \
        const int lane = order == 0 ? lane_i : (order == 1 ? 31 - lane_i : (int)((lane_i * 13u + 7u) & 31u));      \
        call;                                                                                                      \
    }
        ITW_BC7_PROGRAM(ITW_PHASE_ORDERED)
#undef ITW_PHASE_ORDERED
    }
    return 0;
}
