// asan_main.cpp -- TEST-ONLY: the kernels' per-lane logic (emu.cpp) under AddressSanitizer / UndefinedBehaviorSanitizer.
// Every encoder and profile on random, smooth and ragged inputs; the per-warp scratch structs (unions that alias the
// shape-phase tables with the chain-phase state, lane-private palettes, the 128-bit packers) are where an index slip would
// show.  Built and run by tests/test_emu_sanitizers.py; prints "ok <blocks>" on success.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "emu.cpp"

static uint32_t rng_state = 12345u;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

template <typename T>
static void fill(std::vector<T>& v, int w, int h, int kind, uint32_t hi)
{
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            for (int c = 0; c < 4; c++) {
                uint32_t val;
                if (kind == 0) val = rnd() % hi;                                    // noise
                else if (kind == 1) val = (uint32_t)((x * 7 + y * 3 + c * 31) % hi); // smooth
                else val = ((x / 4 + y / 4) & 1) ? (rnd() % 8) : (hi - 1 - rnd() % 8); // flat blocks with tiny variance
                if (kind == 0 && c == 3 && (x & 8)) val = hi - 1;                   // opaque stripes
                v[((size_t)y * w + x) * 4 + c] = (T)val;
            }
}

int main()
{
    long long blocks = 0;
    const int sizes[][2] = {{4, 4}, {12, 4}, {20, 12}, {36, 8}, {68, 8}, {32, 32}};
    std::vector<uint8_t> out(1 << 16);
    for (const auto& wh : sizes) {
        const int w = wh[0], h = wh[1];
        for (int kind = 0; kind < 3; kind++) {
            std::vector<uint8_t> img8((size_t)w * h * 4);
            std::vector<uint16_t> img16((size_t)w * h * 4);
            fill(img8, w, h, kind, 256u);
            fill(img16, w, h, kind, 0x7C00u);
            rgba_surface s8{img8.data(), w, h, w * 4}, s16{reinterpret_cast<uint8_t*>(img16.data()), w, h, w * 8};
            emu_CompressBlocksBC1(&s8, out.data());
            emu_CompressBlocksBC3(&s8, out.data());
            emu_CompressBlocksBC4(&s8, out.data());
            emu_CompressBlocksBC5(&s8, out.data());
            for (int per_warp = 1; per_warp <= 16; per_warp *= 2) {
                if (emu_set_bc7_per_warp(per_warp) != 0) return 1;
                for (int row = 0; row < 10; row++) {
                    bc7_enc_settings st;
                    bc7_fill_profile(&st, row);
                    emu_CompressBlocksBC7(&s8, out.data(), &st);
                    blocks += (w / 4) * (h / 4);
                }
            }
            for (int row = 0; row < 5; row++) {
                bc6h_enc_settings st;
                bc6_fill_profile(&st, row);
                emu_CompressBlocksBC6H(&s16, out.data(), &st);
                blocks += (w / 4) * (h / 4);
            }
        }
    }
    printf("ok %lld\n", blocks);
    return 0;
}
