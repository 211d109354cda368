// none.cuh -- the end of the "none" save (itw_dds_save_none): the R8G8B8A8_UNORM chain goes into the DDS payload as it is.
// The plug-in's CompressToScratchImage swaps the scratch in instead of encoding it (IntelPlugin.cpp:262-268) and SaveToDDSMemory
// writes every image with rows of 4 * w_l bytes, no padding (DirectXTexDDS.cpp:1611-1815).  The device levels are padded to
// multiples of 4 (the chain kernels write them so), so one store pass moves every level of every item from its padded surface to
// its unpadded place in the payload, applying NormalizeNormalMapChain's per-texel step on the way for a normalised normal map
// (IntelPlugin.cpp:2149-2152: nothing reads the normalised levels afterwards, so normalising while storing keeps the plug-in's order).
#pragma once
#include "frontend.cuh"

namespace itw {

// One image of the payload: level l of item i.  A thread stores one quad: four consecutive texels of the image's unpadded run
// (texel j is (j % w, j / w)), so tiny tail levels share the launch with the large ones.
struct NoneImage {
    const uint8_t* src;       // the padded device level
    long long first;          // first quad of this image in the launch
    long long dst;            // byte offset of the image in the payload
    int src_stride;           // bytes between source rows
    int w, h;                 // the level's size
    int vec;                  // w % 4 == 0 and src, src_stride and dst 16-byte aligned: one 128-bit load and store per quad
};
constexpr int kNoneMaxImages = 96;    // six faces of a 16-level chain, and any 2-D chain; the table stays below 4 KiB of parameters
struct NoneLaunch {
    NoneImage img[kNoneMaxImages];
    uint8_t* dst;             // the payload
    int count;
    int normalize;            // NormalizeNormalMapChain on every texel
};

// The stored texel: as the chain holds it, or normalised (the routine normalize_kernel runs)
ITW_HD u32 none_texel(u32 v, int normalize) { return normalize ? front_normalize_rgba8(v) : v; }

#if defined(__CUDACC__)
// Every image of `P` in ONE launch, the images back to back in the quad index.  Per texel 4 B in, 4 B out.
__global__ void __launch_bounds__(256) none_store_kernel(const __grid_constant__ NoneLaunch P)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int lo = 0, hi = P.count - 1;                             // the last image whose first quad is <= q
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (q >= P.img[mid].first) lo = mid;
        else hi = mid - 1;
    }
    const NoneImage& I = P.img[lo];
    const long long n = (long long)I.w * I.h, t0 = (q - I.first) * 4;
    if (t0 >= n) return;
    uint8_t* out = P.dst + I.dst + t0 * 4;
    if (I.vec) {                                              // the quad lies in one row, 16-byte aligned on both sides
        const long long y = t0 / I.w, x = t0 - y * I.w;
        uint4 v = __ldg(reinterpret_cast<const uint4*>(I.src + y * I.src_stride + x * 4));
        v.x = none_texel(v.x, P.normalize);
        v.y = none_texel(v.y, P.normalize);
        v.z = none_texel(v.z, P.normalize);
        v.w = none_texel(v.w, P.normalize);
        *reinterpret_cast<uint4*>(out) = v;
        return;
    }
    // a ragged row (w % 4 != 0) or a payload offset that is only 4-byte aligned: four 32-bit texels, a quad may cross rows
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const long long t = t0 + k;
        if (t >= n) break;
        const long long y = t / I.w, x = t - y * I.w;
        const u32 v = __ldg(reinterpret_cast<const u32*>(I.src + y * I.src_stride + x * 4));
        reinterpret_cast<u32*>(out)[k] = none_texel(v, P.normalize);
    }
}
#endif

}  // namespace itw
