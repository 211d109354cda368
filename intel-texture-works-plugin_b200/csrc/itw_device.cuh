// itw_device.cuh -- building blocks shared by the BCn kernels (sm_90a).
//
// Float model.  The reference encoder (IntelCompressionPlugin/kernel.ispc, cited as K:line) is
// float32 code whose results depend on operation order.  The kernels reproduce the canonical
// strict-IEEE execution of that source (DESIGN.md "Canonical float model"):
//   * device code is compiled with -fmad=false (no FMA contraction), IEEE division and square
//     root (-prec-div=true -prec-sqrt=true), denormals kept (-ftz=false);
//   * float->int goes through cvt_x86(), which reproduces x86 cvttss2si (NaN / out of range ->
//     INT_MIN) instead of CUDA's saturating conversion;
//   * min/max use the SSE operand order ((a<b)?a:b, (a>b)?a:b), not fminf/fmaxf.
// Where a quantity is provably an exact small integer, integer or fused arithmetic may be used
// instead -- the result is identical by construction and each such place says why.
//
// Everything here is __host__ __device__: the kernels' per-lane logic can be executed on the CPU
// by tests/emu (a TEST-ONLY lane-by-lane emulation used to debug without a GPU).  The product
// library never runs this code on the host.
#pragma once
#include <stdint.h>
#include <math.h>
#include <string.h>

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#define ITW_HD __host__ __device__ __forceinline__
#define ITW_HD_NOINLINE __host__ __device__ __noinline__
#else
#define ITW_HD inline
#define ITW_HD_NOINLINE inline __attribute__((noinline))
#endif

#include "itw_tables.cuh"

// `#pragma unroll N` with N from a macro (pragmas are not macro-expanded): ITW_UNROLL(N)
#define ITW_PRAGMA(x) _Pragma(#x)
#define ITW_UNROLL(n) ITW_PRAGMA(unroll n)

namespace itw {

typedef uint32_t u32;

ITW_HD int cvt_x86(float f)
{
    // cvttss2si: truncation; NaN, +-inf and |f| >= 2^31 give 0x80000000
#if defined(__CUDA_ARCH__)
    int r = __float2int_rz(f);
    return (fabsf(f) < 2147483648.0f) ? r : (int)0x80000000;
#else
    if (!(f >= -2147483648.0f && f < 2147483648.0f)) return (int)0x80000000;
    return (int)f;
#endif
}
// plain truncation; only where the operand is proved to be in int range (NaN -> 0 on the GPU, INT_MIN on
// the host emulation: callers must make that difference invisible)
ITW_HD int trunc_i(float f)
{
#if defined(__CUDA_ARCH__)
    return __float2int_rz(f);
#else
    return (f == f) ? (int)f : (int)0x80000000;
#endif
}
ITW_HD float min_sse(float a, float b) { return (a < b) ? a : b; }
ITW_HD float max_sse(float a, float b) { return (a > b) ? a : b; }
ITW_HD float clamp_sse(float v, float lo, float hi) { return min_sse(max_sse(v, lo), hi); }
ITW_HD int mini(int a, int b) { return (a < b) ? a : b; }
ITW_HD int maxi(int a, int b) { return (a > b) ? a : b; }
ITW_HD int clampi(int v, int lo, int hi) { return mini(maxi(v, lo), hi); }
ITW_HD float sq(float v) { return v * v; }
ITW_HD u32 float_bits(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    u32 u; memcpy(&u, &f, 4); return u;
#endif
}
ITW_HD float bits_float(u32 u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}
ITW_HD float inf_f()
{
#if defined(__CUDA_ARCH__)
    return __int_as_float(0x7f800000);
#else
    return INFINITY;
#endif
}

// ---- exact division without the IEEE-division slow path -------------------------------------------
// q = RN(x * RN(1/d)), r = x - q*d (exact in one FMA), result = RN(q + r * RN(1/d)): the classic
// FMA-corrected quotient.  It is NOT correctly rounded for arbitrary operands, so it is only used
// where tests/test_exact_division.py proves it equal to IEEE x/d over the whole operand domain:
//   * d = 255 and any finite x (differs from x/255 only for x = -0 -> +0, which no caller can see);
//   * integer x in [0, 2^24] with d in 1..16 (moment / count);
//   * integer |x| <= 2^18 with integer d in [1, 2^18] (index-search projection; d = 0 gives NaN like 0/0).
ITW_HD float fma_rn(float a, float b, float c)
{
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return fmaf(a, b, c);
#endif
}
// Float steps that must round one by one, in the reference's order, on the GPU as on the host: no contraction into a fused
// multiply-add whatever the compiler flags.
ITW_HD float mul_rn(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
ITW_HD float add_rn(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
ITW_HD float div_rn(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
ITW_HD float div_by_rcp(float x, float d, float rcp_d)
{
    const float q = x * rcp_d;
    return fma_rn(fma_rn(-q, d, x), rcp_d, q);
}
ITW_HD float div255(float x) { return div_by_rcp(x, 255.0f, 1.0f / 255.0f); }

// ---- packed-byte integer helpers (single SASS instructions on sm_90a: IDP.4A, VABSDIFF4, PRMT) ----
ITW_HD u32 dp4a_u8(u32 a, u32 b, u32 c)          // c + sum over the four bytes of a.byte * b.byte
{
#if defined(__CUDA_ARCH__)
    return __dp4a(a, b, c);
#else
    for (int i = 0; i < 4; i++) c += ((a >> (8 * i)) & 255u) * ((b >> (8 * i)) & 255u);
    return c;
#endif
}
ITW_HD u32 absdiff_u8x4(u32 a, u32 b)            // per-byte |a - b|
{
#if defined(__CUDA_ARCH__)
    return __vabsdiffu4(a, b);
#else
    u32 r = 0;
    for (int i = 0; i < 4; i++) {
        int x = (int)((a >> (8 * i)) & 255u) - (int)((b >> (8 * i)) & 255u);
        r |= (u32)(x < 0 ? -x : x) << (8 * i);
    }
    return r;
#endif
}
ITW_HD u32 byte_perm(u32 a, u32 b, u32 sel)      // PRMT: result byte i = byte (sel nibble i) of {b:a}
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, sel);
#else
    unsigned long long w = ((unsigned long long)b << 32) | a;
    u32 r = 0;
    for (int i = 0; i < 4; i++) r |= (u32)((w >> (8 * ((sel >> (4 * i)) & 7u))) & 255u) << (8 * i);
    return r;
#endif
}
ITW_HD int popcount32(u32 v)
{
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}
ITW_HD int popcount16(u32 v)
{
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}

// Shape ids: 0..63 two-subset, 64..127 three-subset (the convention of K:1313-1314).
ITW_HD u32 shape_pattern(int shape) { return ITW_TABLE(shape_pattern)[shape]; }
ITW_HD int shape_mask(int shape, int subset)
{
    u32 m = ITW_TABLE(shape_mask01)[shape];
    u32 m0 = m & 0xFFFFu, m1 = m >> 16;
    return (int)((subset == 0) ? m0 : ((subset == 1) ? m1 : (~(m0 | m1) & 0xFFFFu)));
}
ITW_HD int shape_anchor(int shape, int subset)
{
    return (subset == 0) ? 0
                         : ((subset == 1) ? (int)ITW_TABLE(shape_anchor1)[shape] : (int)ITW_TABLE(shape_anchor2)[shape]);
}
// BC7 interpolation weight of index q at `bits` bits per index; K:675-686.  The three tables
// {0,21,43,64}, {0,9,...,64}, {0,4,...,64} are round(64 q / (2^bits - 1)) = (64 q + n/2) / n with n = 2^bits - 1,
// computed with an exact multiply-shift division (checked against the tables in tests/test_tables.py).
ITW_HD int bc7_weight(int bits, int q)
{
    const int n = (1 << bits) - 1;
    const int m = (bits == 2) ? 5462 : ((bits == 3) ? 2341 : 1093);      // ceil(2^14 / n)
    return ((64 * q + (n >> 1)) * m) >> 14;
}

// OR into a shared-memory word that other lanes of the warp OR into during the same phase (device: shared-memory atomic;
// the CPU emulation runs the lanes of a phase one after the other)
ITW_HD void shared_or(u32* p, u32 v)
{
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}

// LSB-first writer into one 128-bit block held in four registers
struct BitSink {
    u32 w0, w1, w2, w3;
    int pos;
    ITW_HD void reset() { w0 = w1 = w2 = w3 = 0; pos = 0; }
    ITW_HD void put(int nbits, u32 v)
    {
        if (nbits <= 0) return;
        if (nbits < 32) v &= (1u << nbits) - 1u;
        unsigned long long wide = (unsigned long long)v << (pos & 31);
        u32 lo = (u32)wide, hi = (u32)(wide >> 32);
        int word = pos >> 5;
        if (word == 0) { w0 |= lo; w1 |= hi; }
        else if (word == 1) { w1 |= lo; w2 |= hi; }
        else if (word == 2) { w2 |= lo; w3 |= hi; }
        else if (word == 3) { w3 |= lo; }
        pos += nbits;
    }
};

#if defined(__CUDACC__)
// ---- TMA (bulk async copy engine, SASS UBLKCP) + mbarrier helpers: global -> shared staging of texel rows ----
__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "ITW_MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra ITW_MBAR_DONE;\n"
        "bra ITW_MBAR_WAIT;\n"
        "ITW_MBAR_DONE:\n"
        "}\n" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// one contiguous run of `bytes` (multiple of 16, both addresses 16-byte aligned) into shared memory
__device__ __forceinline__ void tma_load_row(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

struct SurfaceView {
    const uint8_t* ptr;  // pointer to texel (0,0) (device memory for the kernels)
    int width, height;   // texels, multiples of 4
    int stride;          // bytes between rows
};

#if defined(__CUDACC__)
// Stage `count` consecutive blocks (raster block order, starting at block `first`) of a surface into shared
// memory as a 4-row tile: stage row y holds texel row y of every block, `block_row_bytes` bytes per block
// (16 for RGBA8, 32 for RGBA16F), `stage_row_bytes` between stage rows.  The run may wrap over several block
// rows of the surface; each contiguous piece is one TMA bulk copy (cp.async.bulk, SASS UBLKCP) completing on
// `bar`.  Called by ONE thread.  Requires 16-byte aligned surface rows (ptr and stride multiples of 16).
__device__ __forceinline__ void tma_prefetch_tile(unsigned char* stage, unsigned stage_row_bytes, unsigned long long* bar,
                                                  const SurfaceView& s, long long first, int count, unsigned block_row_bytes)
{
    const int bw = s.width >> 2;
    fence_proxy_async();                                  // earlier generic-proxy reads of this stage buffer are complete
    mbar_expect_tx(bar, 4u * (unsigned)count * block_row_bytes);
    int pos = 0;
    long long id = first;
    while (count > 0) {
        const int by = (int)(id / bw), bx = (int)(id - (long long)by * bw);
        const int n = (count < bw - bx) ? count : (bw - bx);
#pragma unroll
        for (int y = 0; y < 4; y++)
            tma_load_row(stage + y * stage_row_bytes + pos * block_row_bytes,
                         s.ptr + (size_t)(by * 4 + y) * (size_t)s.stride + (size_t)bx * block_row_bytes, (unsigned)n * block_row_bytes, bar);
        pos += n;
        id += n;
        count -= n;
    }
}
#endif

}  // namespace itw
