// itw_bcn.cu -- host side of libitw_bcn.so: the reference's C-ABI (include/itw_bcn.h section 1,
// replacing 3rdParty/Intel/Source/ispc_texcomp.cpp:20-435) plus the additive entry points.
//
// There is NO CPU fallback in this library: every encode runs the sm_90a kernels or fails with a
// message retrievable through itw_get_last_error().
//
// Threading: the reference is called concurrently from up to 64 pool threads on disjoint row
// bands (win32Threads.cpp:211-274).  All mutable state here is thread_local (one CUDA stream,
// one set of staging buffers and timing events per calling thread), so calls are re-entrant.
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/itw_bcn.h"
#include "bc4_bc5.cuh"
#include "mips.cuh"
#include "decode.cuh"
#include "display.cuh"
#include "open.cuh"
#include "open_raw.cuh"
#include "frontend.cuh"
#include "none.cuh"
#include "view.cuh"
#include "mips_f16.cuh"
#include "itw_params.h"

using namespace itw;

namespace {

std::atomic<uint64_t> g_launches{0};
std::atomic<int> g_default_device{-1};      // itw_set_devices() with ONE device: the process-wide default

constexpr uint32_t fourcc(char a, char b, char c, char d)
{
    return (uint32_t)(uint8_t)a | ((uint32_t)(uint8_t)b << 8) | ((uint32_t)(uint8_t)c << 16) | ((uint32_t)(uint8_t)d << 24);
}

// What the library knows of each block-compressed DXGI format; every host file reads these facts from here.
struct DxgiFormat {
    int dxgi;
    int bpb;                 // bytes per 4x4 block
    int encoder;             // ITW_FORMAT_* that encodes it: _SRGB as its UNORM twin, BC6H_SF16 as BC6H (IntelPlugin.cpp:840-843)
    int decoder;             // ITW_FORMAT_* of display_kernel / open_layer_kernel: _SRGB as its UNORM twin
    bool srgb;
    int twin;                // the _SRGB / UNORM twin; the format itself when it has none
    bool hdr;
    bool alpha_scan;         // the open path checks its alpha (HasAlpha; the plug-in excludes BC1)
    uint32_t fourcc;         // legacy FourCC (DirectXTexDDS.cpp:479-486), 0 = the DX10 extension only
    int family;              // front end: 0 RGBA8 colour, 1 BC4 / BC5, 2 BC6H
    int texel_bytes;         // the encoder's input texel: RGBA8 or RGBA16F
    bool itw;                // an ITW_FORMAT_* id, accepted by the format-taking entry points
};
constexpr DxgiFormat kDxgiFormats[] = {
    // dxgi bpb enc dec  srgb   twin  hdr    scan   legacy FourCC           family texel itw
    {71, 8,  71, 71, false, 72, false, false, fourcc('D', 'X', 'T', '1'), 0, 4, true},
    {72, 8,  71, 71, true,  71, false, false, 0,                          0, 4, false},
    {77, 16, 77, 77, false, 78, false, true,  fourcc('D', 'X', 'T', '5'), 0, 4, true},
    {78, 16, 77, 77, true,  77, false, true,  0,                          0, 4, false},
    {80, 8,  80, 80, false, 80, false, false, fourcc('B', 'C', '4', 'U'), 1, 4, true},
    {83, 16, 83, 83, false, 83, false, false, fourcc('B', 'C', '5', 'U'), 1, 4, true},
    {95, 16, 95, 95, false, 95, true,  false, 0,                          2, 8, true},
    {96, 16, 95, 96, false, 96, true,  false, 0,                          2, 8, true},
    {98, 16, 98, 98, false, 99, false, true,  0,                          0, 4, true},
    {99, 16, 98, 98, true,  98, false, true,  0,                          0, 4, false},
};
// The row of a DXGI format, null when the library does not know it.
inline const DxgiFormat* dxgi_format(int dxgi)
{
    for (const DxgiFormat& f : kDxgiFormats)
        if (f.dxgi == dxgi) return &f;
    return nullptr;
}
// The row of an ITW_FORMAT_* id, null for any other number.
inline const DxgiFormat* itw_format(int format)
{
    const DxgiFormat* f = dxgi_format(format);
    return f && f->itw ? f : nullptr;
}

inline int pad4(int v) { return (v + 3) & ~3; }
template <typename T> inline T lvl(T v, int l) { v >>= l; return v ? v : 1; }      // size of mip level l
inline bool pow2_dims(int w, int h) { return (w & (w - 1)) == 0 && (h & (h - 1)) == 0; }   // GenerateMipMaps then box-filters

// Device staging of one surface encode: host rows go to d_in, blocks that cannot go straight to dst come back through d_out.
struct Staging {
    uint8_t* d_in = nullptr;  size_t d_in_cap = 0;
    uint8_t* d_out = nullptr; size_t d_out_cap = 0;
};
struct ThreadCtx : Staging {
    int device = -1;             // device the resources below belong to
    int wanted_device = -1;      // itw_set_device() request, -1 = keep the current device
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool timed = false;
    uint8_t* d_mid = nullptr; size_t d_mid_cap = 0;      // itw_encode_pixels: the converted surface between the two kernels
    // band pipeline of the compute-bound encoders (encode_banded): copy-in / copy-out streams and per-band events
    cudaStream_t copy_in = nullptr, copy_out = nullptr;
    cudaEvent_t band_in[4] = {nullptr, nullptr, nullptr, nullptr}, band_done[4] = {nullptr, nullptr, nullptr, nullptr};
    int sm_count = 0;
    std::string err;
    // itw_encode_batch: three copy/compute lanes so that H2D of tile i+1, the kernel of tile i and
    // D2H of tile i-1 overlap (tile streaming, SURVEY.md 8e)
    struct Lane : Staging {
        cudaStream_t stream = nullptr;
        bool busy = false;
    } lanes[3];
    // deferred mode (itw_begin_deferred / itw_flush): host calls are enqueued on the lanes round-robin and drained by itw_flush
    bool deferred = false;
    unsigned deferred_next = 0;
    int deferred_rc = 0;
    float pool_ms = -1.0f;       // multi-device call: max over the devices of their kernel time
    void release()
    {
        // best effort: at process exit the runtime may already be unloading, errors are ignored
        if (stream) cudaStreamDestroy(stream);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
        cudaFree(d_in); cudaFree(d_out); cudaFree(d_mid);
        d_mid = nullptr; d_mid_cap = 0;
        if (copy_in) cudaStreamDestroy(copy_in);
        if (copy_out) cudaStreamDestroy(copy_out);
        copy_in = copy_out = nullptr;
        for (int i = 0; i < 4; i++) {
            if (band_in[i]) cudaEventDestroy(band_in[i]);
            if (band_done[i]) cudaEventDestroy(band_done[i]);
            band_in[i] = band_done[i] = nullptr;
        }
        for (auto& l : lanes) { if (l.stream) cudaStreamDestroy(l.stream); cudaFree(l.d_in); cudaFree(l.d_out); l = Lane(); }
        stream = nullptr; ev0 = ev1 = nullptr; d_in = d_out = nullptr; d_in_cap = d_out_cap = 0;
        cudaGetLastError();
    }
    ~ThreadCtx() { release(); }            // pool threads come and go (win32Threads.cpp:98-190)
};
thread_local ThreadCtx tls;

int fail(const char* what, cudaError_t e = cudaSuccess)
{
    char buf[512];
    if (e != cudaSuccess) snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    else snprintf(buf, sizeof(buf), "%s", what);
    tls.err = buf;
    return -1;
}
// fail() with "who: " and a formatted reason
__attribute__((format(printf, 2, 3))) int fail_in(const char* who, const char* fmt, ...)
{
    char buf[320];
    const int n = snprintf(buf, sizeof(buf), "%s: ", who);
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf + n, sizeof(buf) - n, fmt, ap);
    va_end(ap);
    return fail(buf);
}
#define ITW_CUDA(call)                                          \
    do {                                                           \
        cudaError_t e_ = (call);                                   \
        if (e_ != cudaSuccess) return fail(#call, e_);             \
    } while (0)

// A call that enqueued work on its own streams leaves through drain(), also after an error: the caller may free src / dst
// as soon as it returns, and the staging buffers must be idle for the next call.  The first failing step is the one reported.
struct FirstError {
    int rc = 0;
    bool step(cudaError_t e, const char* what) { if (rc == 0 && e != cudaSuccess) rc = fail(what, e); return rc == 0; }
    bool step(int r) { if (rc == 0 && r) rc = -1; return rc == 0; }        // r from a helper that reported through fail()
    int drain(std::initializer_list<cudaStream_t> streams)
    {
        for (cudaStream_t s : streams) step(cudaStreamSynchronize(s), "cudaStreamSynchronize");
        if (rc) cudaGetLastError();
        return rc;
    }
};

int ensure_ctx()
{
    ThreadCtx& c = tls;
    int dev = 0;
    if (c.wanted_device >= 0) {
        ITW_CUDA(cudaSetDevice(c.wanted_device));
        dev = c.wanted_device;
    } else if (g_default_device.load(std::memory_order_relaxed) >= 0) {
        dev = g_default_device.load(std::memory_order_relaxed);
        ITW_CUDA(cudaSetDevice(dev));
    } else {
        ITW_CUDA(cudaGetDevice(&dev));
    }
    if (c.device == dev && c.stream) return 0;
    if (c.stream) {                       // device changed: drop the old resources
        c.release();
        c.device = -1;
        c.timed = false;
    }
    cudaDeviceProp prop;
    ITW_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) return fail("libitw_bcn needs an sm_90a (Hopper) device");
    c.sm_count = prop.multiProcessorCount;
    ITW_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    ITW_CUDA(cudaEventCreate(&c.ev0));
    ITW_CUDA(cudaEventCreate(&c.ev1));
    ITW_CUDA(cudaFuncSetAttribute(bc7_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBc7SmemBytes));
    ITW_CUDA(cudaFuncSetAttribute(bc7_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBc7SmemBytes));
    ITW_CUDA(cudaFuncSetAttribute(bc6h_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBc6SmemBytes));
    ITW_CUDA(cudaFuncSetAttribute(bc6h_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBc6SmemBytes));
    c.device = dev;
    return 0;
}
int grow(uint8_t*& p, size_t& cap, size_t need)
{
    if (need <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    ITW_CUDA(cudaMalloc(&p, need));
    cap = need;
    return 0;
}
bool is_device_pointer(const void* p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// 0 = encode it, 1 = nothing to do, -1 = error.  Zero-height bands are legitimate: CompressImageMT hands them to the
// threads beyond height/4 (win32Threads.cpp:217-230) and the reference's loops simply do not execute (kernel.ispc:600).
int check_surface(const rgba_surface* s, const DxgiFormat& f)
{
    if (!s) return fail("null surface");
    if (s->height == 0 && s->width >= 0 && (s->width & 3) == 0) return 1;
    if (!s->ptr) return fail("null surface");
    if (s->width <= 0 || s->height < 0 || (s->width & 3) || (s->height & 3))
        return fail("surface width/height must be positive multiples of 4 (ispc_texcomp.h:93-95)");
    if ((long long)s->stride < (long long)s->width * f.texel_bytes) return fail("surface stride smaller than a texel row");
    return 0;
}

// An encoder resolved from (format, settings) before anything is enqueued: launch() can then fail only on a CUDA error.
struct Encoder {
    int format;                  // the row's encoder: BC6H_SF16 is encoded by the unsigned encoder
    DxgiFormat f;                // the row of `format`
    Bc7Params bc7;
    Bc6Params bc6;
};
int resolve_encoder(int format, const void* settings, Encoder& e)
{
    const DxgiFormat* f = itw_format(format);
    if (!f) return fail("unknown format");
    e.format = f->encoder;
    e.f = *itw_format(e.format);
    if (e.format == ITW_FORMAT_BC7) {
        if (!settings) return fail("CompressBlocksBC7: null settings");
        e.bc7 = bc7_params_from(*static_cast<const bc7_enc_settings*>(settings));
        if (const char* why = bc7_params_check(e.bc7)) return fail(why);
    } else if (e.format == ITW_FORMAT_BC6H) {
        if (!settings) return fail("CompressBlocksBC6H: null settings");
        e.bc6 = bc6_params_from(*static_cast<const bc6h_enc_settings*>(settings));
        if (const char* why = bc6_params_check(e.bc6)) return fail(why);
    }
    return 0;
}

// Enqueue the kernel for one device-resident surface on `stream`.
int launch(const Encoder& e, const SurfaceView& v, uint8_t* d_dst, cudaStream_t stream)
{
    const long long nblocks = (long long)(v.width >> 2) * (v.height >> 2);
    const bool vec16 = ((reinterpret_cast<uintptr_t>(v.ptr) | (uintptr_t)v.stride) & 15u) == 0;
    const unsigned grid1 = (unsigned)((nblocks + 127) / 128);
    switch (e.format) {
        case ITW_FORMAT_BC1:
            if (vec16) bc1_bc3_kernel<false, true><<<grid1, 128, 0, stream>>>(v, d_dst);
            else       bc1_bc3_kernel<false, false><<<grid1, 128, 0, stream>>>(v, d_dst);
            break;
        case ITW_FORMAT_BC3:
            if (vec16) bc1_bc3_kernel<true, true><<<grid1, 128, 0, stream>>>(v, d_dst);
            else       bc1_bc3_kernel<true, false><<<grid1, 128, 0, stream>>>(v, d_dst);
            break;
        case ITW_FORMAT_BC4:
            if (vec16) bc4_bc5_kernel<false, true><<<grid1, 128, 0, stream>>>(v, d_dst);
            else       bc4_bc5_kernel<false, false><<<grid1, 128, 0, stream>>>(v, d_dst);
            break;
        case ITW_FORMAT_BC5:
            if (vec16) bc4_bc5_kernel<true, true><<<grid1, 128, 0, stream>>>(v, d_dst);
            else       bc4_bc5_kernel<true, false><<<grid1, 128, 0, stream>>>(v, d_dst);
            break;
        case ITW_FORMAT_BC7: {
            // one 16-warp CTA per SM, persistent over the rounds; TMA-staged variant when the surface allows it.  The kernel
            // owns the schedule (how many blocks a warp takes per round); a surface of fewer than SMs x 16 blocks gets one CTA
            // per 16 blocks
            const bool tma = vec16;                                       // 16-byte aligned rows
            const long long cap = (long long)tls.sm_count;
            const long long want = (nblocks + kBc7WarpsPerCta - 1) / kBc7WarpsPerCta;
            const unsigned grid = (unsigned)(want < cap ? want : cap);
            if (tma) bc7_kernel<true><<<grid, kBc7WarpsPerCta * 32, kBc7SmemBytes, stream>>>(v, d_dst, e.bc7, nblocks);
            else     bc7_kernel<false><<<grid, kBc7WarpsPerCta * 32, kBc7SmemBytes, stream>>>(v, d_dst, e.bc7, nblocks);
            break;
        }
        case ITW_FORMAT_BC6H: {
            const long long want = (nblocks + kBc6TileBlocks - 1) / kBc6TileBlocks;
            const long long cap = (long long)tls.sm_count;
            const unsigned grid = (unsigned)(want < cap ? want : cap);
            if (vec16) bc6h_kernel<true><<<grid, kBc6WarpsPerCta * 32, kBc6SmemBytes, stream>>>(v, d_dst, e.bc6, nblocks);
            else       bc6h_kernel<false><<<grid, kBc6WarpsPerCta * 32, kBc6SmemBytes, stream>>>(v, d_dst, e.bc6, nblocks);
            break;
        }
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    ITW_CUDA(cudaGetLastError());
    return 0;
}

int encode_many(int format, const rgba_surface* srcs, uint8_t* const* dsts, int count, const void* settings);

// Host rows -> tight device rows: one linear copy when the rows are already tight (full PCIe rate from pinned memory), else 2-D.
cudaError_t copy_rows_h2d(uint8_t* d, const void* h, size_t h_stride, size_t row_bytes, size_t rows, cudaStream_t s)
{
    if (h_stride == row_bytes) return cudaMemcpyAsync(d, h, row_bytes * rows, cudaMemcpyHostToDevice, s);
    return cudaMemcpy2DAsync(d, row_bytes, h, h_stride, row_bytes, rows, cudaMemcpyHostToDevice, s);
}
// Stage a host pixel source in `buf` (tight rows); P.data / P.row_bytes are redirected.
int stage_pixels(uint8_t*& buf, size_t& cap, FrontParams& P, cudaStream_t s)
{
    const size_t tight = (size_t)P.width * P.planes * (P.depth / 8);
    if (grow(buf, cap, tight * P.height)) return -1;
    ITW_CUDA(copy_rows_h2d(buf, P.data, (size_t)P.row_bytes, tight, (size_t)P.height, s));
    P.data = buf;
    P.row_bytes = (long long)tight;
    return 0;
}

// The input of a staged launch: `bytes` at `ptr`, read in place when it is device memory aligned to `align` (0: never), else copied
// to d_in first.  With `pixels` (ptr == pixels->data, align 1) it is a pixel source that stage_pixels copies to d_in from the host.
struct StagedIn {
    const uint8_t* ptr;
    bool dev;
    unsigned align;
    size_t bytes;
    FrontParams* pixels = nullptr;
};
// The output: `rows` rows of `row_bytes` at `ptr` / `pitch`, written in place when it is device memory with ptr and pitch aligned
// to `align`, else written to d_out at `stage_pitch` and copied back in one 2-D copy.
struct StagedOut {
    uint8_t* ptr;
    size_t pitch;
    bool dev;
    unsigned align;
    size_t row_bytes, stage_pitch, rows;
};
// One kernel of a single-launch call: copy in, launch(d_src, d_dst, dst_stride, stream) bracketed by ev0 / ev1 for
// itw_last_kernel_ms, copy out, drain.  Device operands order the call on the legacy default stream (the rule of CompressBlocks*).
template <typename Launch>
int run_staged(const StagedIn& in, const StagedOut& out, Launch&& launch)
{
    ThreadCtx& c = tls;
    cudaStream_t s = (in.dev || out.dev) ? cudaStreamLegacy : c.stream;
    const bool in_direct = in.dev && in.align && (reinterpret_cast<uintptr_t>(in.ptr) & (in.align - 1)) == 0;
    const bool out_direct = out.dev && ((reinterpret_cast<uintptr_t>(out.ptr) | (uintptr_t)out.pitch) & (out.align - 1)) == 0;
    if (!in_direct && !in.pixels && grow(c.d_in, c.d_in_cap, in.bytes)) return -1;
    if (!out_direct && grow(c.d_out, c.d_out_cap, out.stage_pitch * out.rows)) return -1;
    uint8_t* d_dst = out_direct ? out.ptr : c.d_out;
    FirstError fe;
    if (!in_direct && in.pixels) fe.step(stage_pixels(c.d_in, c.d_in_cap, *in.pixels, s));
    else if (!in_direct) fe.step(cudaMemcpyAsync(c.d_in, in.ptr, in.bytes, in.dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s), "H2D");
    if (fe.rc == 0) fe.step(cudaEventRecord(c.ev0, s), "cudaEventRecord");
    if (fe.rc == 0) fe.step(launch(in_direct ? in.ptr : c.d_in, d_dst, (long long)(out_direct ? out.pitch : out.stage_pitch), s));
    if (fe.rc == 0 && fe.step(cudaEventRecord(c.ev1, s), "cudaEventRecord")) c.timed = true;
    if (fe.rc == 0 && !out_direct)
        fe.step(cudaMemcpy2DAsync(out.ptr, out.pitch, d_dst, out.stage_pitch, out.row_bytes, out.rows,
                                  out.dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s), "D2H");
    return fe.drain({s});
}

// One surface encode on `s` through a staging pair: a host source is copied into d_in, then the launch, then the blocks go
// straight into a 16-byte aligned device dst or through d_out and a copy back.  ev0 / ev1, when given, bracket the launch for
// itw_last_kernel_ms.  Returns false after the first failing step; the caller drains `s`.
bool encode_surface(FirstError& fe, const Encoder& e, const rgba_surface* src, bool src_dev, uint8_t* dst, bool dst_dev, Staging& b,
                    cudaStream_t s, cudaEvent_t ev0 = nullptr, cudaEvent_t ev1 = nullptr)
{
    const size_t row_bytes = (size_t)src->width * e.f.texel_bytes;
    const size_t out_bytes = (size_t)(src->width >> 2) * (src->height >> 2) * e.f.bpb;
    const bool dst_direct = dst_dev && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0;
    if (!src_dev && !fe.step(grow(b.d_in, b.d_in_cap, row_bytes * src->height))) return false;
    if (!dst_direct && !fe.step(grow(b.d_out, b.d_out_cap, out_bytes))) return false;
    SurfaceView v{src->ptr, src->width, src->height, src->stride};
    if (!src_dev) {
        if (!fe.step(copy_rows_h2d(b.d_in, src->ptr, (size_t)src->stride, row_bytes, (size_t)src->height, s), "H2D")) return false;
        v.ptr = b.d_in;
        v.stride = (int)row_bytes;
    }
    uint8_t* d_dst = dst_direct ? dst : b.d_out;
    if (ev0 && !fe.step(cudaEventRecord(ev0, s), "cudaEventRecord")) return false;
    if (!fe.step(launch(e, v, d_dst, s))) return false;
    if (ev1 && !fe.step(cudaEventRecord(ev1, s), "cudaEventRecord")) return false;
    return dst_direct || fe.step(cudaMemcpyAsync(dst, d_dst, out_bytes, dst_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s), "D2H");
}

// Host surface -> host blocks for the COMPUTE-bound encoders (BC7, BC6H): the surface is cut into four row bands whose
// H2D copies, kernels and D2H copies run on three streams, so that all but the first (small) band's input copy and all
// but the last band's output copy hide behind the kernels.  (For BC1-BC5 the copies ARE the cost -- see encode_single.)
// Bands are whole block rows; the kernels see each band as an independent surface, exactly as the reference's own
// callers do (win32Threads.cpp:217-230), so the output is unchanged.
int encode_banded(const Encoder& e, const rgba_surface* src, uint8_t* dst)
{
    ThreadCtx& c = tls;
    if (!c.copy_in) {
        ITW_CUDA(cudaStreamCreateWithFlags(&c.copy_in, cudaStreamNonBlocking));
        ITW_CUDA(cudaStreamCreateWithFlags(&c.copy_out, cudaStreamNonBlocking));
        for (int i = 0; i < 4; i++) {
            ITW_CUDA(cudaEventCreateWithFlags(&c.band_in[i], cudaEventDisableTiming));
            ITW_CUDA(cudaEventCreateWithFlags(&c.band_done[i], cudaEventDisableTiming));
        }
    }
    const size_t row_bytes = (size_t)src->width * e.f.texel_bytes;
    const size_t block_row_bytes = (size_t)(src->width >> 2) * e.f.bpb;
    const int block_rows = src->height >> 2;
    if (grow(c.d_in, c.d_in_cap, row_bytes * src->height)) return -1;
    if (grow(c.d_out, c.d_out_cap, block_row_bytes * block_rows)) return -1;
    // 1/16 of the rows first (its copy is the only exposed one), then three equal parts
    int first[5];
    first[0] = 0;
    first[1] = block_rows / 16 > 0 ? block_rows / 16 : 1;
    const int rest = block_rows - first[1];
    first[2] = first[1] + rest / 3;
    first[3] = first[1] + (2 * rest) / 3;
    first[4] = block_rows;
    // A launch works in rounds of `wave` blocks (every SM one tile); a band that ends inside a round leaves SMs idle until
    // the band's kernel is over -- four ragged bands cost BC7 4 % of a 4096 x 4096 surface.  When the surface is several waves
    // long the band borders are therefore put on wave borders (rounded down to whole block rows): the bands together then
    // need as many rounds as one launch over the whole surface.
    {
        const long long bw = src->width >> 2;
        const long long wave = (long long)c.sm_count * (e.format == ITW_FORMAT_BC7 ? kBc7TileBlocks : kBc6TileBlocks);
        const long long total = bw * block_rows, waves = total / wave;
        if (waves >= 4 && wave >= bw) {
            const long long w0 = waves / 16 > 0 ? waves / 16 : 1;                   // waves of the first band
            const long long part = (waves - w0 + 2) / 3;                           // ... of the second and the third
            first[1] = (int)(w0 * wave / bw);
            first[2] = (int)((w0 + part) * wave / bw);
            first[3] = (int)((w0 + 2 * part) * wave / bw);
            if (first[3] > block_rows) first[3] = block_rows;
            if (first[2] > first[3]) first[2] = first[3];
        }
    }
    FirstError fe;
    for (int b = 0; b < 4; b++) {
        const int r0 = first[b], r1 = first[b + 1];
        if (r1 <= r0) continue;
        const size_t rows = (size_t)(r1 - r0) * 4;
        uint8_t* d_band = c.d_in + (size_t)r0 * 4 * row_bytes;
        const uint8_t* h_band = src->ptr + (size_t)r0 * 4 * (size_t)src->stride;
        if (!fe.step(copy_rows_h2d(d_band, h_band, (size_t)src->stride, row_bytes, rows, c.copy_in), "band H2D")) break;
        if (!fe.step(cudaEventRecord(c.band_in[b], c.copy_in), "cudaEventRecord")) break;
        if (!fe.step(cudaStreamWaitEvent(c.stream, c.band_in[b], 0), "cudaStreamWaitEvent")) break;
        if (b == 0 && !fe.step(cudaEventRecord(c.ev0, c.stream), "cudaEventRecord")) break;
        const SurfaceView v{d_band, src->width, (int)rows, (int)row_bytes};
        uint8_t* d_blocks = c.d_out + (size_t)r0 * block_row_bytes;
        if (!fe.step(launch(e, v, d_blocks, c.stream))) break;
        if (!fe.step(cudaEventRecord(c.band_done[b], c.stream), "cudaEventRecord")) break;
        if (!fe.step(cudaStreamWaitEvent(c.copy_out, c.band_done[b], 0), "cudaStreamWaitEvent")) break;
        if (!fe.step(cudaMemcpyAsync(dst + (size_t)r0 * block_row_bytes, d_blocks, (size_t)(r1 - r0) * block_row_bytes, cudaMemcpyDeviceToHost,
                                     c.copy_out), "band D2H")) break;
    }
    if (fe.rc == 0 && fe.step(cudaEventRecord(c.ev1, c.stream), "cudaEventRecord")) c.timed = true;
    return fe.drain({c.copy_in, c.stream, c.copy_out});
}

// A lane's stream exists and its staging buffers are idle (they may still be in flight from three calls ago).
int lane_ready(ThreadCtx::Lane& L)
{
    if (!L.stream) ITW_CUDA(cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
    if (L.busy) {
        ITW_CUDA(cudaStreamSynchronize(L.stream));
        L.busy = false;
    }
    return 0;
}
void drain_lanes(ThreadCtx& c, FirstError& fe)
{
    for (auto& L : c.lanes)
        if (L.busy) {
            fe.step(cudaStreamSynchronize(L.stream), "cudaStreamSynchronize");
            L.busy = false;
        }
}
// Device-resident operands were produced on the caller's blocking streams: order `s` after what is already enqueued on the
// legacy default stream (the ordering rule of CompressBlocks*, see itw_bcn.h).  Uses ev0, so the call reports no kernel time.
int order_after_legacy(cudaStream_t s)
{
    tls.timed = false;
    if (cudaEventRecord(tls.ev0, cudaStreamLegacy) != cudaSuccess || cudaStreamWaitEvent(s, tls.ev0, 0) != cudaSuccess) return fail("stream ordering");
    return 0;
}

// Deferred mode (itw_begin_deferred .. itw_flush): a host -> host encode is enqueued on one of three lanes (stream +
// staging buffers) and the call returns; the H2D copy of call i+1 overlaps the kernel of call i and the D2H copy of call
// i-1.  The caller keeps src and dst valid until itw_flush().  This is what makes the reference's unchanged slice loop
// (IntelPlugin.cpp:851-879: one CompressImageMT per 256 K-texel slice) cheap: no synchronisation per slice.
int encode_deferred(const Encoder& e, const rgba_surface* src, uint8_t* dst)
{
    ThreadCtx& c = tls;
    ThreadCtx::Lane& L = c.lanes[c.deferred_next++ % 3];
    if (lane_ready(L)) return -1;
    FirstError fe;
    L.busy = true;
    encode_surface(fe, e, src, false, dst, false, L, L.stream);
    c.timed = false;
    return fe.rc;
}

// One device: src and dst may each be host or device memory.
int encode_single(const Encoder& e, const rgba_surface* src, uint8_t* dst)
{
    if (ensure_ctx()) return -1;
    ThreadCtx& c = tls;
    const bool src_dev = is_device_pointer(src->ptr), dst_dev = is_device_pointer(dst);
    if (!src_dev && !dst_dev && c.deferred) {
        const int rc = encode_deferred(e, src, dst);
        if (rc && c.deferred_rc == 0) c.deferred_rc = rc;
        return rc;
    }
    if (!src_dev && !dst_dev && (e.format == ITW_FORMAT_BC7 || e.format == ITW_FORMAT_BC6H) && src->height >= 256)
        return encode_banded(e, src, dst);
    // (Splitting one large host surface into pipelined row bands was measured and rejected for BC1-BC5: the H2D copy is
    //  >90 % of the BC1 end-to-end time, so overlap buys <0.1 ms while eight smaller copies cost 0.3 ms.)
    // Device-resident operands were produced by the caller's own streams.  The legacy default stream orders
    // after every blocking stream (torch's default stream included), which gives the synchronous call the
    // semantics a caller expects; pure host calls use this thread's private non-blocking stream.
    cudaStream_t s = (src_dev || dst_dev) ? cudaStreamLegacy : c.stream;
    FirstError fe;
    if (encode_surface(fe, e, src, src_dev, dst, dst_dev, c, s, c.ev0, c.ev1)) c.timed = true;
    return fe.drain({s});
}

// ---------------------------------------------------------------------------------------------------------------
// Multi-device engine (SURVEY.md 8e, the GPU analogue of the reference's thread pool, win32Threads.cpp:98-274).
// itw_set_devices() creates one worker thread per selected GPU; every worker owns that device's ThreadCtx (streams,
// staging buffers).  A host -> host call is then cut into one row band per device (whole block rows, like the
// reference's per-thread bands, win32Threads.cpp:217-230 -- bands are independent surfaces, so the bytes are those
// of a single-device encode), every worker runs its band through the single-device path above (H2D, kernels and D2H
// on its own PCIe link) and writes straight into the caller's dst.  One process, one call, no collective.
// ---------------------------------------------------------------------------------------------------------------
class DevicePool {
public:
    explicit DevicePool(const std::vector<int>& devices)
    {
        for (int d : devices) workers_.emplace_back(new Worker(d));
    }
    ~DevicePool()
    {
        for (auto& w : workers_) {
            { std::lock_guard<std::mutex> g(w->m); w->quit = true; }
            w->cv.notify_all();
            w->thread.join();
        }
    }
    int size() const { return (int)workers_.size(); }
    int device(int i) const { return workers_[i]->device; }
    // Run jobs[i] on worker i (empty functions are skipped); returns 0 or -1 with the first worker's error as this thread's
    // error.  The calling thread times no kernel of its own; `ms`, when given, receives the largest kernel time of the workers.
    int run(const std::vector<std::function<int()>>& jobs, float* ms = nullptr)
    {
        std::lock_guard<std::mutex> serial(run_mutex_);           // concurrent callers take turns
        for (size_t i = 0; i < workers_.size() && i < jobs.size(); i++) {
            Worker& w = *workers_[i];
            if (!jobs[i]) continue;
            { std::lock_guard<std::mutex> g(w.m); w.job = &jobs[i]; w.done = false; }
            w.cv.notify_all();
        }
        int rc = 0;
        float most = -1.0f;
        std::string err;
        for (size_t i = 0; i < workers_.size() && i < jobs.size(); i++) {
            Worker& w = *workers_[i];
            if (!jobs[i]) continue;
            std::unique_lock<std::mutex> g(w.m);
            w.cv.wait(g, [&] { return w.done; });
            if (w.rc != 0 && rc == 0) { rc = -1; err = w.err; }
            if (w.ms > most) most = w.ms;
        }
        tls.timed = false;
        if (ms) *ms = most;
        return rc ? fail(err.c_str()) : 0;
    }

private:
    struct Worker {
        int device;
        std::mutex m;
        std::condition_variable cv;
        const std::function<int()>* job = nullptr;
        bool done = true, quit = false;
        int rc = 0;
        float ms = -1.0f;
        std::string err;
        std::thread thread;
        explicit Worker(int dev) : device(dev), thread([this] { loop(); }) {}
        void loop()
        {
            tls.wanted_device = device;                           // this thread's ThreadCtx lives on `device`
            for (;;) {
                const std::function<int()>* j;
                {
                    std::unique_lock<std::mutex> g(m);
                    cv.wait(g, [&] { return quit || job; });
                    if (quit) break;
                    j = job;
                }
                tls.err.clear();
                const int r = (*j)();
                float t = -1.0f;
                if (tls.timed && cudaEventElapsedTime(&t, tls.ev0, tls.ev1) != cudaSuccess) { cudaGetLastError(); t = -1.0f; }
                {
                    std::lock_guard<std::mutex> g(m);
                    rc = r; err = tls.err; ms = t; job = nullptr; done = true;
                }
                cv.notify_all();
            }
            tls.release();                                        // free this device's buffers on the owning thread
        }
    };
    std::vector<std::unique_ptr<Worker>> workers_;
    std::mutex run_mutex_;
};
std::mutex g_pool_mutex;
std::shared_ptr<DevicePool> g_pool;                               // null = single-device behaviour
std::shared_ptr<DevicePool> current_pool()
{
    std::lock_guard<std::mutex> g(g_pool_mutex);
    return g_pool;
}
// smallest band worth a device of its own: below this the per-device launch + copy latency outweighs the split
constexpr long long kPoolMinBlocksPerDevice = 4096;

int encode_fanout(DevicePool& pool, const Encoder& e, const rgba_surface* src, uint8_t* dst)
{
    const int block_rows = src->height >> 2;
    const long long blocks_per_row = src->width >> 2;
    int n = pool.size();
    while (n > 1 && ((long long)block_rows * blocks_per_row) / n < kPoolMinBlocksPerDevice) n--;
    if (n > block_rows) n = block_rows;
    const size_t block_row_bytes = (size_t)blocks_per_row * e.f.bpb;
    std::vector<rgba_surface> bands((size_t)n);
    std::vector<std::function<int()>> jobs((size_t)pool.size());
    for (int i = 0; i < n; i++) {
        const int r0 = (int)((long long)block_rows * i / n), r1 = (int)((long long)block_rows * (i + 1) / n);
        bands[i] = rgba_surface{src->ptr + (size_t)r0 * 4 * (size_t)src->stride, src->width, (r1 - r0) * 4, src->stride};
        uint8_t* out = dst + (size_t)r0 * block_row_bytes;
        const rgba_surface* band = &bands[i];
        if (r1 > r0) jobs[i] = [=, &e]() { return encode_single(e, band, out); };
    }
    return pool.run(jobs, &tls.pool_ms);
}

// The CompressBlocks* path.
int encode_any(int format, const rgba_surface* src, uint8_t* dst, const void* settings)
{
    tls.err.clear();
    tls.pool_ms = -1.0f;
    const DxgiFormat* f = itw_format(format);
    if (!f) return fail("unknown format");
    const int chk = check_surface(src, *f);
    if (chk) return chk < 0 ? -1 : 0;
    if (!dst) return fail("null dst");
    Encoder e;
    if (resolve_encoder(format, settings, e)) {
        if (tls.deferred && tls.deferred_rc == 0) tls.deferred_rc = -1;      // reported again by itw_flush
        return -1;
    }
    if (std::shared_ptr<DevicePool> pool = current_pool()) {
        if (pool->size() > 1 && !tls.deferred && (long long)(src->width >> 2) * (src->height >> 2) >= 2 * kPoolMinBlocksPerDevice &&
            !is_device_pointer(src->ptr) && !is_device_pointer(dst))
            return encode_fanout(*pool, e, src, dst);
    }
    return encode_single(e, src, dst);
}


// ---- decoders (decode.cuh): blocks -> RGBA8 (BC1/3/4/5/7) or RGBA16F (BC6H) surface; either side host or device ----
template <int kFormat>
void launch_decode_as(bool vec16, unsigned grid, cudaStream_t s, const uint8_t* blocks, uint8_t* dst, int w, int h, long long stride)
{
    if (vec16) decode_kernel<kFormat, true><<<grid, 128, 0, s>>>(blocks, dst, w, h, stride);
    else       decode_kernel<kFormat, false><<<grid, 128, 0, s>>>(blocks, dst, w, h, stride);
}
int launch_decode(int format, const uint8_t* d_blocks, uint8_t* d_dst, int w, int h, long long stride, cudaStream_t s)
{
    const long long nblocks = (long long)(w >> 2) * (h >> 2);
    const unsigned grid = (unsigned)((nblocks + 127) / 128);
    const bool vec16 = ((reinterpret_cast<uintptr_t>(d_dst) | (uintptr_t)stride) & 15u) == 0;
    switch (format) {
        case ITW_FORMAT_BC1: launch_decode_as<ITW_FORMAT_BC1>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        case ITW_FORMAT_BC3: launch_decode_as<ITW_FORMAT_BC3>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        case ITW_FORMAT_BC4: launch_decode_as<ITW_FORMAT_BC4>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        case ITW_FORMAT_BC5: launch_decode_as<ITW_FORMAT_BC5>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        case ITW_FORMAT_BC6H: launch_decode_as<ITW_FORMAT_BC6H>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        case ITW_FORMAT_BC6H_SF16: launch_decode_as<ITW_FORMAT_BC6H_SF16>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        case ITW_FORMAT_BC7: launch_decode_as<ITW_FORMAT_BC7>(vec16, grid, s, d_blocks, d_dst, w, h, stride); break;
        default: return fail("unknown format");
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    ITW_CUDA(cudaGetLastError());
    return 0;
}
int decode_any(int format, const uint8_t* blocks, const rgba_surface* dst)
{
    tls.err.clear();
    const DxgiFormat* f = itw_format(format);
    if (!f) return fail("unknown format");
    if (const int chk = check_surface(dst, *f)) return chk < 0 ? -1 : 0;
    if (!blocks) return fail("null blocks");
    if (ensure_ctx()) return -1;
    const size_t row_bytes = (size_t)dst->width * f->texel_bytes;
    const size_t in_bytes = (size_t)(dst->width >> 2) * (dst->height >> 2) * f->bpb;
    const StagedIn in{blocks, is_device_pointer(blocks), 16, in_bytes};
    const StagedOut out{dst->ptr, (size_t)dst->stride, is_device_pointer(dst->ptr), 4, row_bytes, row_bytes, (size_t)dst->height};
    return run_staged(in, out, [&](const uint8_t* d_blocks, uint8_t* d_dst, long long stride, cudaStream_t s) {
        return launch_decode(f->decoder, d_blocks, d_dst, dst->width, dst->height, stride, s);
    });
}


// ---- pixel-format front end (frontend.cuh) ----
int front_params(FrontParams& P, int format, const itw_pixel_source* src, uint32_t flags)
{
    const DxgiFormat* f = itw_format(format);
    if (!f) return fail("unknown format");
    if (!src || !src->data) return fail("null pixel source");
    if (src->width <= 0 || src->height <= 0) return fail("pixel source: width/height must be positive");
    if (pad4(src->height) > 65535) return fail("pixel source: height above 65532");      // one grid row per (padded) output row
    if (src->planes < 1 || src->planes > 4) return fail("pixel source: planes must be 1..4");
    if (src->depth != 8 && src->depth != 16 && src->depth != 32) return fail("pixel source: depth must be 8, 16 or 32");
    if (flags & ~31u) return fail("unknown front-end flag");
    const int esize = src->depth / 8;
    const long long tight = (long long)src->width * src->planes * esize;
    const long long row_bytes = src->row_bytes ? src->row_bytes : tight;
    if (row_bytes < tight) return fail("pixel source: row_bytes smaller than a texel row");
    if ((reinterpret_cast<uintptr_t>(src->data) | (uintptr_t)row_bytes) & (uintptr_t)(esize - 1)) return fail("pixel source: misaligned elements");
    const int family = f->family;
    if (flags & ITW_FRONT_HAS_ALPHA) {
        // the converters read plane 3 (IntelPlugin.cpp:310, :758 ...); the 32-bit HDR one reads plane 2 (:361)
        const int need = (family == 2 && src->depth == 32) ? 3 : 4;
        if (src->planes < need) return fail("ITW_FRONT_HAS_ALPHA needs an alpha plane in the source");
    }
    P = FrontParams{static_cast<const uint8_t*>(src->data), src->width, src->height, src->planes, src->depth, row_bytes, family, flags};
    return 0;
}
template <int kDepth>
void launch_front_x4(const FrontParams& P, dim3 grid, cudaStream_t s, uint8_t* d_dst, int dw, int dh, long long dstride)
{
    switch (P.planes) {
        case 1: front_kernel_x4<kDepth, 1><<<grid, 256, 0, s>>>(P, d_dst, dw, dh, dstride); break;
        case 2: front_kernel_x4<kDepth, 2><<<grid, 256, 0, s>>>(P, d_dst, dw, dh, dstride); break;
        case 3: front_kernel_x4<kDepth, 3><<<grid, 256, 0, s>>>(P, d_dst, dw, dh, dstride); break;
        default: front_kernel_x4<kDepth, 4><<<grid, 256, 0, s>>>(P, d_dst, dw, dh, dstride); break;
    }
}
int launch_front(const FrontParams& P, uint8_t* d_dst, int dw, int dh, long long dstride, cudaStream_t s)
{
    const bool quads = (dw & 3) == 0 && ((reinterpret_cast<uintptr_t>(d_dst) | (uintptr_t)dstride) & 15u) == 0 &&
                       ((reinterpret_cast<uintptr_t>(P.data) | (uintptr_t)P.row_bytes) & 3u) == 0;
    if (quads) {
        dim3 grid((unsigned)(((dw + 7) / 8 + 255) / 256), (unsigned)dh);      // two quads per thread
        if (P.depth == 8) launch_front_x4<8>(P, grid, s, d_dst, dw, dh, dstride);
        else if (P.depth == 16) launch_front_x4<16>(P, grid, s, d_dst, dw, dh, dstride);
        else launch_front_x4<32>(P, grid, s, d_dst, dw, dh, dstride);
    } else {
        dim3 grid((unsigned)((dw + 255) / 256), (unsigned)dh);
        front_kernel<<<grid, 256, 0, s>>>(P, d_dst, dw, dh, dstride);
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    ITW_CUDA(cudaGetLastError());
    return 0;
}

// The w x h surface at `src` padded to pw x ph tight rows at `dst` by edge replication (DoPaddingToMultiplesOf4).
int launch_pad(const uint8_t* src, int w, int h, long long stride, int texel_bytes, uint8_t* dst, int pw, int ph, cudaStream_t s)
{
    const dim3 grid((unsigned)((pw + 63) / 64), (unsigned)ph);
    if (texel_bytes == 8) pad_f16_kernel<<<grid, 64, 0, s>>>(src, w, h, stride, dst, pw, (long long)pw * 8);
    else pad_rgba8_kernel<<<grid, 64, 0, s>>>(src, w, h, (int)stride, dst, pw, pw * 4);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail("pad kernel", e);
}
// Every texel of the w x h surface at `dst` set to (lo, hi); `words` 32-bit words per texel.
int launch_fill(uint8_t* dst, int w, int h, long long stride, int words, u32 lo, u32 hi, cudaStream_t s)
{
    fill_texels_kernel<<<dim3((unsigned)((w + 255) / 256), (unsigned)h), 256, 0, s>>>(dst, w, h, stride, words, lo, hi);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail("fill_texels_kernel", e);
}
// Convert(R16G16B16A16_FLOAT -> R8G8B8A8_UNORM) of the w x h RGBA16F image at `src` into `dst` (4-byte aligned, as `dstride`).
int launch_hdr_unorm8(const uint8_t* src, long long sstride, int w, int h, uint8_t* dst, long long dstride, cudaStream_t s)
{
    hdr_unorm8_kernel<<<dim3((unsigned)((w + 255) / 256), (unsigned)h), 256, 0, s>>>(src, sstride, w, h, dst, dstride);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail("hdr_unorm8_kernel", e);
}
// NormalizeNormalMapChain's per-texel step over the w x h surface at `p`: RGBA16F when `hdr`, else RGBA8.
int launch_normalize(uint8_t* p, int w, int h, long long stride, bool hdr, cudaStream_t s)
{
    normalize_kernel<<<dim3((unsigned)((w + 255) / 256), (unsigned)h), 256, 0, s>>>(p, w, h, stride, hdr ? 1 : 0);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail("normalize_kernel", e);
}

// ---- document layers (mip maps from layers, cube face layers, the layer-0 panes) ----
// The planes of a layer that are read: colour planes 0..channel_count-1, and its alpha plane when the document has alpha.
// Bytes of the lw x lh rectangle of `L` staged by stage_layer: one 16-byte aligned tight plane per plane read.
size_t layer_stage_bytes(const itw_layer_source& L, int lw, int lh, int depth, bool alpha)
{
    const size_t plane = ((size_t)lw * lh * (depth / 8) + 15) & ~(size_t)15;
    return plane * (size_t)(L.channel_count + (alpha && L.alpha ? 1 : 0));
}
// Copy the lw x lh top-left rectangle of every plane of `L` that is read (any memory; rows L.row_bytes apart, or one row of the
// dw-texel document) to tight planes from `dst` on, and describe them in plane[], channels, lw and lh of `v`.  `dst` ends past them.
int stage_layer(const itw_layer_source& L, int dw, int lw, int lh, int depth, bool alpha, uint8_t*& dst, LayerLevel& v, cudaStream_t s)
{
    const size_t row = (size_t)lw * (depth / 8), plane = (row * lh + 15) & ~(size_t)15;
    const size_t pitch = L.row_bytes ? (size_t)L.row_bytes : (size_t)dw * (depth / 8);
    v.lw = lw;
    v.lh = lh;
    v.channels = L.channel_count;
    for (int p = 0; p < 4; p++) {
        const void* src = p < L.channel_count ? L.channels[p] : (p == 3 && alpha ? L.alpha : nullptr);
        if (!src) continue;
        v.plane[p] = dst;
        const cudaError_t e = cudaMemcpy2DAsync(dst, row, src, pitch, row, (size_t)lh, cudaMemcpyDefault, s);
        if (e != cudaSuccess) return fail("layer H2D", e);
        dst += plane;
    }
    return 0;
}
// Whether a plane of layers[0..n) that is read is device memory.  A layer whose channel 0 is null (a missing cube face) is not read.
bool layers_on_device(const itw_layer_source* layers, int n, bool alpha)
{
    for (int i = 0; i < n; i++) {
        const itw_layer_source& L = layers[i];
        if (!L.channels[0]) continue;
        for (int p = 0; p < L.channel_count; p++)
            if (is_device_pointer(L.channels[p])) return true;
        if (alpha && L.alpha && is_device_pointer(L.alpha)) return true;
    }
    return false;
}

int convert_any(int format, const itw_pixel_source* src, uint32_t flags, const rgba_surface* dst)
{
    tls.err.clear();
    FrontParams P;
    if (front_params(P, format, src, flags)) return -1;
    if (!dst || !dst->ptr) return fail("null surface");
    const int texel = itw_format(format)->texel_bytes;
    if (!((dst->width == P.width && dst->height == P.height) || (dst->width == pad4(P.width) && dst->height == pad4(P.height))))
        return fail("itw_convert_pixels: dst must have the source size or that size rounded up to multiples of 4");
    if ((long long)dst->stride < (long long)dst->width * texel) return fail("surface stride smaller than a texel row");
    if (ensure_ctx()) return -1;
    const size_t row_bytes = (size_t)dst->width * texel;
    const StagedIn in{P.data, is_device_pointer(P.data), 1, 0, &P};
    const StagedOut out{dst->ptr, (size_t)dst->stride, is_device_pointer(dst->ptr), (unsigned)texel, row_bytes, row_bytes, (size_t)dst->height};
    return run_staged(in, out, [&](const uint8_t*, uint8_t* d_dst, long long stride, cudaStream_t s) {
        return launch_front(P, d_dst, dst->width, dst->height, stride, s);
    });
}
// convert + pad + encode; the intermediate surface never leaves the GPU
int encode_pixels_any(int format, const itw_pixel_source* src, uint32_t flags, const void* settings, uint8_t* dst)
{
    tls.err.clear();
    FrontParams P;
    if (front_params(P, format, src, flags)) return -1;
    if (!dst) return fail("null dst");
    Encoder e;
    if (resolve_encoder(format, settings, e)) return -1;
    if (ensure_ctx()) return -1;
    ThreadCtx& c = tls;
    const int pw = pad4(P.width), ph = pad4(P.height);
    const size_t mid_row = (size_t)pw * e.f.texel_bytes;
    if (grow(c.d_mid, c.d_mid_cap, mid_row * ph)) return -1;
    const bool src_dev = is_device_pointer(P.data), dst_dev = is_device_pointer(dst);
    cudaStream_t s = (src_dev || dst_dev) ? cudaStreamLegacy : c.stream;
    const rgba_surface mid{c.d_mid, pw, ph, (int)mid_row};
    FirstError fe;
    if (!src_dev) fe.step(stage_pixels(c.d_in, c.d_in_cap, P, s));
    if (fe.rc == 0) fe.step(cudaEventRecord(c.ev0, s), "cudaEventRecord");
    if (fe.rc == 0) fe.step(launch_front(P, c.d_mid, pw, ph, (long long)mid_row, s));
    if (fe.rc == 0 && encode_surface(fe, e, &mid, true, dst, dst_dev, c, s, nullptr, c.ev1)) c.timed = true;
    return fe.drain({s});
}

}  // namespace

extern "C" {

// ---- profiles (ispc_texcomp.cpp:20-410) ----
void GetProfile_ultrafast(bc7_enc_settings* s) { bc7_fill_profile(s, 0); }
void GetProfile_veryfast(bc7_enc_settings* s) { bc7_fill_profile(s, 1); }
void GetProfile_fast(bc7_enc_settings* s) { bc7_fill_profile(s, 2); }
void GetProfile_basic(bc7_enc_settings* s) { bc7_fill_profile(s, 3); }
void GetProfile_slow(bc7_enc_settings* s) { bc7_fill_profile(s, 4); }
void GetProfile_alpha_ultrafast(bc7_enc_settings* s) { bc7_fill_profile(s, 5); }
void GetProfile_alpha_veryfast(bc7_enc_settings* s) { bc7_fill_profile(s, 6); }
void GetProfile_alpha_fast(bc7_enc_settings* s) { bc7_fill_profile(s, 7); }
void GetProfile_alpha_basic(bc7_enc_settings* s) { bc7_fill_profile(s, 8); }
void GetProfile_alpha_slow(bc7_enc_settings* s) { bc7_fill_profile(s, 9); }
void GetProfile_bc6h_veryfast(bc6h_enc_settings* s) { bc6_fill_profile(s, 0); }
void GetProfile_bc6h_fast(bc6h_enc_settings* s) { bc6_fill_profile(s, 1); }
void GetProfile_bc6h_basic(bc6h_enc_settings* s) { bc6_fill_profile(s, 2); }
void GetProfile_bc6h_slow(bc6h_enc_settings* s) { bc6_fill_profile(s, 3); }
void GetProfile_bc6h_veryslow(bc6h_enc_settings* s) { bc6_fill_profile(s, 4); }

// ---- the reference's encode entry points (ispc_texcomp.cpp:417-435) ----
void CompressBlocksBC1(const rgba_surface* src, uint8_t* dst) { encode_any(ITW_FORMAT_BC1, src, dst, nullptr); }
void CompressBlocksBC3(const rgba_surface* src, uint8_t* dst) { encode_any(ITW_FORMAT_BC3, src, dst, nullptr); }
void CompressBlocksBC6H(const rgba_surface* src, uint8_t* dst, bc6h_enc_settings* settings) { encode_any(ITW_FORMAT_BC6H, src, dst, settings); }
void CompressBlocksBC7(const rgba_surface* src, uint8_t* dst, bc7_enc_settings* settings) { encode_any(ITW_FORMAT_BC7, src, dst, settings); }

// ---- additive ----
void CompressBlocksBC4(const rgba_surface* src, uint8_t* dst) { encode_any(ITW_FORMAT_BC4, src, dst, nullptr); }
void CompressBlocksBC5(const rgba_surface* src, uint8_t* dst) { encode_any(ITW_FORMAT_BC5, src, dst, nullptr); }

int itw_bytes_per_block(int format)
{
    const DxgiFormat* f = itw_format(format);
    return f ? f->bpb : 0;
}

int itw_encode_device(int format, const rgba_surface* src, uint8_t* dst, const void* settings, void* cuda_stream)
{
    tls.err.clear();
    const DxgiFormat* f = itw_format(format);
    if (!f) return fail("unknown format");
    if (const int chk = check_surface(src, *f)) return chk < 0 ? -1 : 0;
    if (!dst) return fail("null dst");
    if (reinterpret_cast<uintptr_t>(dst) & 15u) return fail("itw_encode_device: dst must be 16-byte aligned");
    Encoder e;
    if (resolve_encoder(format, settings, e)) return -1;
    if (ensure_ctx()) return -1;
    tls.timed = false;
    SurfaceView v{src->ptr, src->width, src->height, src->stride};
    return launch(e, v, dst, static_cast<cudaStream_t>(cuda_stream));
}

int itw_decode(int format, const uint8_t* blocks, const rgba_surface* dst) { return decode_any(format, blocks, dst); }
int itw_convert_pixels(int format, const itw_pixel_source* src, uint32_t flags, const rgba_surface* dst) { return convert_any(format, src, flags, dst); }
int itw_encode_pixels(int format, const itw_pixel_source* src, uint32_t flags, const void* settings, uint8_t* dst_blocks)
{
    return encode_pixels_any(format, src, flags, settings, dst_blocks);
}

int itw_encode_batch(int format, const rgba_surface* srcs, uint8_t* const* dsts, int count, const void* settings)
{
    tls.err.clear();
    return encode_many(format, srcs, dsts, count, settings);
}

}  // extern "C"

namespace {
// Tiles i = first, first+step, ... of the batch on THIS thread's device, pipelined over the three lanes.
int encode_many_single(const Encoder& e, const rgba_surface* srcs, uint8_t* const* dsts, int count, int first, int step)
{
    if (ensure_ctx()) return -1;
    ThreadCtx& c = tls;
    FirstError fe;
    drain_lanes(c, fe);
    bool any_dev = false;                                // then every lane waits for the caller's streams, once per call
    for (int i = first; i < count && !any_dev; i += step) any_dev = is_device_pointer(srcs[i].ptr) || is_device_pointer(dsts[i]);
    if (any_dev)
        for (auto& L : c.lanes)
            if (!fe.step(lane_ready(L)) || !fe.step(order_after_legacy(L.stream))) break;
    unsigned turn = 0;
    for (int i = first; i < count && fe.rc == 0; i += step) {
        if (srcs[i].height == 0) continue;                 // zero-height tiles: nothing to do (check_surface)
        ThreadCtx::Lane& L = c.lanes[turn++ % 3];
        if (!fe.step(lane_ready(L))) break;
        L.busy = true;
        encode_surface(fe, e, &srcs[i], is_device_pointer(srcs[i].ptr), dsts[i], is_device_pointer(dsts[i]), L, L.stream);
    }
    drain_lanes(c, fe);
    tls.timed = false;
    return fe.rc;
}
int encode_many(int format, const rgba_surface* srcs, uint8_t* const* dsts, int count, const void* settings)
{
    tls.pool_ms = -1.0f;
    if (count < 0 || (count > 0 && (!srcs || !dsts))) return fail("itw_encode_batch: bad arguments");
    Encoder e;
    if (resolve_encoder(format, settings, e)) return -1;
    for (int i = 0; i < count; i++) {
        const int chk = check_surface(&srcs[i], e.f);
        if (chk < 0) return -1;
        if (chk == 0 && !dsts[i]) return fail("null dst");
    }
    // tile stream over several devices (SURVEY.md 8e, config C5): host tiles are dealt round-robin, every device runs its
    // own three-lane pipeline; no collective
    if (std::shared_ptr<DevicePool> pool = current_pool()) {
        bool host_only = count >= 2 && pool->size() > 1;
        for (int i = 0; i < count && host_only; i++)
            host_only = srcs[i].ptr && dsts[i] && !is_device_pointer(srcs[i].ptr) && !is_device_pointer(dsts[i]);
        if (host_only) {
            const int n = pool->size() < count ? pool->size() : count;
            std::vector<std::function<int()>> jobs((size_t)pool->size());
            for (int k = 0; k < n; k++) jobs[k] = [=, &e]() { return encode_many_single(e, srcs, dsts, count, k, n); };
            return pool->run(jobs);
        }
    }
    return encode_many_single(e, srcs, dsts, count, 0, 1);
}
}  // namespace

extern "C" {

int itw_set_device(int device)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) return fail("itw_set_device: no such device");
    tls.wanted_device = device;
    return 0;
}

int itw_set_devices(const int* devices, int count)
{
    tls.err.clear();
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return fail("itw_set_devices: no CUDA device"); }
    if (count < 0 || (count > 0 && !devices)) return fail("itw_set_devices: bad arguments");
    std::vector<int> list(devices, devices + count);
    for (size_t i = 0; i < list.size(); i++) {
        if (list[i] < 0 || list[i] >= n) return fail("itw_set_devices: no such device");
        for (size_t j = 0; j < i; j++) if (list[j] == list[i]) return fail("itw_set_devices: duplicate device");
    }
    std::shared_ptr<DevicePool> fresh, old;
    if (list.size() >= 2) fresh = std::make_shared<DevicePool>(list);
    {
        std::lock_guard<std::mutex> g(g_pool_mutex);
        old.swap(g_pool);
        g_pool = fresh;
        g_default_device.store(list.size() == 1 ? list[0] : -1, std::memory_order_relaxed);
    }
    old.reset();                                          // joins the previous workers (after in-flight calls released it)
    return 0;
}
int itw_get_devices(int* devices, int capacity)
{
    std::shared_ptr<DevicePool> pool = current_pool();
    if (!pool) {
        const int d = g_default_device.load(std::memory_order_relaxed);
        if (d >= 0 && devices && capacity > 0) devices[0] = d;
        return d >= 0 ? 1 : 0;
    }
    for (int i = 0; i < pool->size() && devices && i < capacity; i++) devices[i] = pool->device(i);
    return pool->size();
}

int itw_begin_deferred(void)
{
    tls.err.clear();
    if (ensure_ctx()) return -1;
    tls.deferred = true;
    tls.deferred_rc = 0;
    return 0;
}
int itw_flush(void)
{
    ThreadCtx& c = tls;
    FirstError fe{c.deferred_rc};                         // the first failure of a deferred call is the one reported
    drain_lanes(c, fe);
    c.deferred = false;
    c.deferred_rc = 0;
    return fe.rc;
}

// ---- the reference's coarse seam (3rdParty/Intel/Source/win32Threads.h:24, :52-80; win32Threads.cpp:192-330) ----
// CompressImageBC* build the profile on the stack and call CompressBlocks*, exactly like win32Threads.cpp:289-330.
// CompressImageMT / ST take the same arguments as the reference's; here BOTH hand the whole surface to the encoder in
// one call: the reference's per-thread row bands (win32Threads.cpp:217-230) exist to occupy CPU cores, while one GPU
// launch (or one band per selected device, itw_set_devices) already covers the surface -- the bytes are the same
// because bands are independent surfaces.
void CompressImageBC1(const rgba_surface* input, uint8_t* output) { CompressBlocksBC1(input, output); }
void CompressImageBC3(const rgba_surface* input, uint8_t* output) { CompressBlocksBC3(input, output); }
#define ITW_IMAGE_BC7(profile)                                                             \
    void CompressImageBC7_##profile(const rgba_surface* input, uint8_t* output)            \
    {                                                                                      \
        bc7_enc_settings settings;                                                         \
        GetProfile_##profile(&settings);                                                   \
        CompressBlocksBC7(input, output, &settings);                                       \
    }
#define ITW_IMAGE_BC6H(profile)                                                            \
    void CompressImageBC6H_##profile(const rgba_surface* input, uint8_t* output)           \
    {                                                                                      \
        bc6h_enc_settings settings;                                                        \
        GetProfile_bc6h_##profile(&settings);                                              \
        CompressBlocksBC6H(input, output, &settings);                                      \
    }
ITW_IMAGE_BC7(ultrafast) ITW_IMAGE_BC7(veryfast) ITW_IMAGE_BC7(fast) ITW_IMAGE_BC7(basic) ITW_IMAGE_BC7(slow)
ITW_IMAGE_BC7(alpha_ultrafast) ITW_IMAGE_BC7(alpha_veryfast) ITW_IMAGE_BC7(alpha_fast) ITW_IMAGE_BC7(alpha_basic) ITW_IMAGE_BC7(alpha_slow)
ITW_IMAGE_BC6H(veryfast) ITW_IMAGE_BC6H(fast) ITW_IMAGE_BC6H(basic) ITW_IMAGE_BC6H(slow) ITW_IMAGE_BC6H(veryslow)
#undef ITW_IMAGE_BC7
#undef ITW_IMAGE_BC6H

int GetBytesPerBlock(int format)                          // win32Threads.cpp:192-209: everything but BC3/BC6H/BC7 is 8
{
    switch (format) {
        case 77: case 78: case 98: case 99: case 95: case 96: return 16;
        default: return 8;
    }
}
bool CompressImageMT(const rgba_surface* input, uint8_t* output, CompressionFunc* cmpFunc, int compformat)
{
    (void)compformat;
    if (!cmpFunc) { fail("CompressImageMT: null compression function"); return false; }
    (*cmpFunc)(input, output);
    return true;                                          // like the reference (win32Threads.cpp:248, :281); errors: itw_get_last_error()
}
bool CompressImageST(const rgba_surface* input, uint8_t* output, CompressionFunc* cmpFunc, int compformat)
{
    return CompressImageMT(input, output, cmpFunc, compformat);
}
// The reference's thread-pool life cycle (win32Threads.h:52-55) mapped onto the device pool: InitWin32Threads selects
// every visible GPU, DestroyThreads returns to the single-device behaviour, GetProcessorCount reports the GPUs.
int GetProcessorCount(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    return n > 0 ? n : 1;
}
void InitWin32Threads(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); fail("InitWin32Threads: no CUDA device"); return; }
    std::vector<int> all((size_t)n);
    for (int i = 0; i < n; i++) all[i] = i;
    if (n >= 2) itw_set_devices(all.data(), n);
}
void DestroyThreads(void) { itw_set_devices(nullptr, 0); }

const char* itw_get_last_error(void) { return tls.err.c_str(); }

void itw_release(void)
{
    if (tls.stream) cudaStreamSynchronize(tls.stream);
    tls.release();
    tls.device = -1;
    tls.timed = false;
}

uint64_t itw_kernel_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

float itw_last_kernel_ms(void)
{
    float ms = -1.0f;
    if (tls.pool_ms >= 0.0f) return tls.pool_ms;
    if (tls.timed && cudaEventElapsedTime(&ms, tls.ev0, tls.ev1) != cudaSuccess) { cudaGetLastError(); ms = -1.0f; }
    return ms;
}

#if defined(ITW_BC7_PHASE_CLOCKS)
// Measurement build only (tools/bc7_phase_clocks.py): copies the per-phase cycle counters of bc7_kernel (a Bc7Clocks, `bytes`
// must be its size) to `out` after the work enqueued so far has finished, then zeroes them.
int itw_bc7_phase_clocks(void* out, size_t bytes)
{
    if (bytes != sizeof(Bc7Clocks)) return fail("itw_bc7_phase_clocks: wrong size");
    ITW_CUDA(cudaDeviceSynchronize());
    ITW_CUDA(cudaMemcpyFromSymbol(out, g_bc7_clocks, sizeof(Bc7Clocks)));
    static const Bc7Clocks zero{};
    ITW_CUDA(cudaMemcpyToSymbol(g_bc7_clocks, &zero, sizeof(Bc7Clocks)));
    return 0;
}
#endif

}  // extern "C"

#include "itw_dds.inc"
#include "itw_mips.inc"
#include "itw_shard.inc"
#include "itw_preview.inc"
#include "itw_open.inc"
#include "itw_open_raw.inc"
#include "itw_open_conv.inc"
#include "itw_open_other_bc.inc"
#include "itw_open_exp.inc"
#include "itw_open_stack.inc"
#include "itw_cube.inc"
#include "itw_none.inc"
