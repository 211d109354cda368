#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_open_converted.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

What DirectX::Convert's non-WIC _Convert (DirectXTexConvert.cpp:4321-4400) does, texel by texel with filter 0, to the uncompressed files
the plug-in's DoReadStart converts (IntelPlugin.cpp:2534-2560), and the alpha check it runs before:

  3rdParty/DirectXTex/DirectXTex/DirectXTexConvert.cpp  the LOAD_SCANLINE, LOAD_SCANLINE2 and LOAD_SCANLINE3 macros and the cases of
                                                        _LoadScanline of the loaded formats (R16G16B16A16_FLOAT / _SNORM, R16_FLOAT,
                                                        R16G16_FLOAT / _UNORM / _SNORM, R16_SNORM, R11G11B10_FLOAT, R9G9B9E5_SHAREDEXP,
                                                        R8G8_UNORM / _SNORM, R8G8B8A8_SNORM, R8_SNORM, A8_UNORM, B4G4R4A4_UNORM,
                                                        R32G32_FLOAT); _ConvertScanline, its table rows and sRGB helpers, reused
                                                        through build_ref_preview.py; the STORE_SCANLINE macro and _StoreScanline's
                                                        R16G16B16A16_UNORM case
  3rdParty/DirectXTex/DirectXTex/DirectXTexImage.cpp    the non-compressed branch of ScratchImage::IsAlphaAllOpaque (:760-793), through
                                                        build_ref_open_uncompressed.py's cut
  the scope of the path, in a second translation unit:
  3rdParty/DirectXTex/DirectXTex/DirectXTexConvert.cpp  _UseWICConversion (:4161-4266), whole
  3rdParty/DirectXTex/DirectXTex/DirectXTexUtil.cpp     WICTranslate, g_WICFormats and g_WIC2 (:21-50), _DXGIToWIC, _CheckWICColorSpace
                                                        (:84-170) and BitsPerColor (:434), whole
  3rdParty/DirectXTex/DirectXTex/DirectXTex.inl         IsSRGB and HasAlpha, whole

NOT cut, restated in the shim below, and why (each ASSUMED, DESIGN section 2):
  * DirectXMath 3.06, which is not in the tree: XMLoadHalf2 / XMLoadHalf4 (XMConvertHalfToFloat per channel, restated as
    build_ref_frontend.py does), XMLoadShortN2 / 4 (max(-1, s * (1/32767))), XMLoadByteN2 / 4 (max(-1, c * (1/127))), XMLoadUByteN2
    (b * (1/255)), XMLoadUShortN2 (u * (1/65535)), XMLoadFloat2 (a copy), XMLoadFloat3PK (the exact 6e5 / 5e5 decode with
    exponent 31 as Inf / NaN), XMLoadFloat3SE (2^(e - 24) * mantissa, the same as the hand-written loop of the < 306 branch),
    XMLoadUNibble4 (the four nibbles), and XMStoreUShortN4 as trunc(saturate(x) * 65535 + 0.5) with separate roundings, like the
    byte store build_ref_preview.py restates.  The R16_FLOAT, R16_SNORM, R8_SNORM and A8_UNORM cases are DirectXTex's own loops.
  * _StoreScanline's R8G8B8A8_UNORM and R32G32B32A32_FLOAT cases: build_ref_preview.py's restatement.
  * The WIC pixel-format GUIDs (Windows SDK): one distinct dummy GUID per name the cut bodies use, GUID_NULL zero; g_WIC2 keeps the
    reference's initial value, false (no WIC2 runtime), and the _WIN32_WINNT_WIN8 branches are compiled in.  The TEX_FILTER_* values
    are DirectXTex.h's.
  * The ScratchImage image table (item-major, mip-minor images of max(1, w >> l) x max(1, h >> l) texels, tight rows).
Only the .so is kept (git-ignored; travels to the GPU box).  Used by tests/test_dds_open_converted.py and its GPU twin.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_preview as P             # _ConvertScanline, its table and sRGB helpers, the preview shim and its two targets
import build_ref_open_uncompressed as U   # the non-compressed branch of IsAlphaAllOpaque

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_SO = os.path.join(P.OUT_DIR, "libitw_ref_open_converted.so")
IMAGE_CPP = os.path.join(P.DXTEX, "DirectXTexImage.cpp")
UTIL_CPP = os.path.join(P.DXTEX, "DirectXTexUtil.cpp")
TEX_INL = os.path.join(P.DXTEX, "DirectXTex.inl")

# loaded format -> (DXGI id, bytes per texel)
LOADED = {"R16G16B16A16_FLOAT": (10, 8), "R16_FLOAT": (54, 2), "R16G16_FLOAT": (34, 4), "R16G16B16A16_SNORM": (13, 8),
          "R16G16_UNORM": (35, 4), "R16G16_SNORM": (37, 4), "R16_SNORM": (58, 2), "R11G11B10_FLOAT": (26, 4),
          "R9G9B9E5_SHAREDEXP": (67, 4), "R8G8_UNORM": (49, 2), "R8G8_SNORM": (51, 2), "R8G8B8A8_SNORM": (31, 4), "R8_SNORM": (63, 1),
          "A8_UNORM": (65, 1), "B4G4R4A4_UNORM": (115, 2), "R32G32_FLOAT": (16, 8)}
FORMATS = dict(P.FORMATS, R16G16B16A16_UNORM=11, **{k: v[0] for k, v in LOADED.items()})

SHIM_LOAD = r"""
#undef D3DXDecodeBC2
#undef D3DXDecodeBC4S
#undef D3DXDecodeBC5S
#define DIRECTX_MATH_VERSION 306
typedef const void* LPCVOID;
typedef void* LPVOID;
#define __restrict
static inline XMVECTOR XMVectorSet(float x, float y, float z, float w) { return XMVECTOR{{x, y, z, w}}; }
static const XMVECTORF32 g_XMIdentityR3 = {{0.0f, 0.0f, 0.0f, 1.0f}};
// ---- DirectXMath 3.06, restated (ASSUMED: see the recipe's header) ----
typedef uint16_t HALF;
static inline float XMConvertHalfToFloat(HALF Value)
{
    uint32_t Mantissa = (uint32_t)(Value & 0x03FF), Exponent = (Value & 0x7C00);
    if (Exponent == 0x7C00) Exponent = 0x1F;                                     // INF / NAN: an ordinary binade in 3.06
    else if (Exponent != 0) Exponent = (uint32_t)((Value >> 10) & 0x1F);
    else if (Mantissa != 0) {
        Exponent = 1;
        do { Exponent--; Mantissa <<= 1; } while ((Mantissa & 0x0400) == 0);
        Mantissa &= 0x03FF;
    } else Exponent = (uint32_t)-112;
    uint32_t Result = ((Value & 0x8000) << 16) | ((Exponent + 112) << 23) | (Mantissa << 13);
    float f; memcpy(&f, &Result, 4); return f;
}
struct XMHALF4 { HALF x, y, z, w; };
struct XMHALF2 { HALF x, y; };
struct XMSHORTN4 { int16_t x, y, z, w; };
struct XMSHORTN2 { int16_t x, y; };
struct XMUSHORTN2 { uint16_t x, y; };
struct XMUSHORTN4 { uint16_t x, y, z, w; };
struct XMBYTEN4 { int8_t x, y, z, w; };
struct XMBYTEN2 { int8_t x, y; };
struct XMUBYTEN2 { uint8_t x, y; };
struct XMFLOAT2 { float x, y; };
struct XMFLOAT3PK { uint32_t v; };
struct XMFLOAT3SE { uint32_t v; };
struct XMUNIBBLE4 { uint16_t v; };
static inline float snorm16(int16_t s) { float v = (float)s * (1.0f / 32767.0f); return v > -1.0f ? v : -1.0f; }
static inline float snorm8(int8_t c) { float v = (float)c * (1.0f / 127.0f); return v > -1.0f ? v : -1.0f; }
static inline XMVECTOR XMLoadHalf4(const XMHALF4* p) { return XMVECTOR{{XMConvertHalfToFloat(p->x), XMConvertHalfToFloat(p->y), XMConvertHalfToFloat(p->z), XMConvertHalfToFloat(p->w)}}; }
static inline XMVECTOR XMLoadHalf2(const XMHALF2* p) { return XMVECTOR{{XMConvertHalfToFloat(p->x), XMConvertHalfToFloat(p->y), 0.0f, 0.0f}}; }
static inline XMVECTOR XMLoadShortN4(const XMSHORTN4* p) { return XMVECTOR{{snorm16(p->x), snorm16(p->y), snorm16(p->z), snorm16(p->w)}}; }
static inline XMVECTOR XMLoadShortN2(const XMSHORTN2* p) { return XMVECTOR{{snorm16(p->x), snorm16(p->y), 0.0f, 0.0f}}; }
static inline XMVECTOR XMLoadByteN4(const XMBYTEN4* p) { return XMVECTOR{{snorm8(p->x), snorm8(p->y), snorm8(p->z), snorm8(p->w)}}; }
static inline XMVECTOR XMLoadByteN2(const XMBYTEN2* p) { return XMVECTOR{{snorm8(p->x), snorm8(p->y), 0.0f, 0.0f}}; }
static inline XMVECTOR XMLoadUByteN2(const XMUBYTEN2* p) { return XMVECTOR{{p->x * (1.0f / 255.0f), p->y * (1.0f / 255.0f), 0.0f, 0.0f}}; }
static inline XMVECTOR XMLoadUShortN2(const XMUSHORTN2* p) { return XMVECTOR{{p->x * (1.0f / 65535.0f), p->y * (1.0f / 65535.0f), 0.0f, 0.0f}}; }
static inline XMVECTOR XMLoadFloat2(const XMFLOAT2* p) { XMVECTOR r{{0.0f, 0.0f, 0.0f, 0.0f}}; memcpy(r.f, p, 8); return r; }
static inline uint32_t pk_channel(uint32_t Mantissa, uint32_t Exponent, int bits)
{
    if (Exponent == 0x1f) return 0x7f800000 | (Mantissa << (23 - bits));
    if (Exponent == 0) {
        if (Mantissa != 0) {
            Exponent = 1;
            do { Exponent--; Mantissa <<= 1; } while ((Mantissa & (1u << bits)) == 0);
            Mantissa &= (1u << bits) - 1;
        } else Exponent = (uint32_t)-112;
    }
    return ((Exponent + 112) << 23) | (Mantissa << (23 - bits));
}
static inline XMVECTOR XMLoadFloat3PK(const XMFLOAT3PK* p)
{
    const uint32_t v = p->v, r[3] = {pk_channel(v & 63, (v >> 6) & 31, 6), pk_channel((v >> 11) & 63, (v >> 17) & 31, 6),
                                     pk_channel((v >> 22) & 31, v >> 27, 5)};
    XMVECTOR o{{0.0f, 0.0f, 0.0f, 0.0f}};
    memcpy(o.f, r, 12);
    return o;
}
static inline XMVECTOR XMLoadFloat3SE(const XMFLOAT3SE* p)
{
    union { float f; int32_t i; } fi;
    fi.i = 0x33800000 + ((p->v >> 27) << 23);
    const float Scale = fi.f;
    return XMVECTOR{{Scale * float(p->v & 0x1FF), Scale * float((p->v >> 9) & 0x1FF), Scale * float((p->v >> 18) & 0x1FF), 1.0f}};
}
static inline XMVECTOR XMLoadUNibble4(const XMUNIBBLE4* p)
{
    return XMVECTOR{{float(p->v & 0xF), float((p->v >> 4) & 0xF), float((p->v >> 8) & 0xF), float((p->v >> 12) & 0xF)}};
}
static inline void XMStoreUShortN4(XMUSHORTN4* d, XMVECTOR v)
{
    uint16_t* o = &d->x;
    for (int c = 0; c < 4; c++) {
        float x = v.f[c];
        x = (x > 0.0f) ? x : 0.0f;
        x = (x < 1.0f) ? x : 1.0f;
        o[c] = (uint16_t)(int)(x * 65535.0f + 0.5f);
    }
}
"""

LOAD = r"""
// _LoadScanline: the reference's macros and the cases of the loaded formats, cut; every other format aborts
static bool _LoadScanline(XMVECTOR* pDestination, size_t count, LPCVOID pSource, size_t size, DXGI_FORMAT format)
{
    XMVECTOR* __restrict dPtr = pDestination;
    const XMVECTOR* ePtr = pDestination + count;
    switch (static_cast<int>(format)) {
@CASES@
    default:
        abort();
    }
}
// _StoreScanline's R16G16B16A16_UNORM case, cut; the other two targets are build_ref_preview.py's
static bool store_target(void* pDestination, size_t size, DXGI_FORMAT format, const XMVECTOR* pSource, size_t count)
{
    const XMVECTOR* __restrict sPtr = pSource;
    const XMVECTOR* ePtr = pSource + count;
    switch (static_cast<int>(format)) {
    @STORE16@
    default:
        return _StoreScanline(pDestination, size, format, pSource, count);
    }
}
"""

BOTTOM = r"""
struct AlignedFree { void operator()(XMVECTOR* p) const { free(p); } };
typedef std::unique_ptr<XMVECTOR[], AlignedFree> ScopedAlignedArrayXMVECTOR;
static void* _aligned_malloc(size_t n, size_t a) { return aligned_alloc(a, (n + a - 1) / a * a); }
static inline bool XMVector4Less(XMVECTOR a, const XMVECTORF32& b)
{
    return a.f[0] < b.f[0] && a.f[1] < b.f[1] && a.f[2] < b.f[2] && a.f[3] < b.f[3];
}
static size_t texel_bytes(DXGI_FORMAT f)
{
    switch ((int)f) {
@BYTES@
    default: abort();
    }
}
static bool IsAlphaAllOpaque(DXGI_FORMAT format, const uint8_t* payload, size_t w, size_t h, size_t mips, size_t items)
{
    std::vector<Image> _image;
    for (size_t item = 0; item < items; item++)
        for (size_t l = 0; l < mips; l++) {
            const size_t lw = std::max<size_t>(1, w >> l), lh = std::max<size_t>(1, h >> l), pitch = lw * texel_bytes(format);
            _image.push_back(Image{lw, lh, format, pitch, pitch * lh, const_cast<uint8_t*>(payload)});
            payload += pitch * lh;
        }
    const size_t _nimages = _image.size();
    struct { size_t width; } _metadata{w};
@BRANCH@
    return true;
}
}  // namespace itw_ref_preview
using namespace itw_ref_preview;

// _Convert of `n` texels with filter 0: _LoadScanline(loaded), _ConvertScanline(target, loaded, 0), _StoreScanline(target)
extern "C" int ref_convert_texels(uint32_t loaded, uint32_t target, const uint8_t* src, long long n, uint8_t* dst)
{
    ScopedAlignedArrayXMVECTOR buf(reinterpret_cast<XMVECTOR*>(_aligned_malloc(sizeof(XMVECTOR) * n, 16)));
    if (!_LoadScanline(buf.get(), n, src, n * texel_bytes((DXGI_FORMAT)loaded), (DXGI_FORMAT)loaded)) return -1;
    _ConvertScanline(buf.get(), n, (DXGI_FORMAT)target, (DXGI_FORMAT)loaded, 0);
    const size_t out = target == 2 ? 16 : target == 11 ? 8 : 4;
    return store_target(dst, n * out, (DXGI_FORMAT)target, buf.get(), n) ? 0 : -1;
}
// 1 if every texel of every image of the loaded payload is opaque
extern "C" int ref_is_alpha_all_opaque(uint32_t format, const uint8_t* loaded, uint32_t w, uint32_t h, uint32_t mips, uint32_t items)
{
    return IsAlphaAllOpaque((DXGI_FORMAT)format, loaded, w, h, mips, items) ? 1 : 0;
}
// the branch on `n` one-texel images: out[i] = 1 if texel i is opaque
extern "C" void ref_texels_opaque(uint32_t format, const uint8_t* texels, long long n, uint8_t* out)
{
    const size_t b = texel_bytes((DXGI_FORMAT)format);
    for (long long i = 0; i < n; i++) out[i] = IsAlphaAllOpaque((DXGI_FORMAT)format, texels + i * b, 1, 1, 1, 1) ? 1 : 0;
}
"""


WIC_UNIT = r"""
// generated by oracle/build_ref_open_converted.py -- the scope of the converted open path: _UseWICConversion and what it reads
#include <cstddef>
#include <cstdint>
#include <cstring>
#define _In_
#define _Out_
#define _Use_decl_annotations_
#define __cdecl
#define _countof(a) (sizeof(a) / sizeof((a)[0]))
#define _WIN32_WINNT_WIN8 0x0602
#define _WIN32_WINNT 0x0602
typedef unsigned long DWORD;
namespace itw_ref_open_conv_scope {
enum DXGI_FORMAT { @DXGI@ };
struct GUID { uint32_t Data1; uint16_t Data2, Data3; uint8_t Data4[8]; };
typedef GUID WICPixelFormatGUID;
static const GUID GUID_NULL = {0, 0, 0, {0, 0, 0, 0, 0, 0, 0, 0}};
@GUIDS@
enum TEX_FILTER_FLAGS : DWORD { @FILTERS@ };
bool _DXGIToWIC(DXGI_FORMAT format, GUID& guid, bool ignoreRGBvsBGR = false);      // DirectXTexP.h's declaration
@BODIES@
}  // namespace itw_ref_open_conv_scope
using namespace itw_ref_open_conv_scope;
extern "C" int ref_use_wic(uint32_t source, uint32_t target)
{
    WICPixelFormatGUID a, b;
    return _UseWICConversion(0, (DXGI_FORMAT)source, (DXGI_FORMAT)target, a, b) ? 1 : 0;
}
extern "C" unsigned ref_bits_per_color(uint32_t f) { return (unsigned)BitsPerColor((DXGI_FORMAT)f); }
extern "C" int ref_is_srgb(uint32_t f) { return IsSRGB((DXGI_FORMAT)f) ? 1 : 0; }
extern "C" int ref_has_alpha(uint32_t f) { return HasAlpha((DXGI_FORMAT)f) ? 1 : 0; }
"""


def wic_unit(conv, util, inl, tex_h):
    """The second translation unit: _UseWICConversion, _DXGIToWIC, _CheckWICColorSpace, g_WICFormats, BitsPerColor, IsSRGB, HasAlpha."""
    table = U.cut_between(util, r"^struct WICTranslate", "};") + "\n" + U.cut_between(util, r"^static WICTranslate g_WICFormats\[\]", "};")
    wic2 = re.search(r"^static bool g_WIC2 = false;", util, re.M)
    if not wic2:
        raise RuntimeError("g_WIC2 not found")
    bodies = [table, wic2.group(0),
              P.cut_named(util, r"^bool _DXGIToWIC\s*\("),
              P.cut_named(util, r"^DWORD _CheckWICColorSpace\s*\("),
              P.cut_named(util, r"^size_t BitsPerColor\s*\("),
              P.cut_named(inl, r"^inline bool __cdecl IsSRGB\s*\("),
              P.cut_named(inl, r"^inline bool __cdecl HasAlpha\s*\("),
              P.cut_named(conv, r"^static inline bool _UseWICConversion\s*\(")]
    text = "\n".join(bodies)
    guids = sorted(set(re.findall(r"GUID_WICPixelFormat\w+", text)))
    filters = re.findall(r"^\s*(TEX_FILTER_\w+)\s*=\s*(0x[0-9A-Fa-f]+)", tex_h, re.M)
    if not guids or not filters:
        raise RuntimeError("WIC GUID names or TEX_FILTER values not found")
    dxgi = list(U.D.DXGI) + [f"XBOX_{i}" for i in range(len(U.D.DXGI), 121)]
    return (WIC_UNIT.replace("@DXGI@", ", ".join(f"DXGI_FORMAT_{n} = {i}" for i, n in enumerate(dxgi)))
            .replace("@GUIDS@", "\n".join(f"static const GUID {g} = {{{i + 1}u, 0, 0, {{0, 0, 0, 0, 0, 0, 0, 0}}}};"
                                            for i, g in enumerate(guids)))
            .replace("@FILTERS@", ", ".join(f"{n} = {v}" for n, v in filters))
            .replace("@BODIES@", text.replace("_Use_decl_annotations_", "")))


def cut_load_cases(conv):
    body = P.cut_function(conv, conv.index("bool _LoadScanline("))
    out = []
    for name in LOADED:
        m = re.search(r"case DXGI_FORMAT_" + name + r":\s*(?:LOAD_SCANLINE\d?\([^)]*\)|if \( size >=.*?\n        return false;|#if.*?#endif)",
                      body, re.S)
        if not m:
            raise RuntimeError(name + " not found in _LoadScanline")
        out.append(m.group(0))
    macros = "".join(U.cut_between(conv, r"^#define " + mac + r"\( type, func(?:, defvec)? \)", "return false;\n")
                     for mac in ("LOAD_SCANLINE", "LOAD_SCANLINE3", "LOAD_SCANLINE2"))
    return macros + LOAD.replace("@CASES@", "\n".join("    " + c for c in out))


def cut_store16(conv):
    m = re.search(r"case DXGI_FORMAT_R16G16B16A16_UNORM:\s*STORE_SCANLINE\( XMUSHORTN4, XMStoreUShortN4 \)", P.cut_function(
        conv, conv.index("bool _StoreScanline(")))
    if not m:
        raise RuntimeError("_StoreScanline's R16G16B16A16_UNORM case not found")
    return U.cut_between(conv, r"^#define STORE_SCANLINE\( type, func \)", "return false;\n"), m.group(0)


def cut_table(conv):
    a = conv.index("static const ConvertData g_ConvertTable[]")
    body = conv[conv.index("{", a) + 1:conv.index("};", a)]
    rows = []
    for ln in body.splitlines():
        m = re.match(r"\s*\{ DXGI_FORMAT_(\w+),", ln)
        if m and m.group(1) in FORMATS:
            rows.append("    " + ln.strip())
    return "\n".join(rows)


def build(verbose=True):
    have_ref = os.path.exists(P.CONVERT_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {P.REF_ROOT} and no prebuilt {OUT_SO}")
    deps = [os.path.join(P.OUT_DIR, n) for n in ("libitw_ref_frontend.so", "libitw_ref_decode.so")]
    for d in deps:
        if not os.path.exists(d):
            raise FileNotFoundError(f"{d} is built by build_ref_frontend.py / build_ref_decode.py first")
    srcs = [__file__, P.__file__, U.__file__, P.CONVERT_CPP, IMAGE_CPP, UTIL_CPP, TEX_INL] + deps
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in srcs):
        return OUT_SO
    tmp = tempfile.mkdtemp(prefix="itw_ref_open_conv_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        conv = read(P.CONVERT_CPP)
        macro16, case16 = cut_store16(conv)
        top = (P.SHIM_TOP.replace("@FORMATS@", ", ".join(f"DXGI_FORMAT_{n} = {v}" for n, v in FORMATS.items()))
               .replace("@ENUMS@", P.cut_enums(read(P.TEXP_H), read(P.TEX_H)))
               .replace("@TABLE@", cut_table(conv))
               .replace("@SRGB@", P.cut_grayscale(conv) + P.cut_srgb(conv))
               .replace("@CONVERT_BODY@", P.cut_convert_body(conv))
               .replace("#include <cstring>", "#include <cstring>\n#include <memory>\n#include <vector>"))
        bytes_cases = "\n".join(f"    case {v[0]}: return {v[1]};" for v in LOADED.values())
        unit = (top + SHIM_LOAD + cut_load_cases(conv).replace("@STORE16@", case16).replace("static bool store_target", macro16 +
                "static bool store_target")
                + BOTTOM.replace("@BYTES@", bytes_cases).replace("@BRANCH@", U.cut_alpha_branch(read(IMAGE_CPP))))
        path = os.path.join(tmp, "open_conv_ref.cpp")
        open(path, "w").write(unit)
        scope = os.path.join(tmp, "open_conv_scope_ref.cpp")
        open(scope, "w").write(wic_unit(conv, read(UTIL_CPP), read(TEX_INL), read(P.TEX_H)))
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-fno-fast-math", "-mfpmath=sse", "-msse2",
               path, scope, "-o", OUT_SO, "-L" + P.OUT_DIR] + ["-l:" + os.path.basename(d) for d in deps] + ["-Wl,-rpath,$ORIGIN"]
        if verbose:
            print("[build_ref_open_converted]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_open_converted] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
