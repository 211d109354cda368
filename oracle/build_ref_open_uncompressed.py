#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_open_uncompressed.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

What the plug-in's open path (IntelPlugin.cpp:2419-2742) does with an uncompressed DDS file that needs no conversion:

  3rdParty/DirectXTex/DirectXTex/DirectXTexDDS.cpp      CONVERSION_FLAGS, LegacyDDS and g_LegacyDDSMap (:26-131), _GetDXGIFormat
                                                        (:144-197), _DecodeDDSHeader (:199-437), TEXP_LEGACY_FORMAT / _FindLegacyFormat
                                                        and _LegacyExpandScanline (:682-1018), whole
  3rdParty/DirectXTex/DirectXTex/DirectXTexConvert.cpp  _CopyScanline (:189-420), whole; the LOAD_SCANLINE macro and the four cases of
                                                        _LoadScanline these files reach (R32G32B32A32_FLOAT, R16G16B16A16_UNORM,
                                                        R8G8B8A8_UNORM / _SRGB)
  3rdParty/DirectXTex/DirectXTex/DirectXTexImage.cpp    the non-compressed branch of ScratchImage::IsAlphaAllOpaque (:760-793)
  3rdParty/DirectXTex/DirectXTex/DDS.h                  the header structures, DDSPF_* and the flag constants
  3rdParty/DirectXTex/DirectXTex/DirectXTexP.h          TEXP_SCANLINE_FLAGS
  IntelCompressionPlugin/IntelPlugin.h                  F32toF16 and ConvertTo16Bit(unsigned8) (:36-39, :77-80)

NOT cut, restated in the shim below, and why:
  * _CopyImage's row loop (DirectXTexDDS.cpp:1024-1130): its choice between the three row paths these files take (a plain
    _CopyScanline, _CopyScanline with TEXP_SCANLINE_SETALPHA from CONV_FLAGS_NOALPHA, _LegacyExpandScanline for CONV_FLAGS_EXPAND) and
    its pitches (ComputePitch: 3 w bytes with CP_FLAGS_24BPP, else bits-per-pixel w / 8) are restated for these formats; the
    ScratchImage image table (item-major, mip-minor images of max(1, w >> l) x max(1, h >> l) texels) likewise.
  * DirectXMath, which is not in the tree: XMLoadUByteN4 = byte * (1/255), XMLoadUShortN4 = v * (1/65535), XMVectorSplatW /
    XMVector4Less as scalar compares, and XMConvertFloatToHalf as restated by build_ref_frontend.py (DirectXMath 3.06).
  * IsValid / IsPalettized (DirectXTex.inl) and the DXGI_FORMAT numbering (dxgiformat.h).
Only the .so is kept (git-ignored; travels to the GPU box).  Used by tests/test_dds_open_uncompressed.py and its GPU twin.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_dds as D                # the DXGI numbering, the SHIM_TOP of the header cut, cut_function

HERE = os.path.dirname(os.path.abspath(__file__))
DXTEX = os.path.dirname(D.DDS_CPP)
CONVERT_CPP = os.path.join(DXTEX, "DirectXTexConvert.cpp")
IMAGE_CPP = os.path.join(DXTEX, "DirectXTexImage.cpp")
TEXP_H = os.path.join(DXTEX, "DirectXTexP.h")
PLUGIN_H = os.path.join(D.REF_ROOT, "IntelCompressionPlugin", "IntelPlugin.h")
OUT_SO = os.path.join(D.OUT_DIR, "libitw_ref_open_uncompressed.so")

SHIM_MID = r"""
#undef extern
#undef __declspec
using namespace DirectX;
typedef const void* LPCVOID;
#define _In_reads_bytes_(x)
#define _In_reads_opt_(x)
#define _Out_writes_bytes_(x)
#define _Inout_updates_bytes_(x)
#define _When_(a, b)
#define _Out_
#define _Inout_
#define _In_
#define _Success_(x)
#define _Use_decl_annotations_
#define ERROR_INVALID_DATA 13L
// DirectXTex.h: the fields and constants the cut bodies touch
enum TEX_DIMENSION { TEX_DIMENSION_TEXTURE1D = 2, TEX_DIMENSION_TEXTURE2D = 3, TEX_DIMENSION_TEXTURE3D = 4 };
enum { TEX_MISC_TEXTURECUBE = 0x4 };
enum { TEX_MISC2_ALPHA_MODE_MASK = 0x7 };
enum { TEX_ALPHA_MODE_UNKNOWN = 0, TEX_ALPHA_MODE_STRAIGHT = 1, TEX_ALPHA_MODE_PREMULTIPLIED = 2, TEX_ALPHA_MODE_OPAQUE = 3, TEX_ALPHA_MODE_CUSTOM = 4 };
enum { DDS_FLAGS_NONE = 0, DDS_FLAGS_LEGACY_DWORD = 0x1, DDS_FLAGS_NO_LEGACY_EXPANSION = 0x2, DDS_FLAGS_NO_R10B10G10A2_FIXUP = 0x4,
       DDS_FLAGS_FORCE_RGB = 0x8, DDS_FLAGS_NO_16BPP = 0x10, DDS_FLAGS_EXPAND_LUMINANCE = 0x20 };
struct TexMetadata {
    size_t width, height, depth, arraySize, mipLevels;
    uint32_t miscFlags, miscFlags2;
    DXGI_FORMAT format;
    TEX_DIMENSION dimension;
};
// DirectXTex.inl
static bool IsValid(DXGI_FORMAT f) { return (size_t)f >= 1 && (size_t)f <= 120; }
static bool IsPalettized(DXGI_FORMAT f) { return f == DXGI_FORMAT_AI44 || f == DXGI_FORMAT_IA44 || f == DXGI_FORMAT_P8 || f == DXGI_FORMAT_A8P8; }
static bool IsPlanar(DXGI_FORMAT) { return false; }
static bool IsTypeless(DXGI_FORMAT, bool) { return false; }
static bool IsCompressed(DXGI_FORMAT) { return false; }
// DirectXMath, scalar
struct XMVECTOR { float f[4]; };
struct XMVECTORF32 { float f[4]; };
struct XMUBYTEN4 { uint8_t x, y, z, w; };
struct XMUSHORTN4 { uint16_t x, y, z, w; };
static inline XMVECTOR XMLoadUByteN4(const XMUBYTEN4* p)
{
    return XMVECTOR{{p->x * (1.0f / 255.0f), p->y * (1.0f / 255.0f), p->z * (1.0f / 255.0f), p->w * (1.0f / 255.0f)}};
}
static inline XMVECTOR XMLoadUShortN4(const XMUSHORTN4* p)
{
    return XMVECTOR{{p->x * (1.0f / 65535.0f), p->y * (1.0f / 65535.0f), p->z * (1.0f / 65535.0f), p->w * (1.0f / 65535.0f)}};
}
static inline XMVECTOR XMVectorSplatW(XMVECTOR v) { return XMVECTOR{{v.f[3], v.f[3], v.f[3], v.f[3]}}; }
static inline bool XMVector4Less(XMVECTOR a, const XMVECTORF32& b)
{
    return a.f[0] < b.f[0] && a.f[1] < b.f[1] && a.f[2] < b.f[2] && a.f[3] < b.f[3];
}
"""

LOAD_SCANLINE = r"""
// _LoadScanline: the reference's macro and the four cases these files reach, cut; every other format aborts
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
"""

SHIM_BOTTOM = r"""
// ScratchImage::IsAlphaAllOpaque for an uncompressed texture: the image table restated, the non-compressed branch cut
struct Image { size_t width, height; DXGI_FORMAT format; size_t rowPitch, slicePitch; uint8_t* pixels; };
struct AlignedFree { void operator()(XMVECTOR* p) const { free(p); } };
typedef std::unique_ptr<XMVECTOR[], AlignedFree> ScopedAlignedArrayXMVECTOR;
static void* _aligned_malloc(size_t n, size_t a) { return aligned_alloc(a, (n + a - 1) / a * a); }
static size_t texel_bytes(DXGI_FORMAT f) { return f == DXGI_FORMAT_R32G32B32A32_FLOAT ? 16 : f == DXGI_FORMAT_R16G16B16A16_UNORM ? 8 : 4; }
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
}  // namespace itw_ref_open_raw

using namespace itw_ref_open_raw;

// _DecodeDDSHeader with DDS_FLAGS_NONE.  out: width, height, mipLevels, arraySize, format, cube (0/1), convFlags, dimension, payload
// offset (LoadFromDDSMemory's: 128, + 20 with CONV_FLAGS_DX10).  Returns the HRESULT (0 = S_OK).
extern "C" long ref_decode_header(const uint8_t* file, size_t size, uint64_t* out)
{
    TexMetadata m;
    DWORD conv = 0;
    const HRESULT hr = _DecodeDDSHeader(file, size, DDS_FLAGS_NONE, m, conv);
    if (hr != S_OK) return hr;
    out[0] = m.width; out[1] = m.height; out[2] = m.mipLevels; out[3] = m.arraySize; out[4] = (uint64_t)m.format;
    out[5] = (m.miscFlags & TEX_MISC_TEXTURECUBE) ? 1 : 0; out[6] = conv; out[7] = (uint64_t)m.dimension;
    out[8] = 4 + sizeof(DDS_HEADER) + ((conv & CONV_FLAGS_DX10) ? sizeof(DDS_HEADER_DXT10) : 0);
    return 0;
}
// LoadFromDDSMemory's _CopyImage for these files: every image of the payload at `src` (item-major, mip-minor, source pitches) into
// `dst` as the loaded format (tight rows), through the row path _CopyImage picks.  Returns the bytes written, -1 on a failed row.
extern "C" long long ref_copy_image(const uint8_t* src, uint32_t w, uint32_t h, uint32_t mips, uint32_t items, uint32_t format,
                                    uint32_t conv, uint8_t* dst)
{
    const DXGI_FORMAT f = (DXGI_FORMAT)format;
    const DWORD tflags = (conv & CONV_FLAGS_NOALPHA) ? TEXP_SCANLINE_SETALPHA : 0;
    const size_t bpp = (conv & CONV_FLAGS_EXPAND) && (conv & CONV_FLAGS_888) ? 24 : texel_bytes(f) * 8;   // ComputePitch's bits
    uint8_t* d0 = dst;
    for (uint32_t item = 0; item < items; item++)
        for (uint32_t l = 0; l < mips; l++) {
            const size_t lw = std::max<size_t>(1, w >> l), lh = std::max<size_t>(1, h >> l);
            const size_t spitch = (lw * bpp + 7) / 8, dpitch = lw * texel_bytes(f);
            for (size_t y = 0; y < lh; y++) {
                if (conv & CONV_FLAGS_EXPAND) {
                    if (!_LegacyExpandScanline(dst, dpitch, f, src, spitch, _FindLegacyFormat(conv), nullptr, tflags)) return -1;
                } else {
                    _CopyScanline(dst, dpitch, src, spitch, f, tflags);
                }
                src += spitch;
                dst += dpitch;
            }
        }
    return (long long)(dst - d0);
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
// the plug-in's forced white of a 16-bit cube face plane: ConvertTo16Bit(static_cast<unsigned8>(255))
extern "C" unsigned ref_convert_to_16bit_255() { return ConvertTo16Bit(static_cast<unsigned8>(255)); }
"""

HALF = r"""
namespace DirectX { namespace PackedVector {
// DirectXMath 3.06 XMConvertFloatToHalf, as build_ref_frontend.py restates it
inline unsigned short XMConvertFloatToHalf(float Value)
{
    uint32_t Result, IValue; memcpy(&IValue, &Value, 4);
    uint32_t Sign = (IValue & 0x80000000U) >> 16U;
    IValue = IValue & 0x7FFFFFFFU;
    if (IValue > 0x47FFEFFFU) Result = 0x7FFFU;
    else {
        if (IValue < 0x38800000U) {
            uint32_t Shift = 113U - (IValue >> 23U);
            IValue = (Shift < 32U) ? ((0x800000U | (IValue & 0x7FFFFFU)) >> Shift) : 0U;
        } else IValue += 0xC8000000U;
        Result = ((IValue + 0x0FFFU + ((IValue >> 13U) & 1U)) >> 13U) & 0x7FFFU;
    }
    return (unsigned short)(Result | Sign);
}
}  }
typedef uint8_t unsigned8;
typedef uint16_t unsigned16;
"""


def cut_between(src, start_pat, end_text):
    m = re.search(start_pat, src, re.M)
    if not m:
        raise RuntimeError(start_pat + " not found in the reference")
    return src[m.start():src.index(end_text, m.start()) + len(end_text)]


def cut_load_cases(conv):
    body = D.cut_function(conv, conv.index("bool _LoadScanline("))
    out = []
    m = re.search(r"case DXGI_FORMAT_R32G32B32A32_FLOAT:.*?return true;", body, re.S)
    out.append(m.group(0))
    for pat in (r"case DXGI_FORMAT_R16G16B16A16_UNORM:\s*LOAD_SCANLINE\( XMUSHORTN4, XMLoadUShortN4 \)",
                r"case DXGI_FORMAT_R8G8B8A8_UNORM:\s*case DXGI_FORMAT_R8G8B8A8_UNORM_SRGB:\s*LOAD_SCANLINE\( XMUBYTEN4, XMLoadUByteN4 \)"):
        m = re.search(pat, body)
        if not m:
            raise RuntimeError(pat + " not found in _LoadScanline")
        out.append(m.group(0))
    macro = cut_between(conv, r"^#define LOAD_SCANLINE\( type, func \)", "return false;\n")
    return macro + LOAD_SCANLINE.replace("@CASES@", "\n".join("    " + c for c in out))


def cut_alpha_branch(image_cpp):
    body = D.cut_function(image_cpp, re.search(r"^bool ScratchImage::IsAlphaAllOpaque\s*\(", image_cpp, re.M).start())
    m = re.search(r"if\s*\(\s*IsCompressed\(\s*_metadata\.format\s*\)\s*\)", body)
    compressed = D.cut_function(body, m.start())
    rest = body[m.start() + len(compressed):]
    e = re.match(r"\s*else\s*", rest)
    if not e:
        raise RuntimeError("non-compressed branch of IsAlphaAllOpaque not found")
    return D.cut_function(rest, e.end())


def build(verbose=True):
    have_ref = os.path.exists(D.DDS_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {D.REF_ROOT} and no prebuilt {OUT_SO}")
    srcs = [__file__, D.__file__, D.DDS_CPP, D.DDS_H, CONVERT_CPP, IMAGE_CPP, TEXP_H, PLUGIN_H]
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in srcs):
        return OUT_SO
    os.makedirs(D.OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_open_raw_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        dds, conv, image, texp, plugin = (read(p) for p in (D.DDS_CPP, CONVERT_CPP, IMAGE_CPP, TEXP_H, PLUGIN_H))
        hdr = read(D.DDS_H)
        dds_h = hdr[hdr.index("namespace DirectX"):hdr.rindex("}; // namespace")] + "}  // namespace DirectX\n"
        enum = ",\n".join(f"    DXGI_FORMAT_{name} = {i}" for i, name in enumerate(D.DXGI))
        top = D.SHIM_TOP.replace("@DXGI@", enum).replace("#include <cstring>", "#include <cstring>\n#include <cstdlib>\n#include <algorithm>\n"
                                                                                      "#include <memory>\n#include <vector>")
        parts = [
            top, dds_h, SHIM_MID,
            cut_between(texp, r"^\s*enum TEXP_SCANLINE_FLAGS", "};"),
            "\nnamespace itw_ref_open_raw {\n",
            cut_between(dds, r"^enum CONVERSION_FLAGS", "};"),
            cut_between(dds, r"^struct LegacyDDS", "};"),
            cut_between(dds, r"^const LegacyDDS g_LegacyDDSMap\[\]", "\n};"),
            D.cut_function(dds, re.search(r"^static DXGI_FORMAT _GetDXGIFormat\s*\(", dds, re.M).start()),
            D.cut_function(dds, re.search(r"^static HRESULT _DecodeDDSHeader\s*\(", dds, re.M).start()),
            cut_between(dds, r"^enum TEXP_LEGACY_FORMAT", "};"),
            D.cut_function(dds, re.search(r"^inline static TEXP_LEGACY_FORMAT _FindLegacyFormat\s*\(", dds, re.M).start()),
            D.cut_function(dds, re.search(r"^static bool _LegacyExpandScanline\s*\(", dds, re.M).start()),
            D.cut_function(conv, re.search(r"^void _CopyScanline\s*\(", conv, re.M).start()),
            cut_load_cases(conv),
            HALF,
            D.cut_function(plugin, re.search(r"^inline unsigned short F32toF16\s*\(", plugin, re.M).start()),
            D.cut_function(plugin, re.search(r"^inline unsigned16 ConvertTo16Bit\(unsigned8 val\)", plugin, re.M).start()),
            SHIM_BOTTOM.replace("@BRANCH@", cut_alpha_branch(image)),
        ]
        unit = "\n".join(parts).replace("_Success_(return != false)", "")
        path = os.path.join(tmp, "open_raw_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-fno-fast-math", "-mfpmath=sse", "-msse2",
               path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_open_uncompressed]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_open_uncompressed] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
