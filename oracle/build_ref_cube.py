#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_cube.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

The two cube texture types of the save dialog place texels with these bodies, cut WHERE THEY LIE (never copied into the repo):

  IntelCompressionPlugin/IntelPlugin.cpp   IsCubeMapWithSetMipLevelOverride (:1172-1179), ConvertToCubeMapFromCross (:1200-1265),
                                           ConvertToCubeMapFromLayers (:1270-1416), ConvertToHorizontalCrossFromCubeMap (:1421-1501),
                                           and the layer helpers they call, FillLayerDataToWhite (:1664-1689) and
                                           CopyFromLayerChannelIntoImage (:1694-1741)
  IntelCompressionPlugin/IntelPlugin.h     enum TextureTypeEnum and the conversion helpers (build_ref_frontend.cut_inlines)
  3rdParty/DirectXTex/.../DirectXTexMisc.cpp      DirectX::CopyRectangle (:174-274), whole
  3rdParty/DirectXTex/.../DirectXTexConvert.cpp   _ConvertScanline after its table lookups, XMColorSRGBToRGB / RGBToSRGB, the
                                                  g_ConvertTable rows: the same cuts as oracle/build_ref_preview.py
  3rdParty/DirectXTex/.../DirectXTex.h            TEX_FILTER_DEFAULT, TEX_FILTER_SEPARATE_ALPHA, TEX_MISC_TEXTURECUBE

NOT cut, restated in the shim below, and why:
  * ScratchImage: Initialize2D (zeroed, as DirectXTexImage.cpp:398-399 of this tree does), InitializeCube, GetImage(mip, item, 0)
    (item-major, mip-minor), GetImages, GetImageCount, GetMetadata -- the allocation bookkeeping of DirectXTexImage.cpp.
  * _LoadScanline for R8G8B8A8_UNORM / _SRGB (XMLoadUByteN4: byte * (1/255), the DirectXMath behaviour the project assumes
    everywhere) and R16G16B16A16_FLOAT (XMConvertHalfToFloat, DirectXMath 3.06 as build_ref_frontend.py restates it);
    _StoreScanline as build_ref_preview.py restates it; BitsPerPixel / IsCompressed / IsPlanar / IsPalettized for these formats.
  * GenerateMipMaps: the reference's own non-WIC generators as oracle/_ref/libitw_ref_frontend.so exports them
    (ref_mip_chain_rgba8 / ref_mip_chain_f16, cut by build_ref_frontend.py), one chain per array item.  The plug-in's preview
    asks for TEX_FILTER_DEFAULT, which DirectXTex serves through WIC for UNORM formats: not in the tree (DESIGN.md section 7).
  * Photoshop SDK glue: ReadLayerDesc (next, name, channel lists), ReadChannelDesc, ReadLayerData as the rectangle copy of
    build_ref_layers.py, sPSBuffer, SetResult, UserError.
Used by tests/test_cube_vs_reference.py.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_frontend as F          # IntelPlugin.h helpers, the half conversions, the cutting routine
import build_ref_preview as P           # the _ConvertScanline cut and its DirectXMath shim

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = F.OUT_DIR
OUT_SO = os.path.join(OUT_DIR, "libitw_ref_cube.so")
MISC_CPP = os.path.join(P.DXTEX, "DirectXTexMisc.cpp")
MEMBERS = ["IsCubeMapWithSetMipLevelOverride", "ConvertToCubeMapFromCross", "ConvertToCubeMapFromLayers",
           "ConvertToHorizontalCrossFromCubeMap", "FillLayerDataToWhite", "CopyFromLayerChannelIntoImage"]

SHIM_SCRATCH = r"""
struct TexMetadata { size_t width, height, depth, arraySize, mipLevels; uint32_t miscFlags; DXGI_FORMAT format; };
class ScratchImage {                                      // restated bookkeeping of DirectXTexImage.cpp
public:
    HRESULT Initialize2D(DXGI_FORMAT fmt, size_t width, size_t height, size_t arraySize, size_t mipLevels, DWORD flags = 0)
    {
        (void)flags;
        m_ = TexMetadata{width, height, 1, arraySize, mipLevels, 0, fmt};
        const size_t texel = BitsPerPixel(fmt) / 8;
        images_.clear();
        store_.clear();
        for (size_t item = 0; item < arraySize; item++)
            for (size_t l = 0; l < mipLevels; l++) {
                const size_t w = std::max<size_t>(1, width >> l), h = std::max<size_t>(1, height >> l);
                store_.emplace_back(w * h * texel, (uint8_t)0);          // zeroed, DirectXTexImage.cpp:398-399
                images_.push_back(Image{w, h, fmt, w * texel, w * h * texel, store_.back().data()});
            }
        return S_OK;
    }
    HRESULT InitializeCube(DXGI_FORMAT fmt, size_t width, size_t height, size_t nCubes, size_t mipLevels, DWORD flags = 0)
    {
        HRESULT hr = Initialize2D(fmt, width, height, nCubes * 6, mipLevels, flags);
        m_.miscFlags |= TEX_MISC_TEXTURECUBE;
        return hr;
    }
    const Image* GetImages() const { return images_.data(); }
    size_t GetImageCount() const { return images_.size(); }
    const TexMetadata& GetMetadata() const { return m_; }
    const Image* GetImage(size_t mip, size_t item, size_t slice) const
    {
        if (mip >= m_.mipLevels || item >= m_.arraySize || slice) return nullptr;
        return &images_[item * m_.mipLevels + mip];
    }
private:
    TexMetadata m_{};
    std::vector<Image> images_;
    std::vector<std::vector<uint8_t>> store_;
};
"""

SHIM_SCANLINE = r"""
static size_t BitsPerPixel(DXGI_FORMAT f) { return f == DXGI_FORMAT_R32G32B32A32_FLOAT ? 128 : (f == DXGI_FORMAT_R16G16B16A16_FLOAT ? 64 : 32); }
static bool IsCompressed(DXGI_FORMAT f) { return f >= DXGI_FORMAT_BC1_TYPELESS && f <= DXGI_FORMAT_BC7_UNORM_SRGB && f != 89 && f != 91 && f != 93; }
static bool IsPlanar(DXGI_FORMAT) { return false; }
static bool IsPalettized(DXGI_FORMAT) { return false; }
static bool _LoadScanline(XMVECTOR* pDestination, size_t count, const void* pSource, size_t size, DXGI_FORMAT format)
{
    const uint8_t* s = static_cast<const uint8_t*>(pSource);
    if (format == DXGI_FORMAT_R8G8B8A8_UNORM || format == DXGI_FORMAT_R8G8B8A8_UNORM_SRGB) {   // XMLoadUByteN4
        for (size_t i = 0; i < count && (i + 1) * 4 <= size; i++)
            for (int c = 0; c < 4; c++) pDestination[i].f[c] = (float)s[4 * i + c] * (1.0f / 255.0f);
        return true;
    }
    if (format == DXGI_FORMAT_R16G16B16A16_FLOAT) {                                           // XMLoadHalf4
        for (size_t i = 0; i < count && (i + 1) * 8 <= size; i++)
            for (int c = 0; c < 4; c++) {
                unsigned short h;
                memcpy(&h, s + 8 * i + 2 * c, 2);
                pDestination[i].f[c] = PackedVector::XMConvertHalfToFloat(h);
            }
        return true;
    }
    return false;
}
struct Rect { size_t x, y, w, h; Rect() = default; Rect(size_t _x, size_t _y, size_t _w, size_t _h) : x(_x), y(_y), w(_w), h(_h) {} };
#define E_INVALIDARG (-3L)
#define E_OUTOFMEMORY (-2L)
static inline void memcpy_s(void* d, size_t, const void* s, size_t n) { memcpy(d, s, n); }
static inline void* _aligned_malloc(size_t n, size_t) { return malloc(n); }
struct ScopedAlignedArrayXMVECTOR {
    XMVECTOR* p;
    explicit ScopedAlignedArrayXMVECTOR(XMVECTOR* q) : p(q) {}
    ~ScopedAlignedArrayXMVECTOR() { free(p); }
    XMVECTOR* get() const { return p; }
    explicit operator bool() const { return p != nullptr; }
};
"""

SHIM_MIPS = r"""
}  // namespace DirectX
}  // namespace itw_ref_cube
extern "C" int ref_mip_chain_rgba8(const uint8_t* level0, int w, int h, int levels, int srgb, uint8_t* out);
extern "C" int ref_mip_chain_f16(const unsigned short* level0, int w, int h, int levels, unsigned short* out);
namespace itw_ref_cube {
namespace DirectX {
// GenerateMipMaps (levels 0 = the full chain) through the reference's own non-WIC generators, one chain per array item
static HRESULT GenerateMipMaps(const Image* srcImages, size_t nimages, const TexMetadata& metadata, DWORD, size_t levels, ScratchImage& mipChain)
{
    size_t full = 1;
    for (size_t m = std::max(metadata.width, metadata.height); m > 1; m >>= 1) full++;
    if (!levels) levels = full;
    if (nimages != metadata.arraySize || metadata.mipLevels != 1) return E_FAIL;
    mipChain.Initialize2D(metadata.format, metadata.width, metadata.height, metadata.arraySize, levels);
    const size_t texel = BitsPerPixel(metadata.format) / 8;
    size_t total = 0;
    for (size_t l = 0; l < levels; l++) total += std::max<size_t>(1, metadata.width >> l) * std::max<size_t>(1, metadata.height >> l) * texel;
    std::vector<uint8_t> chain(total);
    for (size_t item = 0; item < nimages; item++) {
        const int w = (int)metadata.width, h = (int)metadata.height;
        int rc = metadata.format == DXGI_FORMAT_R16G16B16A16_FLOAT
                     ? ref_mip_chain_f16(reinterpret_cast<const unsigned short*>(srcImages[item].pixels), w, h, (int)levels,
                                         reinterpret_cast<unsigned short*>(chain.data()))
                     : ref_mip_chain_rgba8(srcImages[item].pixels, w, h, (int)levels, metadata.format == DXGI_FORMAT_R8G8B8A8_UNORM_SRGB, chain.data());
        if (rc) return E_FAIL;
        size_t off = 0;
        for (size_t l = 0; l < levels; l++) {
            const Image* dst = mipChain.GetImage(l, item, 0);
            memcpy(dst->pixels, chain.data() + off, dst->slicePitch);
            off += dst->slicePitch;
        }
    }
    return S_OK;
}
"""

SHIM_PLUGIN = r"""
}  // namespace DirectX
using namespace DirectX;
typedef unsigned char unsigned8;
typedef unsigned short unsigned16;
enum { memFullErr = -108 };
struct ReadChannelDesc { ReadChannelDesc* next; const char* plane; long long row_bytes; int depth; };
struct ReadLayerDesc { ReadLayerDesc* next; const char* name; ReadChannelDesc* compositeChannelsList; ReadChannelDesc* layerMask; ReadChannelDesc* transparency; };
struct FakeDocumentInfo { ReadLayerDesc* layersDescriptor; int layerCount; };
struct FakePoint { int h, v; };
struct FakeFormatRecord { int depth; FakePoint imageSize; int planeBytes; FakeDocumentInfo* documentInfo; };
struct FakeData { int encoding_g; bool SetMipLevel; int TextureTypeIndex; int MipLevel; };
struct FakeGlobals { FakeFormatRecord* formatRecord; FakeData* data; };
struct FakeBufferProcs {
    char* New(void*, size_t n) { return static_cast<char*>(malloc(n)); }
    void Dispose(char** p) { free(*p); *p = nullptr; }
};
static FakeBufferProcs g_buffer_procs;
static FakeBufferProcs* sPSBuffer = &g_buffer_procs;
@TEXTURE_TYPES@
@INLINES@
class IntelPlugin {
public:
    FakeGlobals ps;
    int user_errors = 0;
    void SetResult(int) {}
    void UserError(const char*) { user_errors++; }
    // ReadPixelsFromLevel of the rectangle (0, 0)-(width, height) into rows of width * depth bits (IntelPlugin.cpp:1618-1662)
    void ReadLayerData(ReadChannelDesc* pChannel, char* pLayerData, int width, int height)
    {
        const size_t row = (size_t)width * pChannel->depth / 8;
        for (int y = 0; y < height; y++) memcpy(pLayerData + row * y, pChannel->plane + pChannel->row_bytes * y, row);
    }
    bool IsCubeMapWithSetMipLevelOverride();
    void ConvertToCubeMapFromCross(ScratchImage** scrUncompressedImageScratch_);
    bool ConvertToCubeMapFromLayers(ScratchImage** scrUncompressedImageScratch_, bool hasAlpha_);
    void ConvertToHorizontalCrossFromCubeMap(ScratchImage** scrUncompressedImageScratch_);
    void FillLayerDataToWhite(char* pLayerData, int width, int height);
    void CopyFromLayerChannelIntoImage(char* pLayerData, const Image* image, int indexToImage, int indexToLayerChannel);
};
"""

SHIM_BOTTOM = r"""
static void copy_out(const ScratchImage& s, size_t mip, uint8_t* out)
{
    for (size_t i = 0; i < s.GetMetadata().arraySize; i++) {
        const Image* im = s.GetImage(mip, i, 0);
        memcpy(out, im->pixels, im->slicePitch);
        out += im->slicePitch;
    }
}
}  // namespace itw_ref_cube
using namespace itw_ref_cube;
#define ITW_EXPORT extern "C" __attribute__((visibility("default")))

// IsCubeMapWithSetMipLevelOverride for the dialog's SetMipLevel box and texture type
ITW_EXPORT int ref_cube_set_level_override(int set_mip_level, int texture_type)
{
    IntelPlugin p;
    FakeData dat{0, set_mip_level != 0, texture_type, 0};
    p.ps.data = &dat;
    return p.IsCubeMapWithSetMipLevelOverride() ? 1 : 0;
}

// ConvertToCubeMapFromCross: `doc` = the document scratch, doc_w x doc_h tight texels of `doc_format` (28, 29 or 10), as
// CopyDataForEncoding leaves it.  `out` receives the six faces, tight, +X..-Z; *face_w / *face_h their size.
ITW_EXPORT int ref_cube_from_cross(int encoding, int doc_format, int doc_w, int doc_h, const uint8_t* doc, uint8_t* out, int* face_w, int* face_h)
{
    IntelPlugin p;
    FakeFormatRecord rec{0, {doc_w, doc_h}, 0, nullptr};
    FakeData dat{encoding, false, CUBEMAP_CROSSED, 0};
    p.ps.formatRecord = &rec;
    p.ps.data = &dat;
    ScratchImage* s = new ScratchImage();
    s->Initialize2D((DXGI_FORMAT)doc_format, doc_w, doc_h, 1, 1);
    memcpy(s->GetImages()->pixels, doc, s->GetImages()->slicePitch);
    p.ConvertToCubeMapFromCross(&s);
    *face_w = (int)s->GetMetadata().width;
    *face_h = (int)s->GetMetadata().height;
    if (out) copy_out(*s, 0, out);
    delete s;
    return 0;
}

// ConvertToCubeMapFromLayers on a w x h document of `depth` bits: layer i is named names[i], has channel_count[i] planes
// planes[4 i + c] and alpha planes[4 i + 3] (its transparency, or null), all rows w * depth / 8 bytes.  Returns the call's result
// (0 = "not enough layers"); `out` receives the six faces.
ITW_EXPORT int ref_cube_from_layers(int encoding, int depth, int w, int h, const char* const* names, const void* const* planes,
                                    const int* channel_count, int layer_count, int has_alpha, uint8_t* out)
{
    IntelPlugin p;
    std::vector<ReadChannelDesc> ch((size_t)layer_count * 4);
    std::vector<ReadLayerDesc> layers((size_t)layer_count);
    const long long row = (long long)w * depth / 8;
    for (int i = 0; i < layer_count; i++) {
        ReadLayerDesc& L = layers[i];
        L = ReadLayerDesc{i + 1 < layer_count ? &layers[i + 1] : nullptr, names[i], nullptr, nullptr, nullptr};
        for (int c = 0; c < channel_count[i]; c++)
            ch[4 * i + c] = ReadChannelDesc{c + 1 < channel_count[i] ? &ch[4 * i + c + 1] : nullptr, static_cast<const char*>(planes[4 * i + c]), row, depth};
        L.compositeChannelsList = channel_count[i] ? &ch[4 * i] : nullptr;
        if (planes[4 * i + 3]) {
            ch[4 * i + 3] = ReadChannelDesc{nullptr, static_cast<const char*>(planes[4 * i + 3]), row, depth};
            L.transparency = &ch[4 * i + 3];
        }
    }
    FakeDocumentInfo doc{layer_count ? &layers[0] : nullptr, layer_count};
    FakeFormatRecord rec{depth, {w, h}, depth / 8, &doc};
    FakeData dat{encoding, false, CUBEMAP_LAYERS, 0};
    p.ps.formatRecord = &rec;
    p.ps.data = &dat;
    ScratchImage* s = new ScratchImage();
    s->Initialize2D(encoding == DXGI_FORMAT_BC6H_UF16 ? DXGI_FORMAT_R16G16B16A16_FLOAT : DXGI_FORMAT_R8G8B8A8_UNORM, w, h, 1, 1);
    const bool ok = p.ConvertToCubeMapFromLayers(&s, has_alpha != 0);
    if (ok && out) copy_out(*s, 0, out);
    delete s;
    return ok ? 1 : 0;
}

// ConvertToHorizontalCrossFromCubeMap on a one-level cube of w x h faces (`faces`: six tight faces of the cube scratch's format,
// R16G16B16A16_FLOAT for encoding 95, else R8G8B8A8_UNORM), with the dialog's SetMipLevel / MipLevel / texture type.  `out`
// (may be null) receives the cross; *cross_w / *cross_h its size.  Returns the UserError count.
ITW_EXPORT int ref_cross_from_cube(int encoding, int texture_type, int set_mip_level, int mip_level, int w, int h, const uint8_t* faces,
                                   uint8_t* out, int* cross_w, int* cross_h)
{
    IntelPlugin p;
    FakeData dat{encoding, set_mip_level != 0, texture_type, mip_level};
    p.ps.data = &dat;
    ScratchImage* s = new ScratchImage();
    s->InitializeCube(encoding == DXGI_FORMAT_BC6H_UF16 ? DXGI_FORMAT_R16G16B16A16_FLOAT : DXGI_FORMAT_R8G8B8A8_UNORM, w, h, 1, 1);
    for (int i = 0; i < 6; i++) {
        const Image* im = s->GetImage(0, i, 0);
        memcpy(im->pixels, faces + i * im->slicePitch, im->slicePitch);
    }
    p.ConvertToHorizontalCrossFromCubeMap(&s);
    *cross_w = (int)s->GetMetadata().width;
    *cross_h = (int)s->GetMetadata().height;
    if (out) memcpy(out, s->GetImages()->pixels, s->GetImages()->slicePitch);
    delete s;
    return p.user_errors;
}
"""


def cut_members(cpp):
    out = []
    for name in MEMBERS:
        m = re.search(r"^[A-Za-z_][\w \t\*&:]*\bIntelPlugin::" + name + r"\s*\(", cpp, re.M)
        if not m:
            raise RuntimeError(f"IntelPlugin::{name} not found in the reference")
        out.append(F.cut_function(cpp, m.start()))
    return "\n\n".join(out)


def cut_texture_types(hdr):
    m = re.search(r"^enum TextureTypeEnum\s*\{[^}]*\};", hdr, re.M)
    if not m:
        raise RuntimeError("enum TextureTypeEnum not found in IntelPlugin.h")
    return m.group(0) + "\n"


def cut_tex_enums(tex):
    vals = re.findall(r"^\s*(TEX_FILTER_DEFAULT|TEX_FILTER_SEPARATE_ALPHA|TEX_MISC_TEXTURECUBE)\s*=\s*(0x[0-9A-Fa-f]+L?|\d+)", tex, re.M)
    if len(vals) != 3:
        raise RuntimeError("TEX_FILTER_DEFAULT / TEX_FILTER_SEPARATE_ALPHA / TEX_MISC_TEXTURECUBE not found")
    return "enum TEX_CUBE_FLAGS { " + ", ".join(f"{n} = {v.rstrip('L')}" for n, v in vals) + " };\n"


def half_conversions():
    a = F.SHIM_TOP.index("namespace PackedVector {")
    b = F.SHIM_TOP.index("}  // namespace PackedVector") + len("}  // namespace PackedVector")
    return F.SHIM_TOP[a:b] + "\n"


def preview_shim(part):
    """Pieces of build_ref_preview.SHIM_TOP: 'head' = includes and HRESULT macros, 'xm' = the DirectXMath shim, 'convert' = the
    ConvertData table, _ConvertScanline and _StoreScanline frame."""
    s = P.SHIM_TOP
    if part == "head":
        return s[:s.index("namespace itw_ref_preview {")]
    if part == "xm":
        return s[s.index("struct XMVECTOR {"):s.index("@ENUMS@")]
    a, b = s.index("struct ConvertData {"), s.index("static size_t BitsPerPixel(")
    return s[a:b]


def build(verbose=True):
    have_ref = os.path.exists(F.PLUGIN_CPP) and os.path.exists(MISC_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {F.REF_ROOT} and no prebuilt {OUT_SO}")
    dep = os.path.join(OUT_DIR, "libitw_ref_frontend.so")
    if not os.path.exists(dep):
        raise FileNotFoundError(f"{dep} is built by build_ref_frontend.py first")
    deps = [__file__, F.__file__, P.__file__, F.PLUGIN_CPP, F.PLUGIN_H, MISC_CPP, P.CONVERT_CPP, dep]
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in deps):
        return OUT_SO
    os.makedirs(OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_cube_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        conv, hdr, tex = read(P.CONVERT_CPP), read(F.PLUGIN_H), read(P.TEX_H)
        formats = dict(P.FORMATS, R16G16B16A16_FLOAT=10)
        inlines = F.cut_inlines(hdr).replace("DirectX::PackedVector::", "PackedVector::")
        unit = ("// generated by oracle/build_ref_cube.py -- shim around function bodies cut from the reference\n"
                + preview_shim("head") + "#include <map>\n#include <string>\n#include <vector>\n"
                + "namespace itw_ref_cube {\nnamespace DirectX {\n"
                + "enum DXGI_FORMAT { " + ", ".join(f"DXGI_FORMAT_{n} = {v}" for n, v in formats.items()) + " };\n"
                + "struct Image { size_t width, height; DXGI_FORMAT format; size_t rowPitch, slicePitch; uint8_t* pixels; };\n"
                + half_conversions() + preview_shim("xm") + P.cut_enums(read(P.TEXP_H), tex) + cut_tex_enums(tex)
                + preview_shim("convert").replace("@TABLE@", P.cut_table(conv)).replace("@SRGB@", P.cut_grayscale(conv) + P.cut_srgb(conv))
                  .replace("@CONVERT_BODY@", P.cut_convert_body(conv))
                + SHIM_SCANLINE + SHIM_SCRATCH + F.cut_function(read(MISC_CPP), re.search(r"^HRESULT CopyRectangle\s*\(", read(MISC_CPP), re.M).start())
                + SHIM_MIPS
                + SHIM_PLUGIN.replace("@TEXTURE_TYPES@", cut_texture_types(hdr)).replace("@INLINES@", inlines)
                + cut_members(read(F.PLUGIN_CPP)) + SHIM_BOTTOM)
        path = os.path.join(tmp, "cube_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-fvisibility=hidden", "-ffp-contract=off", "-fno-fast-math",
               "-mfpmath=sse", "-msse2", path, "-o", OUT_SO, "-L" + OUT_DIR, "-l:" + os.path.basename(dep), "-Wl,-rpath,$ORIGIN"]
        if verbose:
            print("[build_ref_cube]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_cube] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
