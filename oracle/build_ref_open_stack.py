#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_open_stack.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

What LoadFromDDSMemory (DDS_FLAGS_NONE) makes of a volume texture, a 1-D texture or a texture array, and which image the plug-in's
GetImage(mip, item, slice) calls name (IntelPlugin.cpp:2465, :2665):

  3rdParty/DirectXTex/DirectXTex/DirectXTexDDS.cpp      CONVERSION_FLAGS, LegacyDDS and g_LegacyDDSMap, _GetDXGIFormat and _DecodeDDSHeader
                                                        (its dimension and volume branches included), whole; LoadFromDDSMemory's
                                                        palette step (:1402-1410); _CopyImage's size check (:1028-1062: the EXPAND
                                                        cpFlags choice, _DetermineImageArray, _SetupImageArray over the file's payload)
  3rdParty/DirectXTex/DirectXTex/DirectXTexImage.cpp    _DetermineImageArray, _SetupImageArray, ScratchImage::Initialize and
                                                        ScratchImage::GetImage, whole
  3rdParty/DirectXTex/DirectXTex/DirectXTexMipmaps.cpp  _CountMips, _CalculateMipLevels, _CountMips3D and _CalculateMipLevels3D, whole
  3rdParty/DirectXTex/DirectXTex/DirectXTexUtil.cpp     ComputePitch and BitsPerPixel, whole
  3rdParty/DirectXTex/DirectXTex/DirectXTex.inl         IsValid, IsCompressed, IsPacked, IsPlanar and IsPalettized, whole
  3rdParty/DirectXTex/DirectXTex/DirectXTex.h           the CP_FLAGS enum

The per-texel and per-block rules of each family come from the other recipes' libraries in the tests.

NOT cut, restated in the shim below, and why:
  * The ScratchImage class around the cut members: its fields, Release and the accessors (DirectXTex.h).  An allocation above
    4 GiB fails, as it does on a host without that memory, so a header whose item count is absurd is refused without being
    allocated (Initialize returns E_OUTOFMEMORY).
  * LoadFromDDSMemory's order of the steps: _DecodeDDSHeader, the payload offset, the palette step, Initialize, the size check.
Only the .so is kept (git-ignored; travels to the GPU box).  Used by tests/test_dds_open_stack.py and its GPU twin.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_dds as D                # the DXGI numbering, the SHIM_TOP of the header cut, cut_function
import build_ref_open_uncompressed as U  # cut_between, DXTEX

IMAGE_CPP = os.path.join(U.DXTEX, "DirectXTexImage.cpp")
MIPS_CPP = os.path.join(U.DXTEX, "DirectXTexMipmaps.cpp")
UTIL_CPP = os.path.join(U.DXTEX, "DirectXTexUtil.cpp")
TEX_INL = os.path.join(U.DXTEX, "DirectXTex.inl")
TEX_H = os.path.join(U.DXTEX, "DirectXTex.h")
OUT_SO = os.path.join(D.OUT_DIR, "libitw_ref_open_stack.so")

INCLUDES = r"""
#undef extern
#undef __declspec
#include <new>
#include <vector>
#include <memory>
#include <algorithm>
#include <cstdlib>
using namespace DirectX;
"""

MID = r"""
typedef const void* LPCVOID;
#define __cdecl
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
#define E_OUTOFMEMORY (-4L)
#define FAILED(hr) ((hr) < 0)
enum TEX_DIMENSION { TEX_DIMENSION_TEXTURE1D = 2, TEX_DIMENSION_TEXTURE2D = 3, TEX_DIMENSION_TEXTURE3D = 4 };
enum { TEX_MISC_TEXTURECUBE = 0x4 };
enum { TEX_MISC2_ALPHA_MODE_MASK = 0x7 };
enum { TEX_ALPHA_MODE_UNKNOWN = 0, TEX_ALPHA_MODE_STRAIGHT = 1, TEX_ALPHA_MODE_PREMULTIPLIED = 2, TEX_ALPHA_MODE_OPAQUE = 3, TEX_ALPHA_MODE_CUSTOM = 4 };
enum { DDS_FLAGS_NONE = 0, DDS_FLAGS_LEGACY_DWORD = 0x1, DDS_FLAGS_NO_LEGACY_EXPANSION = 0x2, DDS_FLAGS_NO_R10B10G10A2_FIXUP = 0x4,
       DDS_FLAGS_FORCE_RGB = 0x8, DDS_FLAGS_NO_16BPP = 0x10, DDS_FLAGS_EXPAND_LUMINANCE = 0x20 };
#define ERROR_INVALID_DATA 13L
struct TexMetadata {
    size_t width, height, depth, arraySize, mipLevels;
    uint32_t miscFlags, miscFlags2;
    DXGI_FORMAT format;
    TEX_DIMENSION dimension;
    bool IsCubemap() const { return (miscFlags & TEX_MISC_TEXTURECUBE) != 0; }
};
static const size_t kAllocLimit = size_t(1) << 32;
struct Image {
    size_t width, height;
    DXGI_FORMAT format;
    size_t rowPitch, slicePitch;
    uint8_t* pixels;
    static void* operator new[](size_t n, const std::nothrow_t& t) noexcept { return n > kAllocLimit ? nullptr : ::operator new[](n, t); }
    static void* operator new[](size_t n) { return ::operator new[](n); }
};
static void* _aligned_malloc(size_t n, size_t a) { return n > kAllocLimit ? nullptr : aligned_alloc(a, (n + a - 1) / a * a); }
class ScratchImage {
public:
    ~ScratchImage() { Release(); }
    HRESULT Initialize(const TexMetadata& mdata, DWORD flags = CP_FLAGS_NONE);
    const Image* GetImage(size_t mip, size_t item, size_t slice) const;
    const Image* GetImages() const { return _image; }
    size_t GetImageCount() const { return _nimages; }
    uint8_t* GetPixels() const { return _memory; }
    const TexMetadata& GetMetadata() const { return _metadata; }
    void Release() { delete[] _image; _image = nullptr; free(_memory); _memory = nullptr; _nimages = _size = 0; }
private:
    size_t _nimages = 0, _size = 0;
    TexMetadata _metadata{};
    Image* _image = nullptr;
    uint8_t* _memory = nullptr;
};
"""

BOTTOM = r"""
// _CopyImage's size check on the file's payload: the image table _SetupImageArray lays over `size` bytes at pPixels
static HRESULT copy_size_check(const void* pPixels, size_t size, const TexMetadata& metadata, DWORD cpFlags, DWORD convFlags,
                               const ScratchImage& image, std::vector<Image>& table, size_t& payload)
{
@CHECK@
    table.assign(timages.get(), timages.get() + nimages);
    payload = pixelSize;
    return S_OK;
}

struct Loaded {
    TexMetadata mdata;
    DWORD convFlags = 0;
    size_t offset = 0, payload = 0;
    ScratchImage image;
    std::vector<Image> table;          // the file's images, in ScratchImage's order
};
// LoadFromDDSMemory up to the copy: the header, the offset, the palette, Initialize, the size check
static HRESULT load(const uint8_t* pSource, size_t size, Loaded& L)
{
    TexMetadata& mdata = L.mdata;
    DWORD& convFlags = L.convFlags;
    HRESULT hr = _DecodeDDSHeader(pSource, size, DDS_FLAGS_NONE, mdata, convFlags);
    if (FAILED(hr)) return hr;
    size_t offset = sizeof(uint32_t) + sizeof(DDS_HEADER);
    if (convFlags & CONV_FLAGS_DX10) offset += sizeof(DDS_HEADER_DXT10);
@PALETTE@
    hr = L.image.Initialize(mdata);
    if (FAILED(hr)) return hr;
    L.offset = offset;
    return copy_size_check(pSource + offset, size - offset, mdata, CP_FLAGS_NONE, convFlags, L.image, L.table, L.payload);
}
}  // namespace itw_ref_open_stack

using namespace itw_ref_open_stack;

// out: width, height, depth, mipLevels (Initialize's), arraySize, format, cube, dimension, convFlags, payload offset, image count,
// payload bytes.  Returns the HRESULT (0 = S_OK).
extern "C" long ref_stack_load(const uint8_t* file, size_t size, uint64_t* out)
{
    Loaded L;
    const HRESULT hr = load(file, size, L);
    if (hr != S_OK) return hr;
    const TexMetadata& m = L.image.GetMetadata();
    const uint64_t v[12] = {m.width, m.height, m.depth, m.mipLevels, m.arraySize, (uint64_t)m.format, m.IsCubemap() ? 1u : 0u,
                            (uint64_t)m.dimension, L.convFlags, L.offset, L.image.GetImageCount(), L.payload};
    memcpy(out, v, sizeof(v));
    return 0;
}
// Every image of the file in ScratchImage's order: (file offset, width, height, rowPitch, slicePitch) each; returns the count, or -1
extern "C" long long ref_stack_images(const uint8_t* file, size_t size, uint64_t* out, long long cap)
{
    Loaded L;
    if (load(file, size, L) != S_OK || (long long)L.table.size() > cap) return -1;
    for (size_t i = 0; i < L.table.size(); i++) {
        const Image& im = L.table[i];
        const uint64_t v[5] = {(uint64_t)(im.pixels - file), im.width, im.height, im.rowPitch, im.slicePitch};
        memcpy(out + 5 * i, v, sizeof(v));
    }
    return (long long)L.table.size();
}
// ScratchImage::GetImage(mip, item, slice) of the loaded file: its index in the image table, or -1 when it returns nullptr
extern "C" long long ref_stack_get_image(const uint8_t* file, size_t size, uint64_t mip, uint64_t item, uint64_t slice)
{
    Loaded L;
    if (load(file, size, L) != S_OK) return -2;
    const Image* im = L.image.GetImage(mip, item, slice);
    return im ? (long long)(im - L.image.GetImages()) : -1;
}
"""


def build(verbose=True):
    have_ref = os.path.exists(D.DDS_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {D.REF_ROOT} and no prebuilt {OUT_SO}")
    srcs = [__file__, D.__file__, U.__file__, D.DDS_CPP, D.DDS_H, IMAGE_CPP, MIPS_CPP, UTIL_CPP, TEX_INL, TEX_H]
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in srcs):
        return OUT_SO
    os.makedirs(D.OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_open_stack_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        dds, image, mips, util, inl, tex_h = (read(p) for p in (D.DDS_CPP, IMAGE_CPP, MIPS_CPP, UTIL_CPP, TEX_INL, TEX_H))
        hdr = read(D.DDS_H)
        dds_h = hdr[hdr.index("namespace DirectX"):hdr.rindex("}; // namespace")] + "}  // namespace DirectX\n"
        enum = ",\n".join(f"    DXGI_FORMAT_{name} = {i}" for i, name in enumerate(D.DXGI))
        fn = lambda src, pat: D.cut_function(src, re.search(pat, src, re.M).start())
        load = fn(dds, r"^HRESULT LoadFromDDSMemory\s*\(")
        palette = "    const uint32_t *pal8 = nullptr;\n    " + D.cut_function(load, load.index("if ( convFlags & CONV_FLAGS_PAL8 )"))
        copy = fn(dds, r"^static HRESULT _CopyImage\s*\(")
        check = copy[copy.index("    if ( !size )"):copy.index("    if ( nimages != image.GetImageCount() )")]
        parts = [
            D.SHIM_TOP.replace("@DXGI@", enum), dds_h,
            U.cut_between(tex_h, r"^\s*enum CP_FLAGS", "};"),
            INCLUDES,
            "\nnamespace itw_ref_open_stack {\n",
            MID,
            fn(inl, r"^inline bool __cdecl IsValid\s*\("),
            fn(inl, r"^inline bool __cdecl IsCompressed\s*\("),
            fn(inl, r"^inline bool __cdecl IsPacked\s*\("),
            fn(inl, r"^inline bool __cdecl IsPlanar\s*\("),
            fn(inl, r"^inline bool __cdecl IsPalettized\s*\("),
            fn(util, r"^size_t BitsPerPixel\s*\("),
            fn(util, r"^void ComputePitch\s*\("),
            fn(mips, r"^static size_t _CountMips\s*\("),
            fn(mips, r"^bool _CalculateMipLevels\s*\("),
            fn(mips, r"^static size_t _CountMips3D\s*\("),
            fn(mips, r"^bool _CalculateMipLevels3D\s*\("),
            fn(image, r"^void _DetermineImageArray\s*\("),
            fn(image, r"^bool _SetupImageArray\s*\("),
            fn(image, r"^HRESULT ScratchImage::Initialize\s*\(\s*const TexMetadata"),
            fn(image, r"^const Image\* ScratchImage::GetImage\s*\("),
            U.cut_between(dds, r"^enum CONVERSION_FLAGS", "};"),
            U.cut_between(dds, r"^struct LegacyDDS", "};"),
            U.cut_between(dds, r"^const LegacyDDS g_LegacyDDSMap\[\]", "\n};"),
            fn(dds, r"^static DXGI_FORMAT _GetDXGIFormat\s*\("),
            fn(dds, r"^static HRESULT _DecodeDDSHeader\s*\("),
            BOTTOM.replace("@CHECK@", check).replace("@PALETTE@", palette),
        ]
        unit = "\n".join(parts).replace("_Success_(return != false)", "")
        path = os.path.join(tmp, "open_stack_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_open_stack]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_open_stack] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
