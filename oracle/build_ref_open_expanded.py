#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_open_expanded.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

What LoadFromDDSMemory (DDS_FLAGS_NONE) does to the D3D9 files it expands while it loads (P8, A8P8, A8R3G3B2, A4L4; the plug-in's
DoReadStart, IntelPlugin.cpp:2465):

  3rdParty/DirectXTex/DirectXTex/DirectXTexDDS.cpp      CONVERSION_FLAGS, LegacyDDS and g_LegacyDDSMap, _GetDXGIFormat, _DecodeDDSHeader,
                                                        TEXP_LEGACY_FORMAT / _FindLegacyFormat and _LegacyExpandScanline, whole, as
                                                        build_ref_open_uncompressed.py cuts them; LoadFromDDSMemory's palette step
                                                        (the CONV_FLAGS_PAL8 block, :1402-1410) and _CopyImage's EXPAND row choice (the
                                                        cpFlags block, :1033-1041)
  3rdParty/DirectXTex/DirectXTex/DirectXTexUtil.cpp     ComputePitch's bits-per-pixel choice (CP_FLAGS_24BPP / 16BPP / 8BPP)
  3rdParty/DirectXTex/DirectXTex/DirectXTex.h           the CP_FLAGS enum

The rest of the path reuses other recipes' libraries from the tests: A4L4's B4G4R4A4_UNORM texels go through build_ref_open_converted.py's
_LoadScanline / _ConvertScanline / _StoreScanline and its alpha branch, the R8G8B8A8_UNORM alpha branch is build_ref_open_uncompressed.py's,
and _UseWICConversion is build_ref_open_converted.py's.

NOT cut, restated in the shim below, and why:
  * The rest of _CopyImage and _SetupImageArray: the image table (item-major, mip-minor images of max(1, w >> l) x max(1, h >> l)
    texels), the row loop calling _LegacyExpandScanline per row with the source and destination pitches, and the check that the
    payload holds every image (E_FAIL otherwise).  ComputePitch's default byte alignment, (width * bpp + 7) / 8, is restated with it.
  * BitsPerPixel, which these files never reach (every EXPAND entry sets a CP_FLAGS_*BPP override); it aborts.
Only the .so is kept (git-ignored; travels to the GPU box).  Used by tests/test_dds_open_expanded.py and its GPU twin.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_dds as D                # the DXGI numbering, the SHIM_TOP of the header cut, cut_function
import build_ref_open_uncompressed as U  # the header decoder and legacy expansion cuts, their shim

HERE = os.path.dirname(os.path.abspath(__file__))
UTIL_CPP = os.path.join(U.DXTEX, "DirectXTexUtil.cpp")
TEX_H = os.path.join(U.DXTEX, "DirectXTex.h")
OUT_SO = os.path.join(D.OUT_DIR, "libitw_ref_open_expanded.so")

BOTTOM = r"""
#define FAILED(hr) ((hr) < 0)
static size_t BitsPerPixel(DXGI_FORMAT) { abort(); }
static size_t loaded_bytes(DXGI_FORMAT f) { return f == DXGI_FORMAT_B4G4R4A4_UNORM ? 2 : 4; }
// ComputePitch's bits per pixel (cut) with its default byte alignment
static size_t row_pitch(DXGI_FORMAT fmt, size_t width, DWORD flags)
{
@BPP@
    return (width * bpp + 7) / 8;
}
}  // namespace itw_ref_open_exp

using namespace itw_ref_open_exp;

// LoadFromDDSMemory for an expanded file: _DecodeDDSHeader, the palette step, _CopyImage's row choice and pitches, every row through
// _LegacyExpandScanline with the palette.  dst: the loaded payload (item-major, mip-minor, tight rows of the loaded format); meta:
// width, height, mipLevels, arraySize, format, cube, convFlags, pixel offset.  Returns the loaded bytes, or a failed HRESULT / -1.
extern "C" long long ref_load_expanded(const uint8_t* pSource, size_t size, uint8_t* dst, uint64_t* meta)
{
    DWORD convFlags = 0;
    TexMetadata mdata;
    HRESULT hr = _DecodeDDSHeader(pSource, size, DDS_FLAGS_NONE, mdata, convFlags);
    if (FAILED(hr)) return hr;
    size_t offset = sizeof(uint32_t) + sizeof(DDS_HEADER);
    if (convFlags & CONV_FLAGS_DX10) offset += sizeof(DDS_HEADER_DXT10);
@PALETTE@
    if (!(convFlags & CONV_FLAGS_EXPAND)) return -1;
    DWORD cpFlags = CP_FLAGS_NONE;
@CPFLAGS@
    const DWORD tflags = (convFlags & CONV_FLAGS_NOALPHA) ? TEXP_SCANLINE_SETALPHA : 0;
    meta[0] = mdata.width; meta[1] = mdata.height; meta[2] = mdata.mipLevels; meta[3] = mdata.arraySize; meta[4] = (uint64_t)mdata.format;
    meta[5] = (mdata.miscFlags & TEX_MISC_TEXTURECUBE) ? 1 : 0; meta[6] = convFlags; meta[7] = offset;
    const uint8_t* src = pSource + offset;
    size_t need = 0;
    for (size_t item = 0; item < mdata.arraySize; item++)
        for (size_t l = 0; l < mdata.mipLevels; l++)
            need += row_pitch(mdata.format, std::max<size_t>(1, mdata.width >> l), cpFlags) * std::max<size_t>(1, mdata.height >> l);
    if (need > size - offset) return E_FAIL;                                 // _SetupImageArray
    uint8_t* d0 = dst;
    for (size_t item = 0; item < mdata.arraySize; item++)
        for (size_t l = 0; l < mdata.mipLevels; l++) {
            const size_t lw = std::max<size_t>(1, mdata.width >> l), lh = std::max<size_t>(1, mdata.height >> l);
            const size_t spitch = row_pitch(mdata.format, lw, cpFlags), dpitch = lw * loaded_bytes(mdata.format);
            for (size_t y = 0; y < lh; y++) {
                if (!_LegacyExpandScanline(dst, dpitch, mdata.format, src, spitch, _FindLegacyFormat(convFlags), pal8, tflags)) return -1;
                src += spitch;
                dst += dpitch;
            }
        }
    return (long long)(dst - d0);
}
// _LegacyExpandScanline on one row of `n` texels of the legacy form of `conv` (a g_LegacyDDSMap convFlags) into `format`
extern "C" int ref_expand_texels(uint32_t conv, uint32_t format, const uint8_t* src, long long n, const uint32_t* pal8, uint8_t* dst)
{
    const DWORD cpFlags0 = CP_FLAGS_NONE;
    DWORD convFlags = conv, cpFlags = cpFlags0;
@CPFLAGS@
    const size_t spitch = row_pitch((DXGI_FORMAT)format, (size_t)n, cpFlags), dpitch = (size_t)n * loaded_bytes((DXGI_FORMAT)format);
    return _LegacyExpandScanline(dst, dpitch, (DXGI_FORMAT)format, src, spitch, _FindLegacyFormat(convFlags), pal8, 0) ? 0 : -1;
}
"""


def build(verbose=True):
    have_ref = os.path.exists(D.DDS_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {D.REF_ROOT} and no prebuilt {OUT_SO}")
    srcs = [__file__, D.__file__, U.__file__, D.DDS_CPP, D.DDS_H, U.TEXP_H, UTIL_CPP, TEX_H]
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in srcs):
        return OUT_SO
    os.makedirs(D.OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_open_exp_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        dds, util, texp, tex_h = (read(p) for p in (D.DDS_CPP, UTIL_CPP, U.TEXP_H, TEX_H))
        hdr = read(D.DDS_H)
        dds_h = hdr[hdr.index("namespace DirectX"):hdr.rindex("}; // namespace")] + "}  // namespace DirectX\n"
        enum = ",\n".join(f"    DXGI_FORMAT_{name} = {i}" for i, name in enumerate(D.DXGI))
        top = D.SHIM_TOP.replace("@DXGI@", enum).replace("#include <cstring>", "#include <cstring>\n#include <cstdlib>\n#include <algorithm>")
        load = D.cut_function(dds, re.search(r"^HRESULT LoadFromDDSMemory\s*\(", dds, re.M).start())
        pal_at = load.index("const uint32_t *pal8 = nullptr;")
        palette = load[pal_at:pal_at + len("const uint32_t *pal8 = nullptr;")] + "\n    " + \
            D.cut_function(load, load.index("if ( convFlags & CONV_FLAGS_PAL8 )"))
        copy = D.cut_function(dds, re.search(r"^static HRESULT _CopyImage\s*\(", dds, re.M).start())
        cpflags = D.cut_function(copy, copy.index("if ( convFlags & CONV_FLAGS_EXPAND )"))
        pitch = D.cut_function(util, re.search(r"^void ComputePitch\s*\(", util, re.M).start())
        bpp = U.cut_between(pitch, r"size_t bpp;", "bpp = BitsPerPixel( fmt );")
        cp_enum = U.cut_between(tex_h, r"^\s*enum CP_FLAGS", "};")
        parts = [
            top, dds_h, U.SHIM_MID,
            U.cut_between(texp, r"^\s*enum TEXP_SCANLINE_FLAGS", "};"),
            cp_enum,
            "\nnamespace itw_ref_open_exp {\n",
            U.cut_between(dds, r"^enum CONVERSION_FLAGS", "};"),
            U.cut_between(dds, r"^struct LegacyDDS", "};"),
            U.cut_between(dds, r"^const LegacyDDS g_LegacyDDSMap\[\]", "\n};"),
            D.cut_function(dds, re.search(r"^static DXGI_FORMAT _GetDXGIFormat\s*\(", dds, re.M).start()),
            D.cut_function(dds, re.search(r"^static HRESULT _DecodeDDSHeader\s*\(", dds, re.M).start()),
            U.cut_between(dds, r"^enum TEXP_LEGACY_FORMAT", "};"),
            D.cut_function(dds, re.search(r"^inline static TEXP_LEGACY_FORMAT _FindLegacyFormat\s*\(", dds, re.M).start()),
            D.cut_function(dds, re.search(r"^static bool _LegacyExpandScanline\s*\(", dds, re.M).start()),
            BOTTOM.replace("@BPP@", bpp).replace("@PALETTE@", palette).replace("@CPFLAGS@", cpflags),
        ]
        unit = "\n".join(parts).replace("_Success_(return != false)", "")
        path = os.path.join(tmp, "open_exp_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_open_expanded]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_open_expanded] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
