#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_open_other_bc.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

What DoReadStart (IntelPlugin.cpp:2461-2560) does with the block-compressed files itw_dds_open does not serve -- BC2 (DXT2 / DXT3),
DXT4, BC4 / BC5 SNORM and the typeless BC formats: the alpha check, then DirectX::Decompress into the target.

  3rdParty/DirectXTex/DirectXTex/BC.h                    struct D3DX_BC1 / D3DX_BC2 / D3DX_BC3 (:280-302)
  3rdParty/DirectXTex/DirectXTex/BC.cpp                  DecodeBC1 (:322-370) and D3DXDecodeBC2 (:794-817)
  3rdParty/DirectXTex/DirectXTex/BC4BC5.cpp              struct BC4_SNORM (:98-154), D3DXDecodeBC4S and D3DXDecodeBC5S
  3rdParty/DirectXTex/DirectXTex/DirectXTexCompress.cpp  _DecompressBC (:358-468) and _IsAlphaAllOpaqueBC (:472-554), whole, this time
                                                         linked to the real BC2 / BC4S / BC5S decoders
  3rdParty/DirectXTex/DirectXTex/DirectXTexConvert.cpp   _ConvertScanline, its table rows and sRGB helpers, through build_ref_preview.py;
                                                         the STORE_SCANLINE macro and _StoreScanline's R16G16B16A16_UNORM case, through
                                                         build_ref_open_converted.py
  3rdParty/DirectXTex/DirectXTex/DirectXTexImage.cpp     the compressed branch of ScratchImage::IsAlphaAllOpaque, through build_ref_open.py
  and, in a second translation unit, build_ref_open_converted.py's: BitsPerColor, IsSRGB and HasAlpha (with _UseWICConversion).

NOT cut, restated in the shim below, and why (ASSUMED, DESIGN section 2):
  * DirectXMath: XMLoadU565, XMVectorLerp ("(V1 - V0) * t + V0", a multiply then an add), XMVectorZero and XMVectorSetW as
    build_ref_frontend.py restates them; XMStoreUShortN4 and the byte store as build_ref_open_converted.py / build_ref_preview.py do.
  * D3DXDecodeBC1 / BC3 / BC4U / BC6HU / BC7 are the reference bodies of libitw_ref_frontend.so / libitw_ref_decode.so; D3DXDecodeBC5U
    is build_ref_preview.py's BC4U of each half.
  * BitsPerPixel of the three targets (2: 128, 11: 64, 28 / 29: 32) and the ScratchImage image table (item-major, mip-minor images of
    max(1, w >> l) x max(1, h >> l) texels, rows of ceil(w / 4) blocks).
Only the .so is kept (git-ignored; travels to the GPU box).  Used by tests/test_dds_open_other_bc.py and its GPU twin.
"""
import os
import shutil
import subprocess
import tempfile

import build_ref_preview as P             # _ConvertScanline, its table and sRGB helpers, the preview shim and its decoder wrappers
import build_ref_open as O                # the compressed branch of IsAlphaAllOpaque
import build_ref_open_converted as C       # the R16G16B16A16_UNORM store, the DirectXMath restatements, the scope unit

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_SO = os.path.join(P.OUT_DIR, "libitw_ref_open_other_bc.so")
BC_H = os.path.join(P.DXTEX, "BC.h")
BC_CPP = os.path.join(P.DXTEX, "BC.cpp")
BC45_CPP = os.path.join(P.DXTEX, "BC4BC5.cpp")

SHIM_DECODERS = r"""
// ---- what the cut decoders need from DirectXMath (restated, see the recipe's header) ----
#define _Out_writes_(n)
#define NUM_PIXELS_PER_BLOCK 16
struct XMU565 { uint16_t v; };
static inline XMVECTOR XMLoadU565(const XMU565* p) { return XMVECTOR{{(float)(p->v & 31), (float)((p->v >> 5) & 63), (float)((p->v >> 11) & 31), 0.0f}}; }
static inline XMVECTOR XMVectorLerp(XMVECTOR v0, XMVECTOR v1, float t)
{
    XMVECTOR r;
    for (int i = 0; i < 4; i++) { float l = v1.f[i] - v0.f[i]; float m = l * t; r.f[i] = m + v0.f[i]; }
    return r;
}
static inline XMVECTOR XMVectorZero() { return XMVECTOR{{0.0f, 0.0f, 0.0f, 0.0f}}; }
static inline XMVECTOR XMVectorSetW(XMVECTOR v, float w) { v.f[3] = w; return v; }
static inline bool XMVector4Less(XMVECTOR a, const XMVECTORF32& b)
{
    return a.f[0] < b.f[0] && a.f[1] < b.f[1] && a.f[2] < b.f[2] && a.f[3] < b.f[3];
}
"""

SHIM_STORE = r"""
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
static size_t bits_per_pixel(DXGI_FORMAT f) { return f == DXGI_FORMAT_R32G32B32A32_FLOAT ? 128 : f == DXGI_FORMAT_R16G16B16A16_UNORM ? 64 : 32; }
#define _StoreScanline store_target
#define BitsPerPixel bits_per_pixel
"""

BOTTOM = r"""
#undef _StoreScanline
#undef BitsPerPixel
static bool IsCompressed(DXGI_FORMAT) { return true; }      // every format this library is handed is block-compressed
static size_t block_bytes(DXGI_FORMAT f)
{
    return (f == DXGI_FORMAT_BC1_TYPELESS || f == DXGI_FORMAT_BC1_UNORM || f == DXGI_FORMAT_BC1_UNORM_SRGB || f == DXGI_FORMAT_BC4_TYPELESS ||
            f == DXGI_FORMAT_BC4_UNORM || f == DXGI_FORMAT_BC4_SNORM) ? 8 : 16;
}
}  // namespace itw_ref_preview
using namespace itw_ref_preview;
extern "C" int ref_has_alpha(uint32_t f);          // the scope unit's cut HasAlpha
namespace itw_ref_preview {
// ScratchImage::IsAlphaAllOpaque for a block-compressed texture: HasAlpha, the image table restated, the compressed branch cut
static bool IsAlphaAllOpaque(DXGI_FORMAT format, const uint8_t* payload, size_t w, size_t h, size_t mips, size_t items)
{
    const size_t bpb = block_bytes(format);
    std::vector<Image> _image;
    for (size_t item = 0; item < items; item++)
        for (size_t l = 0; l < mips; l++) {
            const size_t lw = std::max<size_t>(1, w >> l), lh = std::max<size_t>(1, h >> l), pitch = (lw + 3) / 4 * bpb;
            const size_t slice = pitch * ((lh + 3) / 4);
            _image.push_back(Image{lw, lh, format, pitch, slice, const_cast<uint8_t*>(payload)});
            payload += slice;
        }
    const size_t _nimages = _image.size();
    if (!ref_has_alpha((uint32_t)format))
        return true;
@BRANCH@
    return true;
}
}  // namespace itw_ref_preview

// DirectX::Decompress of one image: `blocks` of a w x h `source` image -> `dst` (tight rows of `target` texels)
extern "C" int ref_obc_decompress(int source, const uint8_t* blocks, int w, int h, int target, uint8_t* dst)
{
    const size_t bpb = block_bytes((DXGI_FORMAT)source);
    Image c{(size_t)w, (size_t)h, (DXGI_FORMAT)source, (size_t)((w + 3) / 4) * bpb, 0, const_cast<uint8_t*>(blocks)};
    const size_t texel = target == 2 ? 16 : target == 11 ? 8 : 4;
    Image r{(size_t)w, (size_t)h, (DXGI_FORMAT)target, (size_t)w * texel, (size_t)w * h * texel, dst};
    return (int)_DecompressBC(c, r);
}
// _IsAlphaAllOpaqueBC of `n` one-block images of cols x rows texels (1..4 each): out[i] = 1 if block i is opaque
extern "C" void ref_obc_blocks_opaque(int format, const uint8_t* blocks, long long n, int cols, int rows, uint8_t* out)
{
    const size_t bpb = block_bytes((DXGI_FORMAT)format);
    for (long long i = 0; i < n; i++) {
        Image im{(size_t)cols, (size_t)rows, (DXGI_FORMAT)format, bpb, bpb, const_cast<uint8_t*>(blocks + i * bpb)};
        out[i] = _IsAlphaAllOpaqueBC(im) ? 1 : 0;
    }
}
// 1 if every texel of every image (item-major, mip-minor, tightly packed in `payload`) is opaque, else 0
extern "C" int ref_obc_is_alpha_all_opaque(int format, const uint8_t* payload, int w, int h, int mips, int items)
{
    return IsAlphaAllOpaque((DXGI_FORMAT)format, payload, (size_t)w, (size_t)h, (size_t)mips, (size_t)items) ? 1 : 0;
}
"""


def cut_decoders(bch, bc, bc45):
    a = bch.index("#pragma pack(push,1)")
    structs = bch[a:bch.index("#pragma pack(pop)", a)] + "#pragma pack(pop)\n"
    snorm = bc45.index("struct BC4_SNORM")
    out = [structs, P.cut_function(bc45, snorm) + ";"]
    for src, pat in ((bc, r"^inline static void DecodeBC1\s*\("), (bc, r"^void D3DXDecodeBC2\s*\("),
                     (bc45, r"^void D3DXDecodeBC4S\s*\("), (bc45, r"^void D3DXDecodeBC5S\s*\(")):
        out.append(P.cut_named(src, pat))
    return "\n\n".join(out)


def build(verbose=True):
    have_ref = os.path.exists(P.COMPRESS_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {P.REF_ROOT} and no prebuilt {OUT_SO}")
    deps = [os.path.join(P.OUT_DIR, n) for n in ("libitw_ref_frontend.so", "libitw_ref_decode.so")]
    for d in deps:
        if not os.path.exists(d):
            raise FileNotFoundError(f"{d} is built by build_ref_frontend.py / build_ref_decode.py first")
    srcs = [__file__, P.__file__, O.__file__, C.__file__, P.COMPRESS_CPP, P.CONVERT_CPP, BC_H, BC_CPP, BC45_CPP, C.IMAGE_CPP, C.UTIL_CPP,
            C.TEX_INL] + deps
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in srcs):
        return OUT_SO
    tmp = tempfile.mkdtemp(prefix="itw_ref_open_obc_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        conv, comp = read(P.CONVERT_CPP), read(P.COMPRESS_CPP)
        macro16, case16 = C.cut_store16(conv)
        top = (P.SHIM_TOP.replace("@FORMATS@", ", ".join(f"DXGI_FORMAT_{n} = {v}" for n, v in C.FORMATS.items()))
               .replace("@ENUMS@", P.cut_enums(read(P.TEXP_H), read(P.TEX_H)))
               .replace("@TABLE@", C.cut_table(conv))
               .replace("@SRGB@", P.cut_grayscale(conv) + P.cut_srgb(conv))
               .replace("@CONVERT_BODY@", P.cut_convert_body(conv))
               .replace("#include <cstring>", "#include <cstring>\n#include <vector>"))
        unit = (top + C.SHIM_LOAD + SHIM_DECODERS + cut_decoders(read(BC_H), read(BC_CPP), read(BC45_CPP))
                + "\n" + macro16 + SHIM_STORE.replace("@STORE16@", case16)
                + P.cut_named(comp, r"^static HRESULT _DecompressBC\s*\(") + "\n"
                + P.cut_named(comp, r"^bool _IsAlphaAllOpaqueBC\s*\(") + "\n"
                + BOTTOM.replace("@BRANCH@", O.cut_branch(read(C.IMAGE_CPP))))
        path = os.path.join(tmp, "open_obc_ref.cpp")
        open(path, "w").write(unit)
        scope = os.path.join(tmp, "open_obc_scope_ref.cpp")
        open(scope, "w").write(C.wic_unit(conv, read(C.UTIL_CPP), read(C.TEX_INL), read(P.TEX_H)))
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-fno-fast-math", "-mfpmath=sse", "-msse2",
               path, scope, "-o", OUT_SO, "-L" + P.OUT_DIR] + ["-l:" + os.path.basename(d) for d in deps] + ["-Wl,-rpath,$ORIGIN"]
        if verbose:
            print("[build_ref_open_other_bc]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_open_other_bc] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
