#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_layers.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

The save dialog's "mip maps from layers" option (DoWriteDDS, IntelPlugin.cpp:2093-2145) copies document layers into the mip
levels of the uncompressed scratch image with three member functions of the plug-in:

  IntelCompressionPlugin/IntelPlugin.cpp   FillLayerDataToWhite (:1664-1689), CopyFromLayerChannelIntoImage (:1694-1741),
                                           CopyLayersIntoMipMaps (:1749-1850)
  IntelCompressionPlugin/IntelPlugin.h     the conversion helpers (FloatToByte, ConvertTo8Bit x3, ConvertTo16Bit x3), cut by the
                                           same routine as oracle/build_ref_frontend.py

This recipe cuts those bodies WHERE THEY LIE (never copied into the repo) and compiles them behind a shim into oracle/_ref/
(git-ignored; travels to the GPU box).  The shim supplies, restated because they are Photoshop SDK or DirectXTex:
  * ReadLayerDesc / ReadChannelDesc lists (next, compositeChannelsList, layerMask, transparency); a channel carries a plane
    pointer, its row pitch and its depth;
  * ReadLayerData (:1618-1662) as the copy ReadPixelsFromLevel performs: the top-left width x height rectangle of the channel
    into rows of width * depth bits;
  * sPSBuffer (New / Dispose as malloc / free), SetResult, and a ScratchImage whose image table is handed in by the caller --
    one image for the call that fills level 0, `levels` images for the call that fills the rest, as in DoWriteDDS.
The half conversion is the restated DirectXMath 3.06 one of build_ref_frontend.py.  Used by tests/test_mips_from_layers.py.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_frontend as F          # same reference tree, same shim and cutting helpers

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = F.OUT_DIR
OUT_SO = os.path.join(OUT_DIR, "libitw_ref_layers.so")
MEMBERS = ["FillLayerDataToWhite", "CopyFromLayerChannelIntoImage", "CopyLayersIntoMipMaps"]

SHIM_RECORD = r"""
struct ReadChannelDesc { ReadChannelDesc* next; const char* plane; long long row_bytes; int depth; };
struct ReadLayerDesc { ReadLayerDesc* next; ReadChannelDesc* compositeChannelsList; ReadChannelDesc* layerMask; ReadChannelDesc* transparency; };
struct FakeDocumentInfo { ReadLayerDesc* layersDescriptor; };
struct FakeFormatRecord { int depth; void* data; FakePoint imageSize; int planeBytes; FakeDocumentInfo* documentInfo; };
"""

SHIM_CLASS = r"""
#include <climits>
#include <cstdlib>
#include <vector>
enum { memFullErr = -108, errPlugInHostInsufficient = -30900 };
struct FakeBufferProcs {
    char* New(void*, size_t n) { return static_cast<char*>(malloc(n)); }
    void Dispose(char** p) { free(*p); *p = nullptr; }
};
static FakeBufferProcs g_buffer_procs;
static FakeBufferProcs* sPSBuffer = &g_buffer_procs;
class IntelPlugin {
public:
    FakeGlobals ps;
    void SetResult(int) {}
    // ReadPixelsFromLevel of the rectangle (0, 0)-(width, height) into rows of width * depth bits (IntelPlugin.cpp:1618-1662)
    void ReadLayerData(ReadChannelDesc* pChannel, char* pLayerData, int width, int height)
    {
        const size_t row = (size_t)width * pChannel->depth / 8;
        for (int y = 0; y < height; y++) memcpy(pLayerData + row * y, pChannel->plane + pChannel->row_bytes * y, row);
    }
    void FillLayerDataToWhite(char* pLayerData, int width, int height);
    void CopyFromLayerChannelIntoImage(char* pLayerData, const Image* image, int indexToImage, int indexToLayerChannel);
    void CopyLayersIntoMipMaps(ScratchImage* scrUncompressedImageScratch_, bool hasAlpha_, int startMipIndex, int endMipIndex = INT_MAX);
};
"""

SHIM_BOTTOM = r"""
// ---- C entry point: one CopyLayersIntoMipMaps call of DoWriteDDS ----------------------------------------------------------------
// `images` = image_count tightly packed levels (level l: max(1, doc_w >> l) x max(1, doc_h >> l) RGBA8 / RGBA16F texels), modified in
// place.  Layer i: planes[4 * i + c] for c < channel_count[i] (document-sized, `depth` bits, row pitch row_bytes[i]) and
// planes[4 * i + 3] = its alpha (the transparency channel when mask_slot[i] == 0, the layer mask otherwise) or null.
extern "C" int ref_copy_layers_into_mips(int format, int depth, int doc_w, int doc_h, uint8_t** images, int image_count,
                                         const void* const* planes, const long long* row_bytes, const int* channel_count, const int* mask_slot,
                                         int layer_count, int has_alpha, int start, int end)
{
    if (layer_count <= start) return -1;                 // the plug-in walks `start` layers ahead without a check
    IntelPlugin p;
    std::vector<ReadChannelDesc> ch((size_t)layer_count * 4);
    std::vector<ReadLayerDesc> layers((size_t)layer_count);
    for (int i = 0; i < layer_count; i++) {
        ReadLayerDesc& L = layers[i];
        L = ReadLayerDesc{i + 1 < layer_count ? &layers[i + 1] : nullptr, nullptr, nullptr, nullptr};
        for (int c = 0; c < channel_count[i]; c++) {
            ch[4 * i + c] = ReadChannelDesc{c + 1 < channel_count[i] ? &ch[4 * i + c + 1] : nullptr, static_cast<const char*>(planes[4 * i + c]),
                                            row_bytes[i], depth};
        }
        L.compositeChannelsList = &ch[4 * i];
        if (planes[4 * i + 3]) {
            ch[4 * i + 3] = ReadChannelDesc{nullptr, static_cast<const char*>(planes[4 * i + 3]), row_bytes[i], depth};
            (mask_slot[i] ? L.layerMask : L.transparency) = &ch[4 * i + 3];
        }
    }
    FakeDocumentInfo doc{&layers[0]};
    FakeFormatRecord rec{depth, nullptr, {doc_w, doc_h}, depth / 8, &doc};
    FakeData dat{false, false, format};
    p.ps.formatRecord = &rec;
    p.ps.data = &dat;
    const bool hdr = format == DXGI_FORMAT_BC6H_UF16;
    const size_t texel = hdr ? 8 : 4;
    std::vector<Image> img((size_t)image_count);
    for (int l = 0; l < image_count; l++) {
        const size_t w = std::max(1, doc_w >> l), h = std::max(1, doc_h >> l);
        img[l] = Image{w, h, hdr ? DXGI_FORMAT_R16G16B16A16_FLOAT : DXGI_FORMAT_R8G8B8A8_UNORM, w * texel, w * h * texel, images[l]};
    }
    ScratchImage scratch{img.data(), (size_t)image_count};
    p.CopyLayersIntoMipMaps(&scratch, has_alpha != 0, start, end);
    return 0;
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


def build(verbose=True):
    have_ref = os.path.exists(F.PLUGIN_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {F.REF_ROOT} and no prebuilt {OUT_SO}")
    deps = [__file__, F.__file__, F.PLUGIN_CPP, F.PLUGIN_H]
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in deps):
        return OUT_SO
    os.makedirs(OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_layers_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        record = "struct FakeFormatRecord { int depth; void* data; FakePoint imageSize; };"
        if record not in F.SHIM_TOP:
            raise RuntimeError("build_ref_frontend.SHIM_TOP changed: update the record shim here")
        unit = ("#include <algorithm>\n" + F.SHIM_TOP.replace(record, SHIM_RECORD) + F.cut_inlines(read(F.PLUGIN_H)) + SHIM_CLASS
                + cut_members(read(F.PLUGIN_CPP)) + SHIM_BOTTOM)
        path = os.path.join(tmp, "layers_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-fno-fast-math", "-mfpmath=sse", "-msse2",
               path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_layers]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_layers] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
