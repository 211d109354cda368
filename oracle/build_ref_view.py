#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_view.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

The options dialog shows each pane through IntelPlugin::FetchPreviewRGB (IntelPlugin.cpp:487-739), called twice per repaint by
PreviewDialog::updatePreviewBuffer (PreviewDialog.cpp:260-274).  This recipe cuts, WHERE THEY LIE (never copied into the repo):

  IntelCompressionPlugin/IntelPlugin.cpp   FetchPreviewRGB from its channel table to its end (:585-739): the table and the four
                                           sampling loops (float / R16G16B16A16_FLOAT / 16-bit / byte)
  IntelCompressionPlugin/IntelPlugin.h     enum PREVIEW_OPTIONS, and the conversion helpers (F16toF32, FloatToByte, ConvertTo8Bit x3)
                                           by the same routine as oracle/build_ref_frontend.py

and compiles them behind a shim into oracle/_ref/ (git-ignored; travels to the GPU box).  The shim stands for `ps` and `preview`: the
caller passes what the head of FetchPreviewRGB (:489-583) reads from the format record or the pane -- planes, size, depth or DXGI
format, row pitch, pixels -- and the mip level of :503.  It restates :491-492 (no channel bit means RGB), :501 (exposure, which
InitData sets to 1 at :1889 and nothing changes) and :503-504 (zoom / (1 << mip level)).  The half conversion is the restated
DirectXMath 3.06 one of build_ref_frontend.py.  Used by tests/test_preview_view.py, tests/test_preview_view_gpu.py and
tools/preview_view_bench.py.
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_frontend as F          # same reference tree, same shim and cutting helpers

OUT_DIR = F.OUT_DIR
OUT_SO = os.path.join(OUT_DIR, "libitw_ref_view.so")

SHIM_BOTTOM_HEAD = r"""
// ---- C entry point: FetchPreviewRGB with the pane or document handed in ------------------------------------------------------
extern "C" void ref_fetch_preview_rgb(unsigned8* dst, int width, int height, int xo, int yo, double zoom, int previewOptions, int matteColor,
                                      const void* data, int srcWidth, int srcHeight, int planes, int depthOrFormat, int rowPitch, int mipLevel)
{
    if (!(previewOptions & PREVIEW_CHANNEL_MASK))              // :491-492
        previewOptions |= PREVIEW_CHANNEL_RGB;
    const uint8* pixelData = static_cast<const uint8*>(data);
    float exposure = 1;                                         // ps.data->exposure, :501
    zoom = zoom / (1 << mipLevel);                              // :503-504
"""


def cut_view(cpp):
    m = re.search(r"^[A-Za-z_][\w \t\*&:]*\bIntelPlugin::FetchPreviewRGB\s*\(", cpp, re.M)
    if not m:
        raise RuntimeError("IntelPlugin::FetchPreviewRGB not found in the reference")
    body = F.cut_function(cpp, m.start())
    a = body.find("int channelIndex[4]")
    if a < 0:
        raise RuntimeError("FetchPreviewRGB's channel table not found")
    return body[a:]                                             # through the function's closing brace


def cut_preview_options(hdr):
    m = re.search(r"enum\s+PREVIEW_OPTIONS\s*\{[^}]*\};", hdr)
    if not m:
        raise RuntimeError("enum PREVIEW_OPTIONS not found in IntelPlugin.h")
    return m.group(0)


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
    tmp = tempfile.mkdtemp(prefix="itw_ref_view_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        enum = "enum DXGI_FORMAT { DXGI_FORMAT_R16G16B16A16_FLOAT = 10,"
        if enum not in F.SHIM_TOP:
            raise RuntimeError("build_ref_frontend.SHIM_TOP changed: update the DXGI_FORMAT shim here")
        hdr = read(F.PLUGIN_H)
        unit = (F.SHIM_TOP.replace(enum, "enum DXGI_FORMAT { DXGI_FORMAT_R32G32B32A32_FLOAT = 2, DXGI_FORMAT_R16G16B16A16_FLOAT = 10,")
                + F.cut_inlines(hdr) + "\n" + cut_preview_options(hdr) + "\n" + SHIM_BOTTOM_HEAD + cut_view(read(F.PLUGIN_CPP)) + "\n")
        path = os.path.join(tmp, "view_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-fno-fast-math", "-mfpmath=sse", "-msse2",
               path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_view]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_view] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
