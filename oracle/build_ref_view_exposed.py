#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_view_exposed.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

IntelPlugin::FetchPreviewRGB (IntelPlugin.cpp:487-739) with the exposure the plug-in holds.  build_ref_view.py pins itw_preview_view,
whose exposure is 1 (the value InitData sets at every DoWriteStart, :1889 / :1902); once the user moves the dialog's exposure slider
(PreviewDialog.cpp:868-887), ps.data->exposure is float(pow(2, pos * 0.01)) and the float loop multiplies every texel it shows by it
(:649-651).  This recipe cuts the same body as build_ref_view.py, WHERE IT LIES (never copied into the repo): the channel table, with
its reset of the exposure to 1 for the pure-alpha view (:615-621), and the four sampling loops, behind a shim whose only difference is
that `exposure` (a float, as ps.data->exposure is) is an argument:

  ref_fetch_preview_rgb_exposed(dst, width, height, xo, yo, zoom, previewOptions, matteColor, data, srcWidth, srcHeight, planes,
                                depthOrFormat, rowPitch, mipLevel, exposure)

Only the .so is kept (git-ignored; travels to the GPU box).  Used by tests/test_preview_hdr.py and tests/test_preview_hdr_gpu.py.
"""
import os
import shutil
import subprocess
import tempfile

import build_ref_frontend as F          # same reference tree, same shim and cutting helpers
import build_ref_view as V              # the cut of FetchPreviewRGB and PREVIEW_OPTIONS

OUT_DIR = F.OUT_DIR
OUT_SO = os.path.join(OUT_DIR, "libitw_ref_view_exposed.so")

SHIM_BOTTOM_HEAD = r"""
// ---- C entry point: FetchPreviewRGB with the pane or document and the exposure handed in -------------------------------------
extern "C" void ref_fetch_preview_rgb_exposed(unsigned8* dst, int width, int height, int xo, int yo, double zoom, int previewOptions,
                                              int matteColor, const void* data, int srcWidth, int srcHeight, int planes, int depthOrFormat,
                                              int rowPitch, int mipLevel, float exposureIn)
{
    if (!(previewOptions & PREVIEW_CHANNEL_MASK))              // :491-492
        previewOptions |= PREVIEW_CHANNEL_RGB;
    const uint8* pixelData = static_cast<const uint8*>(data);
    auto exposure = exposureIn;                                 // auto exposure = ps.data->exposure, :501 (a float)
    zoom = zoom / (1 << mipLevel);                              // :503-504
"""


def build(verbose=True):
    have_ref = os.path.exists(F.PLUGIN_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO                      # GPU box: prebuilt .so travelled with the snapshot
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {F.REF_ROOT} and no prebuilt {OUT_SO}")
    deps = [__file__, V.__file__, F.__file__, F.PLUGIN_CPP, F.PLUGIN_H]
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in deps):
        return OUT_SO
    os.makedirs(OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_view_exposed_")
    try:
        read = lambda p: open(p, encoding="utf-8", errors="replace").read()
        enum = "enum DXGI_FORMAT { DXGI_FORMAT_R16G16B16A16_FLOAT = 10,"
        if enum not in F.SHIM_TOP:
            raise RuntimeError("build_ref_frontend.SHIM_TOP changed: update the DXGI_FORMAT shim here")
        hdr = read(F.PLUGIN_H)
        unit = (F.SHIM_TOP.replace(enum, "enum DXGI_FORMAT { DXGI_FORMAT_R32G32B32A32_FLOAT = 2, DXGI_FORMAT_R16G16B16A16_FLOAT = 10,")
                + F.cut_inlines(hdr) + "\n" + V.cut_preview_options(hdr) + "\n" + SHIM_BOTTOM_HEAD + V.cut_view(read(F.PLUGIN_CPP)) + "\n")
        if "auto exposure = ps.data->exposure" not in read(F.PLUGIN_CPP):
            raise RuntimeError("FetchPreviewRGB no longer reads ps.data->exposure: update the shim")
        path = os.path.join(tmp, "view_exposed_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-fno-fast-math", "-mfpmath=sse", "-msse2",
               path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_view_exposed]", " ".join(cmd))
        subprocess.check_call(cmd)
        if os.environ.get("ITW_KEEP_REF_TMP"):
            print("[build_ref_view_exposed] kept", tmp)
    finally:
        if not os.environ.get("ITW_KEEP_REF_TMP"):
            shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
