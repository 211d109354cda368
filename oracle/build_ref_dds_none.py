#!/usr/bin/env python3
"""Build oracle/_ref/libitw_ref_dds_none.so FROM THE REFERENCE'S OWN SOURCES (test infrastructure only).

The header of the "none" save (R8G8B8A8_UNORM, include/itw_bcn.h section 12) is pinned against the same _EncodeDDSHeader
(DirectXTexDDS.cpp:441-675) as the block-compressed files.  This recipe is build_ref_dds.py's cut and shim with one addition: the
shim's ComputePitch also knows R8G8B8A8_UNORM (the default branch of DirectXTexUtil.cpp:601: rows of 4 * w bytes, slices of 4 * w * h), which
IsCompressed already reports as uncompressed.  The block-compressed formats go through build_ref_dds.py's ComputePitch unchanged.
Output: oracle/_ref/ (git-ignored; travels to the GPU box).
"""
import os
import re
import shutil
import subprocess
import tempfile

import build_ref_dds as D

OUT_SO = os.path.join(D.OUT_DIR, "libitw_ref_dds_none.so")

PITCH_RGBA8 = r"""
static void ComputePitch(DXGI_FORMAT f, size_t w, size_t h, size_t& rowPitch, size_t& slicePitch, DWORD flags)
{
    if (f == DXGI_FORMAT_R8G8B8A8_UNORM) {          // 32 bits per texel
        rowPitch = (w * 32 + 7) / 8;
        slicePitch = rowPitch * h;
        return;
    }
    ComputePitchBC(f, w, h, rowPitch, slicePitch, flags);
}
"""


def build(verbose=True):
    have_ref = os.path.exists(D.DDS_CPP)
    if os.path.exists(OUT_SO) and not have_ref:
        return OUT_SO
    if not have_ref:
        raise FileNotFoundError(f"reference not present at {D.REF_ROOT} and no prebuilt {OUT_SO}")
    deps = (__file__, D.__file__, D.DDS_CPP)
    if os.path.exists(OUT_SO) and os.path.getmtime(OUT_SO) > max(os.path.getmtime(p) for p in deps):
        return OUT_SO
    os.makedirs(D.OUT_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="itw_ref_dds_none_")
    try:
        cpp = open(D.DDS_CPP, encoding="utf-8", errors="replace").read()
        hdr = open(D.DDS_H, encoding="utf-8", errors="replace").read()
        dds_h = hdr[hdr.index("namespace DirectX"):hdr.rindex("}; // namespace")] + "}  // namespace DirectX\n"
        m = re.search(r"^HRESULT _EncodeDDSHeader\s*\(", cpp, re.M)
        if not m:
            raise RuntimeError("_EncodeDDSHeader not found in the reference")
        mid = D.SHIM_MID.replace("static void ComputePitch(", "static void ComputePitchBC(")
        assert mid != D.SHIM_MID
        enum = ",\n".join(f"    DXGI_FORMAT_{name} = {i}" for i, name in enumerate(D.DXGI))
        unit = D.SHIM_TOP.replace("@DXGI@", enum) + dds_h + mid + PITCH_RGBA8 + D.cut_function(cpp, m.start()) + D.SHIM_BOTTOM
        path = os.path.join(tmp, "dds_none_ref.cpp")
        open(path, "w").write(unit)
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", path, "-o", OUT_SO]
        if verbose:
            print("[build_ref_dds_none]", " ".join(cmd))
        subprocess.check_call(cmd)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return OUT_SO


if __name__ == "__main__":
    print(build())
