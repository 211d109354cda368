#!/usr/bin/env python3
"""Time the uncompressed pane (itw_preview_uncompressed) against the plug-in's pipeline on the CPU.

Cases: a 4096x4096 document of the "none" encoding with layer 0 (mip maps from layers) at depths 8 and 32; a cube from layers with
1024^2 faces (the 4096x3072 cross); the same cube with the set level L = 3.

    (a) CPU     GetUncompressedImageForPreview restated over the reference's own bodies (tests/preview_uncompressed_lib.py: the
                converters, CopyLayersIntoMipMaps, ConvertToCubeMapFromLayers and ConvertToHorizontalCrossFromCubeMap, compiled -O2),
                then one FetchPreviewRGB of the reference's loops over the pane
    (b) GPU     itw_preview_uncompressed into a device display, then one itw_preview_view of it into a host 1200 x 900 x 3 buffer

    wall ms     one call of each path (pane + one repaint), host operands; medians of --reps, the two paths alternated
    kernel ms   the call's kernels alone (itw_last_kernel_ms)
    parity      the device pane and the dialog buffer of (b) against (a), byte for byte

python tools/preview_uncompressed_bench.py [--reps 7]     (needs a GPU; prints the card and its power limit first)
"""
import argparse
import ctypes
import importlib
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("intel-texture-works-plugin_b200")
B = importlib.import_module("intel-texture-works-plugin_b200.binding")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    import preview_uncompressed_lib as U
    import test_preview_view as V
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    if not U.available() or V.ref_view() is None:
        raise SystemExit("oracle/_ref is missing: run the build first")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    vw, vh = 1200, 900
    zoom = float(np.float32(1) / np.float32(0.3))
    cases = []
    for depth in (8, 32):
        doc = U.document(4096, 4096, 4, depth, seed=depth)
        cases.append((f"2-D none + layer 0, depth {depth}", 28, B.PANE_2D, -1, doc, U.layer(4096, 4096, depth, 3, True, seed=depth + 1),
                      B.FRONT_HAS_ALPHA))
    face = U.document(1024, 1024, 4, 8, seed=5)
    layers = U.cube_layers(1024, 1024, 8, seed=6, channels=(3,) * 6, alpha=(True,) * 6)
    cases.append(("cube from layers 1024^2", 28, B.PANE_CUBE_LAYERS, -1, face, layers, B.FRONT_HAS_ALPHA))
    cases.append(("cube from layers 1024^2, L = 3", 28, B.PANE_CUBE_LAYERS, 3, face, layers, B.FRONT_HAS_ALPHA))
    print(f"# {gpu}; {vw}x{vh} view at zoom {zoom:.6f}; medians of {a.reps} calls per path, alternated")
    print("| case | pane | (a) CPU wall ms | (b) GPU wall ms | (b) kernel ms | parity |")
    print("|---|---|---|---|---|---|")
    for name, fmt, texture, level, doc, lay, flags in cases:
        dh, dw = doc.shape[:2]
        w, h = U.pane_size(texture, level, dw, dh)
        keep = []
        arr = lib.cube_faces([lay] if texture == B.PANE_2D else lay, doc.dtype, keep)
        src = B.PixelSource(doc.ctypes.data, dw, dh, 4, doc.itemsize * 8, 0)
        opts = B.PaneOptions(fmt, texture, level)
        disp = torch.zeros((h, w * 4), dtype=torch.uint8, device="cuda")
        surf = B.RgbaSurface(disp.data_ptr(), w, h, w * 4)
        ps = B.PixelSource(disp.data_ptr(), w, h, 4, 8, w * 4)
        view = B.View(vw, vh, 100, 50, zoom, 0, 0, 0)
        out_a = np.zeros((vh, vw, 3), np.uint8)
        out_b = np.zeros((vh, vw, 3), np.uint8)
        state = {}

        def run_a():
            pane = np.ascontiguousarray(U.oracle_pane(fmt, texture, level, doc, lay, flags)[0])
            V.ref_view().ref_fetch_preview_rgb(out_a.ctypes.data, vw, vh, 100, 50, zoom, 0, 0, pane.ctypes.data, w, h, 4, 28, w * 4, 0)
            state["pane"] = pane

        def run_b():
            assert lib.preview_uncompressed_raw(opts, src, arr, flags, surf, None) == 0, lib.last_error()
            state["kms"] = lib.last_kernel_ms()
            assert lib.preview_view_raw(ps, view, out_b.ctypes.data) == 0, lib.last_error()
        run_a()
        run_b()
        ta, tb, kb = [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            run_a()
            ta.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            run_b()
            tb.append((time.perf_counter() - t0) * 1e3)
            kb.append(state["kms"])
        parity = np.array_equal(disp.cpu().numpy().reshape(h, w, 4), state["pane"]) and np.array_equal(out_a, out_b)
        print(f"| {name} | {w}x{h} | {statistics.median(ta):.1f} | {statistics.median(tb):.2f} | {statistics.median(kb):.3f} | "
              f"{'equal' if parity else 'DIFFERS'} |", flush=True)


if __name__ == "__main__":
    main()
