#!/usr/bin/env python3
"""Time the options dialog's compressed pane with the pane on the host against the pane on the device.

Workload: a 4096x4096 document, BC7 basic at depth 8 with alpha and BC6H basic at depth 32 (the same picture), viewed through a
1200x900 dialog buffer at zoom 1.f / 0.3f, panned over the pane (the offset changes on every repaint).  The two paths alternate in
one process.

    (a) host pane     itw_preview_pixels into host memory (what a host that runs FetchPreviewRGB itself must do), then every repaint
                      runs FetchPreviewRGB's loops -- the reference's own, cut by oracle/build_ref_view.py and compiled -O2 -- on the CPU
    (b) device pane   itw_preview_pixels into a device display that stays there, then every repaint is one itw_preview_view into a
                      host buffer of 1200 x 900 x 3 bytes

    change ms   a settings change: the pane rebuilt (front end, encode, display decompress, and for (a) the copy of the pane to the host)
    repaint ms  one repaint of the pane, dialog buffer on the host; wall clock
    view ms     view_kernel alone: CUDA events around the launch (itw_last_kernel_ms)
    parity      every repaint's bytes of (b) against (a)

Medians of --reps calls.  python tools/preview_view_bench.py [--reps 20]     (needs a GPU; prints the card and its power limit first)
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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--size", type=int, default=4096)
    a = ap.parse_args()
    import torch
    import test_preview_view as V
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    ref = V.ref_view()
    if ref is None:
        raise SystemExit("oracle/_ref/libitw_ref_view.so is missing: run the build first")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    n = a.size
    vw, vh = 1200, 900
    zoom = float(np.float32(1) / np.float32(0.3))
    rng = np.random.default_rng(1)
    y, x = np.mgrid[0:n, 0:n]
    doc8 = np.clip(np.stack([(x // 3 + y // 5 + c * 50) % 256 for c in range(4)], -1) + rng.integers(-8, 9, (n, n, 4)), 0, 255).astype(np.uint8)
    doc32 = np.ascontiguousarray((doc8.astype(np.float32) / 255.0) ** 2.2 * 4.0)
    print(f"# {gpu}; {n}x{n} document, {vw}x{vh} view at zoom {zoom:.6f}; medians of {a.reps} calls per path, alternated")
    print("| encoding | pane | (a) change ms | (b) change ms | (a) repaint ms | (b) repaint ms | (b) view ms | parity |")
    print("|---|---|---|---|---|---|---|---|")
    for name, fmt, prof, doc in (("BC7 basic", 98, "basic", doc8), ("BC6H basic", 95, "bc6h_basic", doc32)):
        s = lib.profile(prof)
        hdr = doc.dtype == np.float32 and fmt == 95
        texel = 16 if hdr else 4
        pane_depth, target = (32, 2) if hdr else (8, 28)
        srcs = (B.PixelSource * 1)(B.PixelSource(doc.ctypes.data, n, n, 4, doc.itemsize * 8, 0))
        host_pane = np.zeros((n, n * texel), np.uint8)
        dev_pane = torch.zeros((n, n * texel), dtype=torch.uint8, device="cuda")
        out_a = np.zeros((vh, vw, 3), np.uint8)
        out_b = np.zeros((vh, vw, 3), np.uint8)

        def change_a():
            lib.preview_pixels_raw(fmt, srcs, 1, B.FRONT_HAS_ALPHA, s, host_pane.ctypes.data, n, n, n * texel)

        def change_b():
            lib.preview_pixels_raw(fmt, srcs, 1, B.FRONT_HAS_ALPHA, s, dev_pane.data_ptr(), n, n, n * texel)

        def repaint_a(ox, oy):
            ref.ref_fetch_preview_rgb(out_a.ctypes.data, vw, vh, ox, oy, zoom, 0, 0, host_pane.ctypes.data, n, n, 4, target, n * texel, 0)

        view = B.View(vw, vh, 0, 0, zoom, 0, 0, 0)
        ps = B.PixelSource(dev_pane.data_ptr(), n, n, 4, pane_depth, n * texel)

        def repaint_b(ox, oy):
            view.x, view.y = ox, oy
            assert lib.preview_view_raw(ps, view, out_b.ctypes.data) == 0, lib.last_error()
        change_a()
        change_b()
        repaint_a(0, 0)
        repaint_b(0, 0)
        ta, tb, ra, rb, kb = [], [], [], [], []
        parity = True
        for i in range(a.reps):
            t0 = time.perf_counter()
            change_a()
            ta.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            change_b()
            tb.append((time.perf_counter() - t0) * 1e3)
        for i in range(a.reps):
            ox, oy = 37 * i - 100, 23 * i - 50                        # panning, past the top-left corner at first
            t0 = time.perf_counter()
            repaint_a(ox, oy)
            ra.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            repaint_b(ox, oy)
            rb.append((time.perf_counter() - t0) * 1e3)
            kb.append(lib.last_kernel_ms())
            parity = parity and np.array_equal(out_a, out_b)
        panes_equal = np.array_equal(host_pane, dev_pane.cpu().numpy())
        verdict = ("equal" if parity else "DIFFERS") + (", panes equal" if panes_equal else ", panes DIFFER")
        print(f"| {name} | {'R32G32B32A32_FLOAT' if hdr else 'R8G8B8A8_UNORM'} {n * n * texel / 2**20:.0f} MiB | {statistics.median(ta):.1f} | "
              f"{statistics.median(tb):.1f} | {statistics.median(ra):.2f} | {statistics.median(rb):.3f} | {statistics.median(kb):.4f} | {verdict} |",
              flush=True)


if __name__ == "__main__":
    main()
