#!/usr/bin/env python3
"""Time the preview dialog for HDR documents (include/itw_bcn.h section 18) on the GPU, against the reference pipeline on the CPU.

Cases, each checked byte for byte against its oracle (tests/preview_hdr_lib.py) before it is timed:
  repaint    one exposure repaint: itw_preview_view_exposed of a 4096 x 4096 x 4 32-bit document (device) into a 1200 x 900 dialog
             buffer (device), zoom 1/4, exposure 2^1.5
  cross      itw_preview_uncompressed_hdr of a 4096 x 3072 x 4 32-bit cross with level 0 set: 1024^2 faces, the 4096 x 3072 RGBA16F
             cross, then its conversion into a device display
  layer 0    itw_preview_uncompressed_hdr of a 4096 x 4096 x 4 32-bit document with a 3-channel layer 0 with alpha (all device)

    call ms    host clock around the synchronous call (median of --reps after one warm-up)
    kernel ms  CUDA events around the call's kernels: itw_last_kernel_ms for the panes, torch events around the repaint
    CPU ms     the reference pipeline on one CPU core (one run): FetchPreviewRGB, or the glue of the pane oracle

python tools/preview_hdr_bench.py [--reps 10]     (needs a GPU; prints the card, its power limit and its top SM clock first)
"""
import argparse
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


def timed(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t) * 1e3)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    import hdr_corpus as HC
    import preview_hdr_lib as H
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"# {gpu}; medians of {a.reps} runs after one warm-up")
    print("| case | call ms | kernel ms | CPU ms (reference) | parity |")
    print("|---|---|---|---|---|")

    # repaint
    doc = np.tile(HC.family_planes("exposure_ramp", 512, 512), (8, 8, 1))
    d_doc = torch.from_numpy(doc).cuda()
    src = B.PixelSource(d_doc.data_ptr(), 4096, 4096, 4, 32, 0)
    view = B.View(1200, 900, 100, 50, 4.0, 0, 0, 0x808080)
    e = float(np.float32(2.0 ** 1.5))
    out = torch.zeros((900, 1200, 3), dtype=torch.uint8, device="cuda")
    call = lambda: lib.preview_view_exposed_raw(src, view, e, out.data_ptr())
    assert call() == 0, lib.last_error()
    t = time.perf_counter()
    want = H.ref_fetch(doc, 4096 * 16, 4096, 4096, 4, 32, 1200, 900, 100, 50, 4.0, 0, 0, 0x808080, e)
    cpu = (time.perf_counter() - t) * 1e3
    parity = np.array_equal(out.cpu().numpy(), want)
    ms = timed(call, a.reps)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ks = []
    for _ in range(a.reps):
        ev0.record()
        call()
        ev1.record()
        ev1.synchronize()
        ks.append(ev0.elapsed_time(ev1))
    print(f"| repaint 4096^2 -> 1200 x 900 | {ms:.3f} | {statistics.median(ks):.3f} | {cpu:.0f} | {parity} |", flush=True)

    # the two panes
    cross = np.tile(HC.family_planes("log_uniform", 384, 512), (8, 8, 1))
    layer0 = ([doc[..., 2].copy(), doc[..., 1].copy(), doc[..., 0].copy()], doc[..., 3].copy())
    for name, texture, level, d, layers, w, h in (("cross 4096 x 3072, level 0", B.PANE_CUBE_CROSS, 0, cross, None, 4096, 3072),
                                                 ("4096^2 with layer 0", B.PANE_2D, -1, doc, layer0, 4096, 4096)):
        keep = []
        dd = torch.from_numpy(d).cuda()
        s = B.PixelSource(dd.data_ptr(), d.shape[1], d.shape[0], 4, 32, 0)
        arr = None
        if layers is not None:
            arr = (B.LayerSource * 6)()
            arr[0].channel_count = 3
            for c, pl in enumerate(layers[0]):
                t_ = torch.from_numpy(pl).cuda()
                keep.append(t_)
                arr[0].channels[c] = t_.data_ptr()
            t_ = torch.from_numpy(layers[1]).cuda()
            keep.append(t_)
            arr[0].alpha = t_.data_ptr()
        disp = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        o = B.PaneOptions(95, texture, level)
        call = lambda: lib.preview_uncompressed_hdr_raw(o, s, arr, B.FRONT_HAS_ALPHA, B.RgbaSurface(disp.data_ptr(), w, h, w * 4))
        assert call() == 0, lib.last_error()
        t = time.perf_counter()
        want = H.oracle_pane(texture, level, d, layers, B.FRONT_HAS_ALPHA)
        cpu = (time.perf_counter() - t) * 1e3
        parity = np.array_equal(disp.cpu().numpy(), want)
        ms = timed(call, a.reps)
        ks = []
        for _ in range(a.reps):
            call()
            ks.append(lib.last_kernel_ms())
        print(f"| {name} | {ms:.3f} | {statistics.median(ks):.3f} | {cpu:.0f} | {parity} |", flush=True)


if __name__ == "__main__":
    main()
