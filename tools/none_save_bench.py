#!/usr/bin/env python3
"""Time the "none" save (itw_dds_save_none) on the GPU, next to a BC7 `basic` save of the same document.

Cases: a 4096x4096 RGBA8 2-D document with its full chain; the same document as a normal map with NormalizeNormalMapChain; a cube
from six 2048x2048 face layers with the full chain.  Host document, host layers and a host file, as the plug-in passes them.

    wall ms       one call, host operands in and the file out; median of --reps
    kernel ms     the call's kernels (itw_last_kernel_ms): front end / faces, chain, store
    store us      none_store_kernel alone (torch.profiler, one profiled call in a run of its own after the timed ones)
    store GB/s    2 x payload bytes (every texel read once and written once) over the store's time, and that over 3.35 TB/s, the
                  H100 SXM data-sheet HBM3 bandwidth (a kernel bound by memory, so the share of that bound)
    BC7 wall ms   itw_dds_encode_pixels / itw_dds_encode_cube with BC7 (98) `basic` of the same document and options
    parity        the timed file against the oracle of tests/none_lib.py, byte for byte

python tools/none_save_bench.py [--reps 5]     (needs a GPU; prints the card, its power limit and its top SM clock first)
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
HBM_TBS = 3.35


def store_us(fn):
    """Device time of none_store_kernel in one call of `fn`, from torch.profiler's CUDA activities."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.events():
        if "none_store_kernel" in e.name and e.device_type.name == "CUDA":
            total += e.device_time
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import none_lib as N
    import preview_uncompressed_lib as U
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    doc = U.document(4096, 4096, 4, 8, seed=1)
    face = U.document(2048, 2048, 4, 8, seed=2)
    faces = U.cube_layers(2048, 2048, 8, seed=3, channels=(3,) * 6, alpha=(True,) * 6)
    A = B.FRONT_HAS_ALPHA
    cases = [("2-D 4096^2, full chain", B.NoneOptions(B.PANE_2D, 1, -1), doc, None, A),
             ("normal map 4096^2, normalise", B.NoneOptions(B.PANE_2D, 1, -1), doc, None, A | B.FRONT_NORMALIZE),
             ("cube from layers 2048^2, full chain", B.NoneOptions(B.PANE_CUBE_LAYERS, 1, -1), face, faces, A)]
    basic = lib.profile("basic")
    print(f"# {gpu}; medians of {a.reps} calls; HBM bound {HBM_TBS} TB/s (data sheet)")
    print("| case | file MB | wall ms | kernel ms | store us | store GB/s | of HBM | BC7 basic wall ms | parity |")
    print("|---|---|---|---|---|---|---|---|---|")
    for name, o, d, layers, flags in cases:
        n, desc, fw, fh = lib.none_layout(o, d.shape[1], d.shape[0])
        payload = n - 128
        state = {}

        def run():
            state["file"] = lib.dds_save_none(o, d, layers, flags)
            state["kms"] = lib.last_kernel_ms()

        if o.texture == B.PANE_2D:
            bdesc = B.DdsDesc(desc.width, desc.height, desc.mip_levels, 1, 98, 0)
            run_bc7 = lambda: lib.dds_encode_pixels(bdesc, [d], flags, basic)
        else:
            copts = B.CubeOptions(98, B.CUBE_LAYERS, 1, -1)
            run_bc7 = lambda: lib.dds_encode_cube(copts, d, layers, flags, basic)
        run()
        run_bc7()
        tw, tk, tb = [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            run()
            tw.append((time.perf_counter() - t0) * 1e3)
            tk.append(state["kms"])
            t0 = time.perf_counter()
            run_bc7()
            tb.append((time.perf_counter() - t0) * 1e3)
        us = store_us(run)
        gbs = 2 * payload / (us * 1e-6) / 1e9 if us > 0 else float("nan")
        parity = np.array_equal(state["file"], N.oracle_save(o, d, layers, flags)) if N.available() else None
        print(f"| {name} | {n / 1e6:.1f} | {statistics.median(tw):.2f} | {statistics.median(tk):.3f} | {us:.1f} | {gbs:.0f} | "
              f"{gbs / (HBM_TBS * 1e3):.2f} | {statistics.median(tb):.1f} | "
              f"{'equal' if parity else ('not checked' if parity is None else 'DIFFERS')} |", flush=True)


if __name__ == "__main__":
    main()
