#!/usr/bin/env python3
"""Time itw_dds_encode_layers ("mip maps from layers") against itw_dds_encode_pixels on the same document.

A 4096x4096 document with all 13 levels and 13 layers (each layer holds its level in the top-left corner, as the open path's
ITW_OPEN_MIPS layout does), saved as BC7 basic and BC1 at depth 8 with alpha, and as BC6H basic at depth 32.

    device ms   sum of the kernel times of one call (torch.profiler with CUDA activities, a run of its own)
    layer ms    layer_kernel's share of it (level 0, and one launch for levels 1-12)
    e2e ms      host planes in -> DDS file on the host, wall clock, median of --reps calls (profiler off)
    H2D MB      bytes copied to the device, computed from the shapes: the composite (skipped when layer 0 has three
                channels), and per layer only the read rectangle of each plane

    python tools/layers_bench.py [--size 4096] [--reps 5]     (needs a GPU; prints the card and its power limit first)
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
pkg = importlib.import_module("intel-texture-works-plugin_b200")
B = importlib.import_module("intel-texture-works-plugin_b200.binding")


def kernel_ms(fn):
    """(all kernels, layer_kernel) device milliseconds of one call of `fn`."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = layer = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA" or "memcpy" in e.name.lower() or "memset" in e.name.lower():
            continue
        us = e.device_time
        total += us
        if "layer_kernel" in e.name:
            layer += us
    return total / 1e3, layer / 1e3


def wall_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    n = a.size
    levels = n.bit_length()
    rng = np.random.default_rng(1)
    y, x = np.mgrid[0:n, 0:n]
    doc8 = np.clip(np.stack([(x + c * 50) % 256 for c in range(4)], -1) + rng.integers(-8, 9, (n, n, 4)), 0, 255).astype(np.uint8)
    doc32 = (doc8.astype(np.float32) / 255.0) ** 2.2
    print(f"# {gpu}; {n}x{n} document, {levels} levels, {levels} layers; e2e medians of {a.reps} calls")
    print("| encoding | depth | encode_pixels device ms | encode_layers device ms | layer_kernel ms | encode_pixels e2e ms | "
          "encode_layers e2e ms | H2D MB pixels | H2D MB layers |")
    print("|---|---|---|---|---|---|---|---|---|")
    for name, dxgi, prof, doc in (("BC7 basic", 98, "basic", doc8), ("BC1", 71, None, doc8), ("BC6H basic", 95, "bc6h_basic", doc32)):
        d = B.DdsDesc(n, n, levels, 1, dxgi, 0)
        s = lib.profile(prof) if prof else None
        esize = doc.itemsize
        layers = []
        for l in range(levels):                     # level l of a box-filtered chain, top-left in a document-sized layer
            f = 1 << l
            lw = max(1, n >> l)
            small = doc[::f, ::f][:lw, :lw]
            full = np.zeros_like(doc)
            full[:small.shape[0], :small.shape[1]] = small
            layers.append(([np.ascontiguousarray(full[..., c]) for c in range(3)], np.ascontiguousarray(full[..., 3])))
        flags = B.FRONT_HAS_ALPHA
        pix = lambda: lib.dds_encode_pixels(d, [doc], flags, s)
        lay = lambda: lib.dds_encode_layers(d, doc, layers, flags, s)
        pix()
        lay()
        pdev, _ = kernel_ms(pix)
        ldev, lk = kernel_ms(lay)
        pe2e, le2e = wall_ms(pix, a.reps), wall_ms(lay, a.reps)
        h2d_pix = n * n * 4 * esize
        h2d_lay = sum(max(1, n >> l) ** 2 * 4 * esize for l in range(levels))     # 3 channels + alpha per layer, composite skipped
        print(f"| {name} | {esize * 8} | {pdev:.3f} | {ldev:.3f} | {lk:.3f} | {pe2e:.1f} | {le2e:.1f} | {h2d_pix / 1e6:.1f} | "
              f"{h2d_lay / 1e6:.1f} |", flush=True)


if __name__ == "__main__":
    main()
