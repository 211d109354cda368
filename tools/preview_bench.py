#!/usr/bin/env python3
"""Time the preview path on the GPU: itw_preview_pixels (planes -> display, one call, nothing leaves the device in between) against
the two-call composition a host makes otherwise (itw_encode_pixels to host memory + itw_decode), and the display kernel alone
(itw_decompress on device operands, CUDA events, median of repeated runs) against the 3.35 TB/s HBM3 bound of the H100 SXM.

    python tools/preview_bench.py [--size 4096] [--reps 10]     (prints one table; needs a GPU)
"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import importlib  # noqa: E402

pkg = importlib.import_module("intel-texture-works-plugin_b200")
B = importlib.import_module("intel-texture-works-plugin_b200.binding")
HBM = 3.35e12


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    n = a.size
    rng = np.random.default_rng(1)
    y, x = np.mgrid[0:n, 0:n]
    doc8 = np.clip(np.stack([(x + c * 50) % 256 for c in range(4)], -1) + rng.integers(-8, 9, (n, n, 4)), 0, 255).astype(np.uint8)
    doc16 = (doc8[..., :3].astype(np.uint32) * 32768 // 255).astype(np.uint16)
    cases = [("BC7 basic", 98, "basic", doc8, B.FRONT_HAS_ALPHA), ("BC7 slow", 98, "slow", doc8, B.FRONT_HAS_ALPHA),
             ("BC1", 71, None, doc8, B.FRONT_HAS_ALPHA), ("BC6H basic (16-bit)", 95, "bc6h_basic", doc16, 0)]
    print(f"# {gpu}; {n}x{n} document; medians of {a.reps} runs")
    print("| case | preview_pixels ms | encode_pixels + decode ms | display kernel ms | display GB/s | share of 3.35 TB/s |")
    print("|---|---|---|---|---|---|")
    for name, fmt, prof, doc, flags in cases:
        settings = lib.profile(prof) if prof else None
        fname = {98: "BC7", 71: "BC1", 95: "BC6H"}[fmt]
        one = timed(lambda: lib.preview_pixels(fmt, [doc], flags, settings), a.reps)
        two = timed(lambda: lib.decode(fname, lib.encode_pixels(fname, doc, flags, settings), n, n), a.reps)
        blocks = lib.encode_pixels(fname, doc, flags, settings)
        target = 28                                               # the display target of an 8- / 16-bit document
        d_blocks = torch.from_numpy(blocks).cuda()
        d_out = torch.empty(n * n * 4, dtype=torch.uint8, device="cuda")
        ks = []
        for i in range(a.reps + 1):
            lib.decompress_raw(fmt, d_blocks.data_ptr(), n, n, target, d_out.data_ptr(), n * 4)
            if i:
                ks.append(lib.last_kernel_ms())
        k = statistics.median(ks)
        nbytes = blocks.size + n * n * 4
        print(f"| {name} | {one:.2f} | {two:.2f} | {k:.4f} | {nbytes / (k * 1e-3) / 1e9:.0f} | {nbytes / (k * 1e-3) / HBM:.2f} |")


if __name__ == "__main__":
    main()
