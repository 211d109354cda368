#!/usr/bin/env python3
"""Time the open path of the other block-compressed files (itw_dds_open_other_bc + one itw_dds_read_other_bc_layer per layer) on the GPU.

Cases: 4096x4096 files with their full chains (13 levels) of BC2 (DX10 74, random blocks: alpha below 0.99 somewhere, so the scan
runs over every level), BC5_SNORM (FourCC BC5S, no alpha: no scan) and BC6H_TYPELESS (DX10 94, 16-bit planes), each opened with mips as
layers (13 layers of 4096x4096, four planes); and one image into three planes (no alpha, no layers: the plug-in's background layer) of
BC4_SNORM (8 bits) and BC6H_TYPELESS (16 bits), 4096x4096 without a chain.  Host file, host layers, as the plug-in passes them.

    wall ms       open + every layer, host file in and host layers out; median of --reps
    scan us       the alpha scan kernel (torch.profiler, one profiled open after the timed ones)
    layer us      the layer kernels of every layer together (torch.profiler, same run)
    scan GB/s     payload bytes read over the scan's time
    layer GB/s    bytes read (each level once) plus bytes written (every layer) over the layer kernels' time; both against
                  3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth

python tools/open_other_bc_bench.py [--reps 5]     (needs a GPU; prints the card, its power limit and its top SM clock first)
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("intel-texture-works-plugin_b200")
B = importlib.import_module("intel-texture-works-plugin_b200.binding")
HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import open_other_bc_lib as L
    import open_uncompressed_bench as OB                          # the profiler helper
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    W, chain = 4096, 13

    def open_obc(file, options=B.OPEN_MIPS):
        f = np.ascontiguousarray(file)
        info = lib.dds_other_bc_layout(lib.dds_open_other_bc(f.ctypes.data, f.size), options)
        dt = {8: np.uint8, 16: np.uint16}[info.depth]
        out = [np.empty((info.height, info.width, info.planes), dt) for _ in range(info.calls)]
        for c in range(info.calls):
            assert lib.dds_read_other_bc_layer_raw(f.ctypes.data, f.size, info, c, out[c].ctypes.data) == 0, lib.last_error()
        return info, out

    cases = [("BC2 (DX10 74) 4096^2, 13 levels", L.dx10_file(74, W, W, chain, seed=1), B.OPEN_MIPS),
             ("BC5_SNORM (BC5S) 4096^2, 13 levels", L.legacy_file("BC5S", W, W, chain, seed=2), B.OPEN_MIPS),
             ("BC6H_TYPELESS (DX10 94) 4096^2, 13 levels", L.dx10_file(94, W, W, chain, seed=3), B.OPEN_MIPS),
             ("BC4_SNORM (BC4S) 4096^2, one image", L.legacy_file("BC4S", W, W, 1, seed=4), 0),
             ("BC6H_TYPELESS (DX10 94) 4096^2, one image", L.dx10_file(94, W, W, 1, seed=5), 0)]
    scan_k, layer_k = "open_alpha_kernel", "open_layer_kernel"
    print(f"# {gpu}; medians of {a.reps} runs; HBM bound {HBM_TBS} TB/s (data sheet)")
    print("| case | file MB | layers | planes x depth | wall ms | scan us | scan GB/s | layer us | layer GB/s | of HBM (scan / layer) |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for name, file, opt in cases:
        info, _ = open_obc(file, opt)
        tw = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            open_obc(file, opt)
            tw.append((time.perf_counter() - t0) * 1e3)
        us = OB.kernel_us(lambda: open_obc(file, opt), (scan_k, layer_k))
        payload = file.size - (148 if bytes(file[84:88]) == b"DX10" else 128)
        layer_out = info.calls * info.width * info.height * info.planes * info.depth // 8
        sg = payload / (us[scan_k] * 1e-6) / 1e9 if us[scan_k] > 0 else float("nan")
        lg = (payload + layer_out) / (us[layer_k] * 1e-6) / 1e9 if us[layer_k] > 0 else float("nan")
        print(f"| {name} | {file.size / 1e6:.1f} | {info.calls} | {info.planes} x {info.depth} | {statistics.median(tw):.1f} | "
              f"{us[scan_k]:.1f} | {sg:.0f} | {us[layer_k]:.1f} | {lg:.0f} | {sg / (HBM_TBS * 1e3):.2f} / {lg / (HBM_TBS * 1e3):.2f} |",
              flush=True)


if __name__ == "__main__":
    main()
