#!/usr/bin/env python3
"""Time the converted open path (itw_dds_open_converted + one itw_dds_read_converted_layer per layer) on the GPU.

Cases: 4096x4096 files with their full chains (13 levels) of FourCC 113 (R16G16B16A16_FLOAT, random halves of [0, 1) with alpha
below 0.99 somewhere, so the scan runs), DX10 R11G11B10_FLOAT (no alpha: no scan) and A4R4G4B4 (random words: scan, 8-bit
planes); each opened with mips as layers (13 layers of 4096x4096, four planes).  Two more cases open one image into three planes (no
alpha, no layers: the plug-in's background layer), the layer kernel's three-plane instantiations: an R11G11B10_FLOAT file at depth 16
and an A8L8 (R8G8_UNORM) file at depth 8, 4096x4096 without a chain.  Host file, host layers, as the plug-in passes them.

    wall ms       open + every layer, host file in and host layers out; median of --reps
    scan us       the alpha scan kernel (torch.profiler, one profiled open after the timed ones)
    layer us      the layer kernels of every layer together (torch.profiler, same run)
    scan GB/s     payload bytes read over the scan's time
    layer GB/s    bytes read (each level once) plus bytes written (every layer) over the layer kernels' time; both against
                  3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth

python tools/open_converted_bench.py [--reps 5]     (needs a GPU; prints the card, its power limit and its top SM clock first)
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
    import open_converted_lib as C
    import open_uncompressed_bench as OB                          # the profiler helper
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    W, chain = 4096, 13
    rng = np.random.default_rng(1)
    n = C.U.payload_bytes(W, W, chain, 1, 8) // 2
    halves = rng.uniform(0.0, 1.0, n).astype(np.float16).view(np.uint16)
    f113 = C.legacy_file("FourCC113", W, W, chain, payload=halves.tobytes())
    r11 = C.dx10_file(26, W, W, chain, seed=2)
    a4 = C.legacy_file("A4R4G4B4", W, W, chain, seed=3)
    r11_one = C.dx10_file(26, W, W, 1, seed=4)
    a8l8_one = C.legacy_file("A8L8", W, W, 1, seed=5)

    def open_conv(file, options=B.OPEN_MIPS):
        f = np.ascontiguousarray(file)
        info = lib.dds_converted_layout(lib.dds_open_converted(f.ctypes.data, f.size), options)
        dt = {8: np.uint8, 16: np.uint16, 32: np.float32}[info.depth]
        out = [np.empty((info.height, info.width, info.planes), dt) for _ in range(info.calls)]
        for c in range(info.calls):
            assert lib.dds_read_converted_layer_raw(f.ctypes.data, f.size, info, c, out[c].ctypes.data) == 0, lib.last_error()
        return info, out

    cases = [("RGBA16F (FourCC 113) 4096^2, 13 levels", f113, B.OPEN_MIPS), ("R11G11B10F (DX10) 4096^2, 13 levels", r11, B.OPEN_MIPS),
             ("A4R4G4B4 4096^2, 13 levels", a4, B.OPEN_MIPS), ("R11G11B10F (DX10) 4096^2, one image", r11_one, 0),
             ("A8L8 4096^2, one image", a8l8_one, 0)]
    scan_k, layer_k = "open_raw_alpha_kernel", "open_raw_layer_kernel"
    print(f"# {gpu}; medians of {a.reps} runs; HBM bound {HBM_TBS} TB/s (data sheet)")
    print("| case | file MB | layers | planes x depth | wall ms | scan us | scan GB/s | layer us | layer GB/s | of HBM (scan / layer) |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for name, file, opt in cases:
        info, _ = open_conv(file, opt)
        tw = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            open_conv(file, opt)
            tw.append((time.perf_counter() - t0) * 1e3)
        us = OB.kernel_us(lambda: open_conv(file, opt), (scan_k, layer_k))
        payload = file.size - (148 if bytes(file[84:88]) == b"DX10" else 128)
        layer_out = info.calls * info.width * info.height * info.planes * info.depth // 8
        sg = payload / (us[scan_k] * 1e-6) / 1e9 if us[scan_k] > 0 else float("nan")
        lg = (payload + layer_out) / (us[layer_k] * 1e-6) / 1e9 if us[layer_k] > 0 else float("nan")
        print(f"| {name} | {file.size / 1e6:.1f} | {info.calls} | {info.planes} x {info.depth} | {statistics.median(tw):.1f} | "
              f"{us[scan_k]:.1f} | {sg:.0f} | {us[layer_k]:.1f} | {lg:.0f} | {sg / (HBM_TBS * 1e3):.2f} / {lg / (HBM_TBS * 1e3):.2f} |",
              flush=True)


if __name__ == "__main__":
    main()
