#!/usr/bin/env python3
"""Time the expanded open path (itw_dds_open_expanded + one itw_dds_read_expanded_layer per layer) on the GPU.

Cases: 4096x4096 files with their full chains (13 levels) of P8 (random indices, a random palette), A8P8 (random words, a random
palette) and A4L4 (random bytes); each opened with mips as layers (13 layers of 4096x4096, four 8-bit planes).  Host file, host layers,
as the plug-in passes them.  Kernel times are itw_last_kernel_ms (CUDA events around the one launch of each call).

    scan ms       the alpha scan (median of --reps opens)
    layers ms     the layer stores of every layer together (median of --reps reads of the whole set)
    scan GB/s     payload bytes read over the scan's time
    layers GB/s   bytes read (each level once) plus bytes written (every layer) over the layer stores' time; both against
                  3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth

python tools/open_expanded_bench.py [--reps 5]     (needs a GPU; prints the card, its power limit and its top SM clock first)
"""
import argparse
import importlib
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("intel-texture-works-plugin_b200")
B = importlib.import_module("intel-texture-works-plugin_b200.binding")
HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import open_expanded_lib as E
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    W, chain = 4096, 13
    cases = [(f"{name} 4096^2, 13 levels", E.file_of(name, W, W, chain, seed=i + 1)) for i, name in enumerate(("P8", "A8P8", "A4L4"))]
    print(f"# {gpu}; medians of {a.reps} runs; HBM bound {HBM_TBS} TB/s (data sheet)")
    print("| case | file MB | layers | scan ms | scan GB/s | layers ms | layers GB/s | of HBM (scan / layers) |")
    print("|---|---|---|---|---|---|---|---|")
    for name, file in cases:
        f = np.ascontiguousarray(file)
        info = lib.dds_expanded_layout(lib.dds_open_expanded(f.ctypes.data, f.size), B.OPEN_MIPS)
        out = [np.empty((info.height, info.width, info.planes), np.uint8) for _ in range(info.calls)]
        scans, stores = [], []
        for _ in range(a.reps + 1):                                  # the first round warms up
            lib.dds_open_expanded(f.ctypes.data, f.size)
            scans.append(lib.last_kernel_ms())
            ms = 0.0
            for c in range(info.calls):
                assert lib.dds_read_expanded_layer_raw(f.ctypes.data, f.size, info, c, out[c].ctypes.data) == 0, lib.last_error()
                ms += lib.last_kernel_ms()
            stores.append(ms)
        scan, store = statistics.median(scans[1:]), statistics.median(stores[1:])
        payload = f.size - info.payload_offset
        layer_out = info.calls * info.width * info.height * info.planes
        sg = payload / (scan * 1e-3) / 1e9
        lg = (payload + layer_out) / (store * 1e-3) / 1e9
        print(f"| {name} | {f.size / 1e6:.1f} | {info.calls} | {scan:.3f} | {sg:.0f} | {store:.2f} | {lg:.0f} | "
              f"{sg / (HBM_TBS * 1e3):.2f} / {lg / (HBM_TBS * 1e3):.2f} |", flush=True)


if __name__ == "__main__":
    main()
