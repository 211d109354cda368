#!/usr/bin/env python3
"""Time the stack open path (itw_dds_open_stack + one itw_dds_read_stack_layer per layer) on the GPU.

Cases: a 256x256x256 BC7 volume with its 9 levels (random blocks), a 256x256x256 R8G8B8A8 volume with its 9 levels and a 64-item
1024x1024 R16G16B16A16_FLOAT 2-D array with its 11 levels (random texels with opaque alpha, so the scan reads every byte).  Each is
opened with mips as layers: 9 layers of 256x256 (a volume's layer is slice 0 of its level), or 11 layers of 1024x1024 read from item 0.
Host file, host layers, as the plug-in passes them.  Kernel times are itw_last_kernel_ms (CUDA events around the one launch of each
call).

    scan ms       the alpha scan over every image (median of --reps opens)
    layers ms     the layer stores of every layer together (median of --reps reads of the whole set)
    scan GB/s     payload bytes read over the scan's time
    layers GB/s   bytes of the images read plus bytes written (every layer) over the layer stores' time; both against 3.35 TB/s,
                  the H100 SXM data-sheet HBM3 bandwidth

python tools/open_stack_bench.py [--reps 5]     (needs a GPU; prints the card, its power limit and its top SM clock first)
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


def opaque_payload(label, n, seed):
    rng = np.random.default_rng(seed)
    p = rng.integers(0, 256, n, dtype=np.uint8)
    if label == "A8B8G8R8":
        p.reshape(-1, 4)[:, 3] = 255
    elif label == "DX10-10":
        p.view("<u2").reshape(-1, 4)[:, 3] = 0x3C00
    return p.tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import open_stack_lib as S
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    cases = []
    for name, label, shape, w, d, mips, items in (("BC7 256^3 volume, 9 levels", "BC7", "dx10-volume", 256, 256, 9, 1),
                                                  ("R8G8B8A8 256^3 volume, 9 levels", "A8B8G8R8", "legacy-volume", 256, 256, 9, 1),
                                                  ("RGBA16F 64 x 1024^2 array, 11 levels", "DX10-10", "2d-array-2", 1024, 1, 11, 64)):
        head = S.header(label, shape, w, w, d, mips, count=items if items > 1 else None)
        n = S.payload_bytes(label, w, w, d, mips, items)
        cases.append((name, np.frombuffer(head + opaque_payload(label, n, len(cases) + 1), np.uint8).copy()))
    print(f"# {gpu}; medians of {a.reps} runs; HBM bound {HBM_TBS} TB/s (data sheet)")
    print("| case | file MB | layers | scan ms | scan GB/s | layers ms | layers GB/s | of HBM (scan / layers) |")
    print("|---|---|---|---|---|---|---|---|")
    for name, f in cases:
        info = lib.dds_stack_layout(lib.dds_open_stack(f.ctypes.data, f.size), B.OPEN_MIPS)
        dtype = {8: np.uint8, 16: np.uint16, 32: np.float32}[info.depth]
        out = [np.empty((info.height, info.width, info.planes), dtype) for _ in range(info.calls)]
        scans, stores = [], []
        for _ in range(a.reps + 1):                                  # the first round warms up
            lib.dds_open_stack(f.ctypes.data, f.size)
            scans.append(lib.last_kernel_ms())
            ms = 0.0
            for c in range(info.calls):
                assert lib.dds_read_stack_layer_raw(f.ctypes.data, f.size, info, c, out[c].ctypes.data) == 0, lib.last_error()
                ms += lib.last_kernel_ms()
            stores.append(ms)
        scan, store = statistics.median(scans[1:]), statistics.median(stores[1:])
        payload = f.size - info.payload_offset
        label = "BC7" if "BC7" in name else "A8B8G8R8" if "R8G8" in name else "DX10-10"
        read = sum(S.image_bytes(label, info.width, info.height, m) for m in range(info.calls))
        layer_out = sum(o.nbytes for o in out)
        sg = payload / (scan * 1e-3) / 1e9
        lg = (read + layer_out) / (store * 1e-3) / 1e9
        print(f"| {name} | {f.size / 1e6:.1f} | {info.calls} | {scan:.3f} | {sg:.0f} | {store:.2f} | {lg:.0f} | "
              f"{sg / (HBM_TBS * 1e3):.2f} / {lg / (HBM_TBS * 1e3):.2f} |", flush=True)


if __name__ == "__main__":
    main()
