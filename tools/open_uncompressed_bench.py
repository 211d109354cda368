#!/usr/bin/env python3
"""Time the uncompressed open path (itw_dds_open_uncompressed + one itw_dds_read_uncompressed_layer per layer) on the GPU, next to
the block-compressed open path (itw_dds_open + itw_dds_read_layer) of a BC7 file of the same document.

Cases: a 4096x4096 document with its full chain (13 levels) saved as an R8G8B8A8_UNORM "none" file, as an R32G32B32A32_FLOAT file
(FourCC 116), and as a BC7 `alpha_basic` file; each opened with mips as layers (13 layers, the layer of level l in the top-left corner of a
4096x4096 layer).  Host file, host layers, as the plug-in passes them.

    wall ms       open + every layer, host file in and host layers out; median of --reps
    scan us       the alpha scan kernel (torch.profiler, one profiled open after the timed ones)
    layer us      the layer kernels of every layer together (torch.profiler, same run)
    scan GB/s     payload bytes read over the scan's time
    layer GB/s    bytes read (each level once) plus bytes written (13 full layers) over the layer kernels' time; both against
                  3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth
    layer 0 = doc the none file's layer 0 against the document it was saved from

python tools/open_uncompressed_bench.py [--reps 5]     (needs a GPU; prints the card, its power limit and its top SM clock first)
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


def kernel_us(fn, names):
    """Device time of the kernels whose names contain one of `names`, in one call of `fn`, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for n in names:
            if n in e.name:
                out[n] += e.device_time
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import open_uncompressed_lib as U
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    W = 4096
    rng = np.random.default_rng(1)
    doc = rng.integers(0, 256, (W, W, 4), dtype=np.uint8)
    doc[..., 3] = np.maximum(doc[..., 3], 128)
    none = lib.dds_save_none(B.NoneOptions(B.PANE_2D, 1, -1), doc, None, B.FRONT_HAS_ALPHA)
    chain = 13
    fpay = rng.uniform(0.0, 1.0, U.payload_bytes(W, W, chain, 1, 16) // 4).astype(np.float32)
    f32 = U.legacy_file("A32B32G32R32F", W, W, chain, payload=fpay.tobytes())
    bdesc = B.DdsDesc(W, W, chain, 1, 98, 0)
    bc7 = lib.dds_encode_pixels(bdesc, [doc], B.FRONT_HAS_ALPHA, lib.profile("alpha_basic"))

    def open_raw(file):
        f = np.ascontiguousarray(file)
        info = lib.dds_uncompressed_layout(lib.dds_open_uncompressed(f.ctypes.data, f.size), B.OPEN_MIPS)
        dt = {8: np.uint8, 16: np.uint16, 32: np.float32}[info.depth]
        out = [np.empty((info.height, info.width, info.planes), dt) for _ in range(info.calls)]
        for c in range(info.calls):
            assert lib.dds_read_uncompressed_layer_raw(f.ctypes.data, f.size, info, c, out[c].ctypes.data) == 0, lib.last_error()
        return info, out

    def open_bc(file):
        f = np.ascontiguousarray(file)
        info = lib.dds_open_layout(lib.dds_open(f.ctypes.data, f.size), B.OPEN_MIPS)
        out = [np.empty((info.height, info.width, info.planes), np.float32 if info.depth == 32 else np.uint8) for _ in range(info.calls)]
        for c in range(info.calls):
            lib.dds_read_layer_raw(f.ctypes.data, f.size, info, c, out[c].ctypes.data)
        return info, out

    cases = [("none RGBA8 4096^2, 13 levels", none, open_raw, 4, "open_raw_alpha_kernel", "open_raw_layer_kernel"),
             ("RGBA32F (FourCC 116) 4096^2, 13 levels", f32, open_raw, 16, "open_raw_alpha_kernel", "open_raw_layer_kernel"),
             ("BC7 alpha_basic 4096^2, 13 levels", bc7, open_bc, 1, "open_alpha_kernel", "open_layer_kernel")]
    print(f"# {gpu}; medians of {a.reps} runs; HBM bound {HBM_TBS} TB/s (data sheet)")
    print("| case | file MB | layers | wall ms | scan us | scan GB/s | layer us | layer GB/s | of HBM (scan / layer) | layer 0 = doc |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for name, file, fn, texel, scan_k, layer_k in cases:
        info, layers = fn(file)
        tw = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn(file)
            tw.append((time.perf_counter() - t0) * 1e3)
        us = kernel_us(lambda: fn(file), (scan_k, layer_k))
        payload = file.size - (148 if file.size >= 148 and bytes(file[84:88]) == b"DX10" else 128)
        layer_out = info.calls * info.width * info.height * info.planes * info.depth // 8
        sg = payload / (us[scan_k] * 1e-6) / 1e9 if us[scan_k] > 0 else float("nan")
        lg = (payload + layer_out) / (us[layer_k] * 1e-6) / 1e9 if us[layer_k] > 0 else float("nan")
        same = np.array_equal(layers[0], doc) if fn is open_raw and texel == 4 else None
        print(f"| {name} | {file.size / 1e6:.1f} | {info.calls} | {statistics.median(tw):.1f} | {us[scan_k]:.1f} | {sg:.0f} | "
              f"{us[layer_k]:.1f} | {lg:.0f} | {sg / (HBM_TBS * 1e3):.2f} / {lg / (HBM_TBS * 1e3):.2f} | "
              f"{'equal' if same else ('-' if same is None else 'DIFFERS')} |", flush=True)


if __name__ == "__main__":
    main()
