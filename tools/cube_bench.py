#!/usr/bin/env python3
"""Time itw_dds_encode_cube on a cross document against itw_dds_encode_pixels with six row-offset sources into the same document.

Workload: a 4096x3072 horizontal cross (1024x1024 faces) at depth 8 with alpha, saved as BC7 basic and as BC6H basic (the same document
at depth 32), with the full chain (11 levels) and with the set mip level L = 3 (a one-level 128x128 cube).  The two calls alternate in one
process.

    blocks      4x4 blocks encoded, from the shapes: the six-source call always encodes the full chain
    device ms   sum of the kernel times of one call (torch.profiler with CUDA activities, a run of its own; copies and memsets excluded)
    e2e ms      host document in -> DDS file on the host, wall clock, median of --reps calls per path, the paths alternated
    parity      every byte of the timed cube file against the oracle pipeline of tests/cube_lib.py at the same size (the oracle runs
                on the CPU, one thread per face); full-chain rows also against the six-source file

    python tools/cube_bench.py [--reps 5]     (needs a GPU; prints the card and its power limit first)
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
CELLS = ((2, 1), (0, 1), (1, 0), (1, 2), (1, 1), (3, 1))


def kernel_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA" or "memcpy" in e.name.lower() or "memset" in e.name.lower():
            continue
        total += e.device_time
    return total / 1e3


def blocks(w, h, levels):
    return sum(((max(1, w >> l) + 3) // 4) * ((max(1, h >> l) + 3) // 4) for l in levels) * 6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--face", type=int, default=1024)
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    n = a.face
    W, H = 4 * n, 3 * n
    full = n.bit_length()
    rng = np.random.default_rng(1)
    y, x = np.mgrid[0:H, 0:W]
    doc8 = np.clip(np.stack([(x // 3 + y // 5 + c * 50) % 256 for c in range(4)], -1) + rng.integers(-8, 9, (H, W, 4)), 0, 255).astype(np.uint8)
    doc32 = np.ascontiguousarray((doc8.astype(np.float32) / 255.0) ** 2.2 * 4.0)
    print(f"# {gpu}; {W}x{H} cross, {n}x{n} faces; e2e medians of {a.reps} calls per path, alternated")
    print("| encoding | mips | blocks cube | blocks six sources | cube device ms | six-source device ms | cube e2e ms | six-source e2e ms | parity |")
    print("|---|---|---|---|---|---|---|---|---|")
    import cube_lib as C
    for name, dxgi, prof, doc in (("BC7 basic", 98, "basic", doc8), ("BC6H basic", 95, "bc6h_basic", doc32)):
        s = lib.profile(prof) if prof else None
        esize = doc.itemsize * 4
        srcs = (B.PixelSource * 6)(*[B.PixelSource(doc.ctypes.data + (cy * n * W + cx * n) * esize, n, n, 4, doc.itemsize * 8, W * esize)
                                     for cx, cy in CELLS])
        d = B.DdsDesc(n, n, full, 6, dxgi, 1)
        nbytes = lib.lib.itw_dds_file_bytes(ctypes.byref(d))
        six_out = np.zeros(nbytes, np.uint8)
        f = lib.lib.itw_dds_encode_pixels
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(B.DdsDesc), ctypes.POINTER(B.PixelSource), ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
        sp = ctypes.cast(ctypes.byref(s), ctypes.c_void_p)

        def six():
            assert f(ctypes.byref(d), srcs, B.FRONT_HAS_ALPHA, sp, six_out.ctypes.data, nbytes) == nbytes, lib.last_error()
        for level in (-1, 3):
            o = B.CubeOptions(dxgi, B.CUBE_CROSS, 1, level)
            cube = lambda: lib.dds_encode_cube(o, doc, None, B.FRONT_HAS_ALPHA, s)
            got = cube()
            six()
            t0 = time.perf_counter()
            want = C.oracle_save(o, doc, None, B.FRONT_HAS_ALPHA, prof, threads=min(6, len(os.sched_getaffinity(0))))
            parity = ("equal to oracle" if np.array_equal(got, want) else "DIFFERS from oracle") + f" ({time.perf_counter() - t0:.0f} s on the CPU)"
            if level < 0:
                parity += ", equal to six-source" if np.array_equal(got, six_out) else ", DIFFERS from six-source"
            cdev, sdev = kernel_ms(cube), kernel_ms(six)
            tc, ts = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                cube()
                tc.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                six()
                ts.append((time.perf_counter() - t0) * 1e3)
            label = f"full ({full})" if level < 0 else f"L = {level}"
            bc = blocks(n, n, range(full) if level < 0 else [level])
            print(f"| {name} | {label} | {bc} | {blocks(n, n, range(full))} | {cdev:.3f} | {sdev:.3f} | {statistics.median(tc):.1f} | "
                  f"{statistics.median(ts):.1f} | {parity} |", flush=True)


if __name__ == "__main__":
    main()
