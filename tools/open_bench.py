#!/usr/bin/env python3
"""Time the open path on the GPU: a 4096x4096 BC7 and a 4096x4096 BC6H file with full mip chains, opened as the plug-in opens them
with mips as layers (itw_dds_open, itw_dds_open_layout(ITW_OPEN_MIPS), one itw_dds_read_layer per level).

    device   CUDA events around the kernels (the alpha scan and every layer store, itw_last_kernel_ms), summed over the open
    e2e      host file -> host layers (pageable memory, as Photoshop hands out its buffers), wall clock
    ref      the reference pipeline on the CPU: the cut IsAlphaAllOpaque + DirectX::Decompress + the plug-in's copy loop
             (tests/open_lib.py), layers spread over the cores this process may use; its layers are also the parity check
    store    the layer store's bytes (blocks read + layer written) over its kernel time, against the 3.35 TB/s HBM3 of the H100 SXM

    python tools/open_bench.py [--size 4096] [--reps 5]     (prints one table; needs a GPU and oracle/_ref from build())
"""
import argparse
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import importlib  # noqa: E402

pkg = importlib.import_module("intel-texture-works-plugin_b200")
B = importlib.import_module("intel-texture-works-plugin_b200.binding")
HBM = 3.35e12


def _ref_layer(args):
    import open_lib as O
    file, d_fields, start, call = args
    return O.read_continue(file, B.DdsDesc(*d_fields), start, call)


def ref_open(file, d, options, workers):
    """The reference pipeline, its wall time and its layers."""
    import open_lib as O
    t0 = time.perf_counter()
    start = O.read_start(d, O.ref_all_opaque(file, d), options)
    fields = (d.width, d.height, d.mip_levels, d.array_size, d.dxgi_format, d.is_cubemap)
    with ProcessPoolExecutor(workers) as ex:
        layers = list(ex.map(_ref_layer, [(file, fields, start, c) for c in range(start["calls"])]))
    return time.perf_counter() - t0, layers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    lib = pkg.ItwBcn()
    lib.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    workers = len(os.sched_getaffinity(0))
    n = a.size
    levels = n.bit_length()
    rng = np.random.default_rng(1)
    y, x = np.mgrid[0:n, 0:n]
    doc8 = np.clip(np.stack([(x + c * 50) % 256 for c in range(4)], -1) + rng.integers(-8, 9, (n, n, 4)), 0, 255).astype(np.uint8)
    doc16 = (doc8.astype(np.uint32) * 32768 // 255).astype(np.uint16)
    cases = [("BC7", 98, "alpha_basic", doc8), ("BC6H", 95, "bc6h_basic", doc16)]
    print(f"# {gpu}; {n}x{n}, {levels} levels, opened with mips as layers; medians of {a.reps} runs; reference on {workers} cores")
    print("| file | layers | alpha scan ms | layer stores ms | device ms | e2e ms | reference s | store GB/s | of 3.35 TB/s | parity |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for name, fmt, prof, doc in cases:
        d = B.DdsDesc(n, n, levels, 1, fmt, 0)
        file = lib.dds_encode_pixels(d, [doc], B.FRONT_HAS_ALPHA, lib.profile(prof))
        info = lib.dds_open_layout(lib.dds_open(file.ctypes.data, file.size), B.OPEN_MIPS)
        dtype = np.float32 if info.depth == 32 else np.uint8
        outs = [np.empty((info.height, info.width, info.planes), dtype) for _ in range(info.calls)]

        def run():
            times = [0.0, 0.0]
            i = lib.dds_open(file.ctypes.data, file.size)
            times[0] = lib.last_kernel_ms() if info.desc.dxgi_format in (77, 78, 98, 99) else 0.0
            lib.dds_open_layout(i, B.OPEN_MIPS)
            for c in range(i.calls):
                lib.dds_read_layer_raw(file.ctypes.data, file.size, i, c, outs[c].ctypes.data)
                times[1] += lib.last_kernel_ms()
            return times

        run()
        e2e, scan, store = [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            s, l = run()
            e2e.append((time.perf_counter() - t0) * 1e3)
            scan.append(s)
            store.append(l)
        scan_ms, store_ms, e2e_ms = statistics.median(scan), statistics.median(store), statistics.median(e2e)
        layer_bytes = info.calls * info.height * info.width * info.planes * info.depth // 8
        block_bytes = sum(((max(1, n >> l) + 3) // 4) ** 2 * 16 for l in range(levels))
        gbs = (layer_bytes + block_bytes) / (store_ms * 1e-3)
        ref_s, want = ref_open(file, d, B.OPEN_MIPS, workers)
        parity = all(g.tobytes() == w.tobytes() for g, w in zip(outs, want)) and len(want) == len(outs)
        print(f"| {name} | {info.calls} | {scan_ms:.3f} | {store_ms:.3f} | {scan_ms + store_ms:.3f} | {e2e_ms:.1f} | {ref_s:.2f} | "
              f"{gbs / 1e9:.0f} | {gbs / HBM:.2f} | {'equal' if parity else 'DIFFERS'} |", flush=True)


if __name__ == "__main__":
    main()
