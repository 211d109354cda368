"""Two builds of the library in one process, alternated: BC7 device-resident encode time and output equality.

Both libraries encode bench.py's inputs (the same seeded surfaces, rotated so that no step finds its input in L2) with CUDA
events on one stream.  For every workload each build first encodes every surface of the rotation once and the outputs are
compared whole; then the builds alternate, `--runs` times each, `--warmup` untimed steps followed by `--steps` timed ones.
Prints the card, its power limit and SM clock, the median ms per step of each build with the range, and the change.

    python tools/bc7_ab.py --a before/libitw_bcn.so --b intel-texture-works-plugin_b200/libitw_bcn.so
    python tools/bc7_ab.py --a A.so --b B.so --workloads slow:4096,basic:4096,slow:8192 --runs 5 --steps 10 --warmup 3
"""
import argparse
import hashlib
import importlib
import os
import statistics
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
PKG = "intel-texture-works-plugin_b200"


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--a", required=True, help="library of the first build (the baseline)")
    ap.add_argument("--b", required=True, help="library of the second build")
    ap.add_argument("--workloads", default="slow:4096,basic:4096,alpha_slow:4096,alpha_basic:4096,slow:8192")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    binding = importlib.import_module(PKG + ".binding")
    synth = importlib.import_module(PKG + ".synth")
    torch.cuda.set_device(0)
    libs = [binding.ItwBcn(os.path.abspath(p)) for p in (args.a, args.b)]
    for lib in libs:
        lib.set_device(0)
    stream = torch.cuda.current_stream()
    print("GPU (before):", gpu_state(), flush=True)
    mismatched = 0
    for wl in args.workloads.split(","):
        prof, size = wl.split(":")
        size = int(size)
        in_bytes = size * size * 4
        nrot = max(2, -(-(256 << 20) // in_bytes))                           # as bench.py
        d_in = [torch.from_numpy(synth.random_rgba8(size, size, seed=0xB2000002 + i)).cuda() for i in range(nrot)]
        d_out = torch.empty((size // 4) * (size // 4) * 16, dtype=torch.uint8, device="cuda")
        settings = [lib.profile(prof) for lib in libs]

        def step(k, i):
            libs[k].encode_device("BC7", d_in[i % nrot].data_ptr(), size, size, size * 4, d_out.data_ptr(), settings[k],
                                  stream.cuda_stream)

        digests = [[], []]
        for k in range(2):
            for i in range(nrot):
                step(k, i)
                stream.synchronize()
                digests[k].append(hashlib.sha256(d_out.cpu().numpy().tobytes()).hexdigest())
        same = digests[0] == digests[1]
        mismatched += 0 if same else 1
        times = [[], []]
        for _ in range(args.runs):
            for k in range(2):
                for i in range(args.warmup):
                    step(k, i)
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
                for i in range(args.steps):
                    evs[i][0].record(stream)
                    step(k, args.warmup + i)
                    evs[i][1].record(stream)
                stream.synchronize()
                times[k].append(sum(a.elapsed_time(b) for a, b in evs) / args.steps)
        med = [statistics.median(t) for t in times]
        print(f"{prof} {size}^2: A {med[0]:.2f} ({min(times[0]):.2f}-{max(times[0]):.2f})  B {med[1]:.2f} "
              f"({min(times[1]):.2f}-{max(times[1]):.2f}) ms  change {100.0 * (med[1] / med[0] - 1.0):+.1f} %  "
              f"outputs of all {nrot} surfaces {'identical' if same else 'DIFFER'}", flush=True)
        del d_in, d_out
    print("GPU (after):", gpu_state(), flush=True)
    sys.exit(1 if mismatched else 0)


if __name__ == "__main__":
    main()
