"""Per-phase cycle breakdown of bc7_kernel: where the cycles of a BC7 encode go, phase by phase.

Builds the library with -DITW_BC7_PHASE_CLOCKS (thread 0 of every CTA reads clock64() after every barrier of the kernel and
adds the cycles since its previous reading to that phase site) to a separate path, encodes device-resident surfaces, and
prints each site's share of the summed CTA cycles, the mean cycles of a full round and those of the last round, and the
cycles of each pass of the chain phase with the two units it ran.

    python tools/bc7_phase_clocks.py                      # slow and basic at 4096 x 4096
    python tools/bc7_phase_clocks.py --build-only --out /tmp/clocks/libitw_bcn.so
    python tools/bc7_phase_clocks.py --lib /tmp/clocks/libitw_bcn.so --profiles slow --size 8192
"""
import argparse
import ctypes
import importlib
import os
import subprocess
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
PKG = "intel-texture-works-plugin_b200"
SITES = 40                                                  # kBc7ClockSites
MAX_ROLES = 18                                              # kBc7MaxRoles


class Bc7Clocks(ctypes.Structure):                           # csrc/bc7.cuh
    _fields_ = [("site", ctypes.c_uint64 * SITES), ("name", (ctypes.c_char * 48) * SITES),
                ("full_sum", ctypes.c_uint64), ("full_count", ctypes.c_uint64),
                ("last_sum", ctypes.c_uint64), ("last_max", ctypes.c_uint64), ("last_ctas", ctypes.c_uint64),
                ("pass_sum", ctypes.c_uint64 * MAX_ROLES), ("pass_count", ctypes.c_uint64 * MAX_ROLES),
                ("pass_unit", (ctypes.c_int * 2) * MAX_ROLES)]


def unit_name(s, u):
    """Label of chain unit u under settings s (bc7_chain's numbering): a mode slot, a rotation of modes 4/5 or mode 6."""
    if u < 0:
        return "-"
    if u < 5:
        return "m" + "02137"[u]
    nrot = max(s.channels - s.mode45_channel0, 0) if s.mode_selection[2] else 0
    return f"R{s.mode45_channel0 + u - 5}" if u < 5 + nrot else "m6"


def build(out):
    sys.path.insert(0, os.path.join(ROOT, PKG))
    try:
        import build as product_build
    finally:
        sys.path.pop(0)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    cmd = [os.environ.get("NVCC", "nvcc")] + product_build.NVCC_FLAGS + ["-DITW_BC7_PHASE_CLOCKS"] + product_build.sources() + ["-o", out]
    print("[build]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return out


def measure(lib_path, profiles, size, steps):
    import torch
    binding = importlib.import_module(PKG + ".binding")
    synth = importlib.import_module(PKG + ".synth")
    lib = binding.ItwBcn(lib_path)
    clocks_fn = lib.lib.itw_bc7_phase_clocks
    clocks_fn.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
    clocks_fn.restype = ctypes.c_int
    torch.cuda.set_device(0)
    lib.set_device(0)
    src = torch.from_numpy(synth.random_rgba8(size, size, seed=0xB2000002)).cuda()
    dst = torch.empty((size // 4) * (size // 4) * 16, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()
    c = Bc7Clocks()

    def read():
        if clocks_fn(ctypes.byref(c), ctypes.sizeof(c)) != 0:
            raise RuntimeError(lib.lib.itw_get_last_error().decode())

    for prof in profiles:
        settings = lib.profile(prof)
        lib.encode_device("BC7", src.data_ptr(), size, size, size * 4, dst.data_ptr(), settings, stream.cuda_stream)  # warm-up
        read()
        for _ in range(steps):
            lib.encode_device("BC7", src.data_ptr(), size, size, size * 4, dst.data_ptr(), settings, stream.cuda_stream)
        read()
        total = sum(c.site)
        print(f"\nBC7 {prof}, {size}x{size}, {steps} encodes, {torch.cuda.get_device_name(0)}")
        print(f"{'site':>4}  {'share':>7}  {'Mcycles':>10}  phase")
        for i in range(SITES):
            if c.site[i]:
                print(f"{i:>4}  {100.0 * c.site[i] / total:6.2f}%  {c.site[i] / 1e6:10.2f}  {c.name[i].value.decode()}")
        full = c.full_sum / c.full_count if c.full_count else 0.0
        print(f"summed CTA cycles: {total / 1e6:.2f} M")
        print(f"full rounds: {c.full_count // steps} CTA-rounds per encode, mean {full:,.0f} cycles")
        if c.last_ctas:
            print(f"last round: {c.last_ctas // steps} CTAs per encode, longest {c.last_max:,} cycles "
                  f"({c.last_max / full:.3f} of a full round), mean {c.last_sum / c.last_ctas:,.0f}" if full else
                  f"last round: {c.last_ctas // steps} CTAs per encode, longest {c.last_max:,} cycles")
        else:
            print("last round: none (the surface is a whole number of full rounds)")
        chain = sum(c.pass_sum)
        if chain:
            print("chain passes of the full rounds (lane 0 of warp 0 of each CTA):")
            print(f"{'pass':>4}  {'units':<12}  {'of chain':>8}  {'of all':>7}  {'cycles/pass':>11}")
            for p in range(MAX_ROLES):
                if c.pass_count[p]:
                    units = ", ".join(unit_name(settings, u) for u in c.pass_unit[p] if u >= 0)
                    print(f"{p:>4}  {units:<12}  {100.0 * c.pass_sum[p] / chain:7.2f}%  "
                          f"{100.0 * c.pass_sum[p] / total:6.2f}%  {c.pass_sum[p] / c.pass_count[p]:11,.0f}")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", help="an already built -DITW_BC7_PHASE_CLOCKS library (default: build one to a temporary directory)")
    ap.add_argument("--out", help="where to build the library (default: a temporary directory)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--profiles", default="slow,basic")
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    path = args.lib
    if not path:
        path = build(args.out or os.path.join(tempfile.mkdtemp(prefix="bc7_clocks_"), "libitw_bcn.so"))
    if args.build_only:
        print(path)
        return
    measure(path, args.profiles.split(","), args.size, args.steps)


if __name__ == "__main__":
    main()
