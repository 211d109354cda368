"""Build tests/emu/libitw_emu.so: the product's kernel logic compiled for the CPU (TEST-ONLY).

compile_cpu() holds the g++ flags of every CPU build of the kernel logic: the emulation, the routine-check drivers and the
sanitizer build differ only in what they add."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
OUT = os.path.join(HERE, "libitw_emu.so")
CSRC = os.path.join(ROOT, "intel-texture-works-plugin_b200", "csrc")
FLAGS = ["-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fwrapv", "-mfpmath=sse", "-msse2", "-Wno-unknown-pragmas"]
SHARED = ["-O2", "-fPIC", "-shared"]


def compile_cpu(src, out, extra=SHARED, verbose=False):
    """g++ `src` -> `out` with FLAGS plus `extra` (by default a shared library)."""
    cmd = ["g++"] + FLAGS + list(extra) + [src, "-o", out]
    if verbose:
        print("[build_emu]", " ".join(cmd))
    subprocess.check_call(cmd)
    return out


def build(verbose=True):
    deps = [os.path.join(HERE, "emu.cpp")] + [os.path.join(CSRC, n) for n in os.listdir(CSRC)]
    if os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    return compile_cpu(os.path.join(HERE, "emu.cpp"), OUT, verbose=verbose)


if __name__ == "__main__":
    print(build())
