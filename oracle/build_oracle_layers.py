#!/usr/bin/env python3
"""Build oracle/libitw_oracle_layers.so from oracle/itw_oracle_layers.cpp (test infrastructure only): the handwritten oracle of
the layer-to-mip-level copy, with the g++ flags of oracle/Makefile's libitw_oracle.so (the float rules of DESIGN.md section 2).
Rebuilt only when a source is newer than the library."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_SO = os.path.join(HERE, "libitw_oracle_layers.so")
SOURCES = [os.path.join(HERE, n) for n in ("itw_oracle_layers.cpp", "itw_oracle_frontend.cpp")] + \
          [os.path.join(HERE, "..", "include", "itw_bcn.h")]
FLAGS = ["-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fwrapv", "-mfpmath=sse", "-msse2", "-Wall", "-Wextra"]


def build(verbose=True):
    if os.path.exists(OUT_SO) and all(os.path.getmtime(s) <= os.path.getmtime(OUT_SO) for s in SOURCES):
        return OUT_SO
    cmd = ["g++"] + FLAGS + ["-shared", "-Wl,--no-undefined", "-o", OUT_SO, SOURCES[0]]
    if verbose:
        print("[build_oracle_layers]", " ".join(cmd))
    subprocess.check_call(cmd)
    return OUT_SO


if __name__ == "__main__":
    print(build())
