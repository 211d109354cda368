"""The kernels' per-lane logic (tests/emu) compiled with -fsanitize=address,undefined and run over every encoder and profile:
out-of-bounds indices into the per-warp scratch structs, misaligned accesses and signed overflows in the kernel logic show up
here without a GPU (tools/sanitize.sh runs compute-sanitizer over the device build)."""
import os
import subprocess
import tempfile

import itw_testlib as T

HERE = os.path.dirname(os.path.abspath(__file__))


def test_kernel_logic_under_asan_and_ubsan():
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "emu_asan")
        T.build_emu().compile_cpu(os.path.join(HERE, "emu", "asan_main.cpp"), exe,
                                  ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")
        res = subprocess.run([exe], capture_output=True, text=True, env=env, timeout=1200)
    assert res.returncode == 0, res.stderr[-3000:]
    assert res.stdout.startswith("ok "), res.stdout
