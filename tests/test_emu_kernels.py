"""Kernel LOGIC on a CPU: the tests marked `gpu` (parity against the unmodified
reference runtime, golden and recorded vectors, API behaviour, streaming,
vectored mode) run against the SIMT-emulated build of the library (tests/emu: the kernels' own
sources compiled as plain C++, one fiber per CUDA thread, warp intrinsics as
rendezvous).

This is TEST infrastructure in the sense of oracle/: the emulated library lives
under tests/emu/_build, is loaded only here, and says nothing about the hardware
(no PTX semantics, no timing).  The product library still has no CPU scan path
(tests/test_abi.py::test_no_gpu_fails_loudly)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gpu_suite_on_the_simt_emulator():
    env = dict(os.environ, HSB200_EMU="1", HSB200_WARPS="4", HSB_EMU_SMS="3")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests"), "-q", "-x", "-m", "gpu",
                        "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 180, tail
