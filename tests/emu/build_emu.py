"""Build tests/emu/_build/libhs_b200_simt_emu.so: the library's own sources compiled
as plain C++ against the SIMT emulator (simt_emu.h) and the restated CUDA runtime
(cuda_runtime.h) of this directory.  TEST infrastructure only -- see simt_emu.h."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "hyperscan_b200", "csrc")
# HSB_EMU_SANITIZE=1: AddressSanitizer build (run pytest with LD_PRELOAD=libasan.so and
# ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0) -- a memcheck for host and kernel logic
SANITIZE = os.environ.get("HSB_EMU_SANITIZE") == "1"
# HSB_EMU_COVERAGE=1: gcov build (--coverage -O0); each test run adds its counts to the .gcda files beside the
# objects, which kernel_coverage.py reads
COVERAGE = os.environ.get("HSB_EMU_COVERAGE") == "1"
OUT_DIR = os.path.join(HERE, "_build_asan" if SANITIZE else "_build_cov" if COVERAGE else "_build")
OUT = os.path.join(OUT_DIR, "libhs_b200_simt_emu.so")
HOST = ["host/api_host.cpp", "host/rose_build.cpp", "host/hwlm_build.cpp", "host/db_walk.cpp",
        "host/pair_table.cpp", "host/dfa_build.cpp", "host/limex_build.cpp", "host/regex_nfa.cpp"]
DEVICE = ["device/scan_kernels.cu", "device/api_device.cu", "device/accel_kernels.cu", "device/dfa_kernels.cu"]


def _deps():
    d = [os.path.join(HERE, f) for f in ("simt_emu.h", "simt_emu.cpp", "cuda_runtime.h")]
    for r, _, fs in os.walk(CSRC):
        d += [os.path.join(r, f) for f in fs if f.endswith((".h", ".cpp", ".cu"))]
    d.append(os.path.join(ROOT, "include", "hs_b200.h"))
    return d


def build(verbose=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    if os.path.exists(OUT) and all(os.path.getmtime(s) <= os.path.getmtime(OUT) for s in _deps()):
        return OUT
    objs = []
    common = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-fno-strict-aliasing", "-Wno-unused-value"]
    if SANITIZE:
        common += ["-fsanitize=address", "-fno-omit-frame-pointer"]
    if COVERAGE:
        common = [f for f in common if f != "-O1"] + ["--coverage", "-O0"]
    jobs = [(os.path.join(CSRC, s), common) for s in HOST]
    jobs += [(os.path.join(CSRC, s), common + ["-x", "c++", "-DHSB_HOST_EMU", "-I", HERE]) for s in DEVICE]
    jobs += [(os.path.join(HERE, "simt_emu.cpp"), common)]
    procs = []
    for src, cmd in jobs:
        obj = os.path.join(OUT_DIR, os.path.basename(src) + ".o")
        objs.append(obj)
        full = cmd + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(full), flush=True)
        procs.append((full, subprocess.Popen(full)))
    for full, pr in procs:
        if pr.wait() != 0:
            raise RuntimeError("emulator build failed: " + " ".join(full))
    link = (["-fsanitize=address"] if SANITIZE else []) + (["--coverage"] if COVERAGE else [])
    subprocess.run(["g++", "-shared"] + link + ["-o", OUT] + objs, check=True)
    return OUT


if __name__ == "__main__":
    print(build(verbose=True))
