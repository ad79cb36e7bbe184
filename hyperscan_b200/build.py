"""Build the native libraries in-tree.

  hyperscan_b200/lib/libhs_b200.so   the product: C ABI (include/hs_b200.h) +
                                     sm_90a kernels (nvcc, -gencode
                                     arch=compute_90a,code=sm_90a)
  oracle/_build/liboracle.so         the CPU restatement (test infrastructure)
  oracle/_ref/libhsref_<isa>.so      the unmodified reference runtime, only where a
                                     checkout of intel/hyperscan 5.4.2 is found
                                     (HS_REFERENCE overrides the default location in
                                     build_oracle; oracle/ref/Makefile); without it the
                                     tests use the answers recorded in
                                     tests/golden/ref_answers

Everything is rebuilt only when a source is newer than the output.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "hyperscan_b200", "csrc")
LIBDIR = os.path.join(ROOT, "hyperscan_b200", "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

HOST_SRCS = ["host/api_host.cpp", "host/rose_build.cpp", "host/hwlm_build.cpp", "host/db_walk.cpp",
             "host/pair_table.cpp", "host/dfa_build.cpp", "host/limex_build.cpp", "host/regex_nfa.cpp"]
CUDA_SRCS = ["device/scan_kernels.cu", "device/api_device.cu", "device/accel_kernels.cu", "device/dfa_kernels.cu"]


def _newer(srcs, out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(s) > t for s in srcs)


def _headers():
    hs = []
    for d, _, fs in os.walk(CSRC):
        hs += [os.path.join(d, f) for f in fs if f.endswith(".h")]
    hs.append(os.path.join(ROOT, "include", "hs_b200.h"))
    return hs


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)


def build_product(verbose=False):
    os.makedirs(OBJDIR, exist_ok=True)
    hdrs = _headers()
    objs = []
    for s in HOST_SRCS:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJDIR, os.path.basename(s) + ".o")
        if _newer([src] + hdrs, obj):
            _run(["g++", "-O3", "-std=c++17", "-fPIC", "-c", src, "-o", obj], verbose)
        objs.append(obj)
    for s in CUDA_SRCS:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        obj = os.path.join(OBJDIR, os.path.basename(s) + ".o")
        if _newer([src] + hdrs, obj):
            _run([NVCC] + ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-O3",
                                  "-c", src, "-o", obj], verbose)
        objs.append(obj)
    out = os.path.join(LIBDIR, "libhs_b200.so")
    if _newer(objs, out):
        _run([NVCC] + ARCH + ["-shared", "-cudart", "static", "-o", out] + objs, verbose)
    return out


def build_oracle(verbose=False):
    outs = []
    odir = os.path.join(ROOT, "oracle")
    src = os.path.join(odir, "hs_oracle.c")
    if os.path.exists(src):
        bdir = os.path.join(odir, "_build")
        os.makedirs(bdir, exist_ok=True)
        out = os.path.join(bdir, "liboracle.so")
        if _newer([src], out):
            _run(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-o", out, src], verbose)
        outs.append(out)
    ref = os.environ.get("HS_REFERENCE", "/root/reference")
    if os.path.isdir(os.path.join(ref, "src")):
        _run(["make", "-s", "-C", os.path.join(odir, "ref"), "-j", str(os.cpu_count() or 4), "REF=" + ref], verbose)
    return outs


def build_all(verbose=False):
    lib = build_product(verbose)
    build_oracle(verbose)
    return lib


if __name__ == "__main__":
    print(build_all(verbose="-q" not in sys.argv))
