"""Call counts of every dfaStagedKernel<ENGINE, SMEM_TABLE, CH, ILP, FUSED, SEG, MASK> instantiation, read from
the coverage build of the SIMT-emulated library (HSB_EMU_COVERAGE=1 python -m pytest tests -m gpu, then this
script).  Counts add up over runs; delete tests/emu/_build_cov/*.gcda to start again.  TEST infrastructure only.

gcov's per-function summary (-f) is wrong for these templates, so the counts come from the `function ... called N`
lines of its branch output."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
GCDA = os.path.join(HERE, "_build_cov", "dfa_kernels.cu.gcda")
LINE = re.compile(r"^function .*?(dfaStagedKernel<[^>]*>)\(.*? called (\d+)")


def counts(gcda=GCDA):
    """{instantiation: calls}"""
    out = subprocess.run(["gcov", "-b", "-m", "-t", "-o", os.path.dirname(gcda), gcda], capture_output=True,
                         text=True, check=True, cwd=os.path.dirname(gcda)).stdout
    got = {}
    for line in out.splitlines():
        m = LINE.match(line)
        if m:
            got[m.group(1)] = got.get(m.group(1), 0) + int(m.group(2))
    return got


def main():
    gcda = sys.argv[1] if len(sys.argv) > 1 else GCDA
    if not os.path.exists(gcda):
        sys.exit("%s not found: run the emulated suite with HSB_EMU_COVERAGE=1 first" % gcda)
    got = counts(gcda)
    for name in sorted(got):
        print("%10d  %s" % (got[name], name))
    print("%d instantiations, %d never called" % (len(got), sum(1 for v in got.values() if not v)))


if __name__ == "__main__":
    main()
