#!/usr/bin/env python
"""Instruction histogram per kernel of the built CUDA objects (cuobjdump -sass), so that
claims about what a loop compiles to -- how many LDS / PRMT / LOP3 per step, whether the
TMA build carries UBLKCP, stack use -- can be checked.

  python tools/sass_summary.py > sass_summary.txt
"""
import collections
import hashlib
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "hyperscan_b200", "lib", "obj")
KEEP = ["LDS", "STS", "LDG", "STG", "LD", "ST", "LDL", "STL", "ATOM", "ATOMS", "RED", "PRMT", "LOP3", "SHF", "IMAD",
        "IADD3", "SHFL", "VOTE", "UBLKCP", "SYNCS", "CCTL", "BAR", "CALL", "BRA", "ISETP", "SEL", "POPC", "FLO"]


def demangle(name):
    try:
        return subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip() or name
    except OSError:
        return name


def main():
    for obj in sorted(os.listdir(OBJ)):
        if not obj.endswith(".cu.o"):
            continue
        path = os.path.join(OBJ, obj)
        src = os.path.join(ROOT, "hyperscan_b200", "csrc", "device", obj[:-2])
        sha = hashlib.sha256(open(src, "rb").read()).hexdigest()[:16] if os.path.exists(src) else "?"
        print("== %s (source sha256/16 %s)" % (obj, sha))
        res = subprocess.run(["cuobjdump", "-res-usage", path], capture_output=True, text=True).stdout
        usage = {}
        cur = None
        for line in res.splitlines():
            m = re.search(r"Function (\S+):", line)
            if m:
                cur = m.group(1)
            elif cur and "REG:" in line:
                usage[cur] = " ".join(x for x in line.split() if x.split(":")[0] in ("REG", "STACK", "SHARED", "LOCAL"))
        sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
        fn, hist, total, loops = None, None, 0, []

        def flush():
            if fn is None:
                return
            name = demangle(fn)
            name = re.sub(r"hsb::\(anonymous namespace\)::", "", name)
            print("  %s" % name[:150])
            print("    %s | %d instructions | backward branches (loops): %d" % (usage.get(fn, ""), total, len(loops)))
            print("    " + "  ".join("%s %d" % (k, hist[k]) for k in KEEP if hist.get(k)))
            big = sorted(loops, key=lambda x: -x[1])[:3]
            for (tgt, n, h) in big:
                print("    loop @%#x: %d instr: %s" % (tgt, n, "  ".join("%s %d" % (k, h[k]) for k in KEEP if h.get(k))))

        ins = []
        for line in sass.splitlines():
            m = re.search(r"Function : (\S+)", line)
            if m:
                flush()
                fn, hist, total, loops, ins = m.group(1), collections.Counter(), 0, [], []
                continue
            m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
            if m and fn:
                addr, text = int(m.group(1), 16), m.group(2).strip()
                op = (text.split()[1] if text.startswith("@") else text.split()[0]).split(".")[0]
                ins.append((addr, op))
                hist[op] += 1
                total += 1
                b = re.search(r"BRA.*0x([0-9a-f]+)", text)
                if b and int(b.group(1), 16) < addr:
                    tgt = int(b.group(1), 16)
                    body = collections.Counter(o for (a, o) in ins if tgt <= a <= addr)
                    loops.append((tgt, sum(body.values()), body))
        flush()


if __name__ == "__main__":
    main()
