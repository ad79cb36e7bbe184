#!/usr/bin/env python
"""Regular-expression sets split over K engines run as outfixes (DESIGN.md section 10e), for K from 64 to 1 024:
kernel ms of a whole scan of a resident corpus at 1 GiB (2^20 blocks of 1 KiB), at 4 096 blocks of 1 KiB and at 4
blocks of 16 MiB (cut into segments by the default rule), and the segment state of that last scan (run on the GPU
box; tools/multi_outfix_bench.py measures sets of a few engines):
    python tools/many_engines_bench.py [--ks 64,128,256,512,1024] [--mb 1024] [--reps 1]

Each engine holds one leader expression of 200-300 positions (two do not fit one engine), in turn McClellan-16, a
LimEx-512 and McClellan-8, beside a `#tag[0-9]+!` expression of its own, so a set of K leaders splits into exactly
K engines, a third of each kind.  Each figure is the median of --reps scans after one warm-up scan, from the
library's CUDA events around the scan's kernels (hs_b200_last_kernel_ms).  The segment state is bounded from above
as (segments per run) x (engines of a run) x 2 states x 64 bytes (the LimEx-512 state).  One JSON line per set
and corpus, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402


def _tag(i):
    return bytes(b"klmnop"[(i // 6 ** j) % 6] for j in range(4))


def expressions(k):
    """k engines' expressions and a sample match of each engine's own expression"""
    out, samples = [], []
    for i in range(k):
        out += [[b"q[a-d]{300}z"], [b"r[0-3]{300}s", b"x[ab]*a[ab]{10}y"], [b"t[0-3]{200}u", b"x" + _tag(i) + b"y+"]][i % 3]
        out.append(b"#" + _tag(i) + b"[0-9]+!")
        samples.append(b"#" + _tag(i) + b"42!")
    return out, samples


def _time(db, corpus, reps):
    scratch = capi.Scratch(db)
    ms = []
    for i in range(1 + reps):
        capi.scan_corpus(db, corpus, scratch, fetch=False)
        if i >= 1:
            ms.append(scratch.last_kernel_ms())
    n = len(capi.scan_corpus(db, corpus, scratch))   # delivered matches
    st = scratch.segment_stats()
    runs, segments = st["runs"], st["segments"]
    scratch.free()
    return float(np.median(ms)), n, runs, segments


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="64,128,256,512,1024")
    ap.add_argument("--mb", type=int, default=1024)
    ap.add_argument("--small", type=int, default=4096, help="blocks of the small corpus")
    ap.add_argument("--long-mb", type=int, default=16, help="length of each of the 4 long blocks")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    ks = [int(x) for x in args.ks.split(",")]
    _, samples = expressions(max(ks))
    corpora = []
    for nb, bl in (((args.mb << 20) // 1024, 1024), (args.small, 1024), (4, args.long_mb << 20)):
        data, off, ln, _ = synth.block_corpus(nb, bl, samples, plant_per_kb=0.5, seed=7)
        corpora.append((nb, bl, capi.Corpus.upload(data, off, ln)))
    for k in ks:
        exprs, _ = expressions(k)
        t0 = time.time()
        db = capi.compile_multi(exprs, [0] * len(exprs), list(range(len(exprs))))
        compile_s = time.time() - t0
        assert db.info().engine_count == k
        for nb, bl, corpus in corpora:
            ms, n, runs, segments = _time(db, corpus, args.reps)
            line = {"engines": k, "blocks": nb, "block_len": bl, "kernel_ms": round(ms, 3),
                    "GBps": round(nb * bl / (ms * 1e-3) / 1e9, 2), "engine_GBps": round(k * nb * bl / (ms * 1e-3) / 1e9, 1),
                    "records": n, "compile_s": round(compile_s, 1)}
            if runs:
                per_run = segments / runs
                line.update({"segment_runs": runs, "segments_per_run": round(per_run, 1),
                             "segment_state_bytes_max": int(per_run * ((k + 2) // 3) * 2 * 64)})
            print(json.dumps(line), flush=True)
    for _, _, corpus in corpora:
        corpus.free()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card}))


if __name__ == "__main__":
    main()
