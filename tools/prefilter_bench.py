#!/usr/bin/env python
"""A rule-shaped set of 64 prefiltered expressions (HS_FLAG_PREFILTER, DESIGN.md section 10b): back-references,
look-around and long counted repeats such as [^\\n]{300,}, as network-signature rules write them.  Kernel ms of a
whole scan of a resident corpus at 1 GiB (2^20 blocks of 1 KiB) and at 4 blocks of 16 MiB (cut into segments by the
default rule), beside the same set compiled without its prefilter-only constructs, so that the cost of the
any-byte runs and widened repeats shows (run on the GPU box):
    python tools/prefilter_bench.py [--mb 1024] [--long-mb 16] [--reps 3]

Each figure is the median of --reps scans after one warm-up scan, from the library's CUDA events around the scan's
kernels (hs_b200_last_kernel_ms).  One JSON line per set and corpus, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402

PREFILTER = 128


def _word(i):
    return bytes(b"klmnopqr"[(i // 8 ** j) % 8] for j in range(3))


def rules():
    """64 expressions, and for each a plain form without the prefilter-only constructs and a sample match"""
    out = []
    for i in range(64):
        w = _word(i)
        out.append([
            (b"%s=(['\"])[^\\n]*?\\1" % w, b"%s=[\"'][^\\n]*?[\"']" % w, b"%s='x'" % w),
            (b"/%s(?!\\.php)[a-z]+" % w, b"/%s[a-z]+" % w, b"/%sabc" % w),
            (b"(?<=GET )/%s[^\\n]{300,}\\r" % w, b"/%s[^\\n]{30,}\\r" % w, b"GET /%s" % w + b"a" * 300 + b"\r"),
            (b"(?i)%s:(?>\\s*)(\\d+)\\s+\\1" % w, b"(?i)%s:\\s*\\d+\\s+\\d+" % w, b"%s: 42 42" % w),
        ][i % 4])
    return out


def _time(db, corpus, reps):
    scratch = capi.Scratch(db)
    ms = []
    for i in range(1 + reps):
        capi.scan_corpus(db, corpus, scratch, fetch=False)
        if i >= 1:
            ms.append(scratch.last_kernel_ms())
    n = len(capi.scan_corpus(db, corpus, scratch))   # delivered matches
    st = scratch.segment_stats()
    scratch.free()
    return float(np.median(ms)), n, st["runs"], st["segments"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=1024)
    ap.add_argument("--long-mb", type=int, default=16, help="length of each of the 4 long blocks")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    rs = rules()
    samples = [s for _, _, s in rs]
    sets = []
    for name, exprs, flags in (("prefilter", [p for p, _, _ in rs], PREFILTER), ("plain", [q for _, q, _ in rs], 0)):
        t0 = time.time()
        db = capi.compile_multi(exprs, [flags] * len(exprs), list(range(len(exprs))))
        sets.append((name, db, time.time() - t0))
    for nb, bl in (((args.mb << 20) // 1024, 1024), (4, args.long_mb << 20)):
        data, off, ln, _ = synth.block_corpus(nb, bl, samples, plant_per_kb=0.5, seed=7)
        corpus = capi.Corpus.upload(data, off, ln)
        del data
        for name, db, compile_s in sets:
            ms, n, runs, segments = _time(db, corpus, args.reps)
            info = db.info()
            print(json.dumps({"set": name, "blocks": nb, "block_len": bl, "kernel_ms": round(ms, 3),
                              "GBps": round(nb * bl / (ms * 1e-3) / 1e9, 2), "records": n,
                              "runtime_impl": info.runtime_impl, "engines": info.engine_count,
                              "segment_runs": runs, "segments": segments, "compile_s": round(compile_s, 2)}), flush=True)
        corpus.free()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card}))


if __name__ == "__main__":
    main()
