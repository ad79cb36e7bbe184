#!/usr/bin/env python
"""A regular-expression set too large for one automaton, split over several engines run as outfixes (DESIGN.md
section 10e), on a resident corpus of uniform blocks: kernel ms of each engine's group compiled alone and of the
whole scan, at 1 GiB (2^20 blocks of 1 KiB) and at 4 096 blocks (run on the GPU box):
    python tools/multi_outfix_bench.py [--mb 1024] [--small 4096] [--exprs 64]

The groups are found the way the compiler packs them: greedily in expression order, a group closes when the next
expression no longer fits its one automaton (that set stops compiling to a single engine).  Each figure is the
median of --reps scans after two warm-up scans, from the library's CUDA events around the scan's kernels
(hs_b200_last_kernel_ms).  One JSON line per database and corpus, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402


def expressions(n, seed=4):
    """a prefix of three letters, a counted class and a repeated suffix: 8-60 positions each"""
    rng = np.random.default_rng(seed)
    out, samples = [], []
    for _ in range(n):
        pre = bytes(rng.choice(list(b"abcdefghijklmnopqrstuvwxyz"), size=3).tolist())
        lo = int(rng.integers(3, 12))
        hi = lo + int(rng.integers(0, 45))
        out.append(pre + b"[0-9a-f]{%d,%d}[xyz]+" % (lo, hi))
        samples.append(pre + bytes(rng.choice(list(b"0123456789abcdef"), size=hi).tolist()) + b"x")
    return out, samples


def groups(exprs):
    out = [[]]
    for i, e in enumerate(exprs):
        trial = out[-1] + [i]
        try:
            fits = capi.compile_multi([exprs[k] for k in trial], [0] * len(trial), trial).info().runtime_impl == 2
        except capi.HsError:
            fits = False
        if fits or not out[-1]:
            out[-1] = trial
        else:
            out.append([i])
    return out


def _time(db, corpus, reps):
    scratch = capi.Scratch(db)
    ms = []
    for i in range(2 + reps):
        capi.scan_corpus(db, corpus, scratch, fetch=False)
        if i >= 2:
            ms.append(scratch.last_kernel_ms())
    n = len(capi.scan_corpus(db, corpus, scratch))   # delivered matches
    scratch.free()
    return float(np.median(ms)), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=1024)
    ap.add_argument("--small", type=int, default=4096, help="blocks of the small corpus")
    ap.add_argument("--block-len", type=int, default=1024)
    ap.add_argument("--exprs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    exprs, samples = expressions(args.exprs)
    ids = list(range(len(exprs)))
    whole = capi.compile_multi(exprs, [0] * len(exprs), ids)
    info = whole.info()
    assert info.runtime_impl == 0 and info.engine_count >= 2, "the set fits one engine: raise --exprs"
    parts = groups(exprs)
    assert len(parts) == info.engine_count
    dbs = [("group%d" % g, capi.compile_multi([exprs[k] for k in p], [0] * len(p), p)) for g, p in enumerate(parts)]
    dbs.append(("whole", whole))
    bl = args.block_len
    ok = True
    for nb in ((args.mb << 20) // bl, args.small):
        data, off, ln, _ = synth.block_corpus(nb, bl, samples, plant_per_kb=0.5, seed=7)
        corpus = capi.Corpus.upload(data, off, ln)
        total_ms, total_n = 0.0, 0
        for name, db in dbs:
            ms, n = _time(db, corpus, args.reps)
            if name != "whole":
                total_ms += ms
                total_n += n
            else:
                ok &= n == total_n
            print(json.dumps({"db": name, "engines": db.info().engine_count, "engine_id": db.info().engine_id,
                              "blocks": nb, "block_len": bl, "kernel_ms": round(ms, 4),
                              "GBps": round(nb * bl / (ms * 1e-3) / 1e9, 1), "records": n}), flush=True)
        print(json.dumps({"blocks": nb, "sum_of_groups_ms": round(total_ms, 4)}), flush=True)
        corpus.free()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card, "records_match": bool(ok)}))


if __name__ == "__main__":
    main()
