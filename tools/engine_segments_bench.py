#!/usr/bin/env python
"""Engine runs over long blocks (DESIGN.md section 10f): GB/s of one large buffer and of 1 MiB blocks, segmented by
the default rule, and of the one-lane walk of one buffer (engine_segment=-1), for the databases below (run on the GPU
box):
    python tools/engine_segments_bench.py [--big-mb 1024] [--wrong-mb 64] [--base-mb 64] [--reps 3]

The segmented figures are the median of --reps scans after one warm-up scan; the one-lane walk, seconds per scan,
is timed once.  Kernel time from the library's CUDA events around the scan's kernels (hs_b200_last_kernel_ms).  The
matches of the segmented and the one-lane runs are compared on the --base-mb buffer.  The corpus is random bytes of
ALPHA with a planted sample every 4 KiB; the wrong-guess set has its own alphabet (no X, no o) with `foo` only at
offset 0, so that every guess past its first segment is wrong, and its shapes are --wrong-mb large (its walk is
sequential).  One JSON line per database and shape, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi  # noqa: E402

ALPHA = b"abcdefghijklmnopqrstuvwxyz0123456789 ./GETqwXfoo"
WRONG_ALPHA = b"abcdefghijklmnpqrstuvwxyz0123456789 ./"
# name -> (expressions, flags, regex_dfa, planted samples)
SETS = {
    "mcclellan8_5": ([rb"ab+c", rb"[0-9]{2,}\.[0-9]", rb"^GET\s", rb"(foo|bar)x*z", rb"q.{2,4}w$"],
                     [0, 0, 0, capi.HS_FLAG_CASELESS, 0], 1, [b"abbbc", b"123.4", b"GET /", b"fooxxz", b"q123w"]),
    "mcclellan16": ([rb"q[a-d]{300}z"], [0], 1, [b"q" + b"abcd" * 75 + b"z"]),
    "limex128": ([rb"a[a-f0-9]{60}z", rb"x[0-9]{2,30}y"], [0, 0], 0, [b"a" + b"0a" * 30 + b"z", b"x1234y"]),
    "limex512": ([rb"q[a-d0-3]{270}z", rb"ab+c"], [0, 0], 0, [b"q" + b"a0" * 135 + b"z", b"abbc"]),
    "wrong_guess": ([rb"foo[^X]*bar"], [0], 1, [b"bar"]),
}


def corpus_bytes(total, seed, samples, alpha=ALPHA):
    rng = np.random.default_rng(seed)
    d = rng.choice(np.frombuffer(alpha, np.uint8), size=total)
    for p in rng.integers(0, total - 600, size=total // 4096).tolist():
        s = samples[p % len(samples)]
        d[p:p + len(s)] = np.frombuffer(s, np.uint8)
    d[:3] = np.frombuffer(b"foo", np.uint8)
    return d


def scan(db, data, nblocks, reps, seg, warmup=1):
    """median kernel ms of `reps` scans, the matches, and the segment counters of the last scan"""
    capi.set_runtime_option("engine_segment", seg)
    bl = data.size // nblocks
    off = np.arange(nblocks, dtype=np.uint64) * bl
    ln = np.full(nblocks, bl, dtype=np.uint32)
    corpus = capi.Corpus.upload(data, off, ln)
    scratch = capi.Scratch(db)
    ms = []
    for i in range(warmup + reps):
        st0 = scratch.segment_stats()
        got = capi.scan_corpus(db, corpus, scratch)
        if i >= warmup:
            ms.append(scratch.last_kernel_ms())
    st1 = scratch.segment_stats()
    corpus.free()
    scratch.free()
    capi.set_runtime_option("engine_segment", 0)
    return float(np.median(ms)), got, {k: st1[k] - st0[k] for k in st1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big-mb", type=int, default=1024)
    ap.add_argument("--wrong-mb", type=int, default=64)
    ap.add_argument("--base-mb", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sets", default=",".join(SETS))
    args = ap.parse_args()
    ok = True
    for name in args.sets.split(","):
        exprs, flags, dfa, samples = SETS[name]
        capi.set_build_option("regex_dfa", dfa)
        db = capi.compile_multi(exprs, flags, list(range(1, len(exprs) + 1)))
        capi.set_build_option("regex_dfa", 1)
        info = db.info()
        wrong = name == "wrong_guess"
        mb = args.wrong_mb if wrong else args.big_mb
        big = corpus_bytes(mb << 20, 1, samples, WRONG_ALPHA if wrong else ALPHA)
        for shape, nb in (("one_buffer", 1), ("1MiB_blocks", mb)):
            ms, got, st = scan(db, big, nb, args.reps, 0)
            print(json.dumps({"db": name, "engine_id": info.engine_id, "shape": shape, "blocks": nb,
                              "bytes": int(big.size), "kernel_ms": round(ms, 3),
                              "GBps": round(big.size / (ms * 1e-3) / 1e9, 3), "matches": int(got.size),
                              "segments": st["segments"], "rewalked_segments": st["rewalks"],
                              "rewalked_bytes": st["rewalk_bytes"]}), flush=True)
        base = big[: args.base_mb << 20].copy() if args.base_mb <= mb else corpus_bytes(
            args.base_mb << 20, 1, samples, WRONG_ALPHA if wrong else ALPHA)
        ms1, one, _ = scan(db, base, 1, 1, -1, warmup=0)
        ms2, seg, st = scan(db, base, 1, args.reps, 0)
        same = bool(np.array_equal(one, seg))
        ok &= same
        print(json.dumps({"db": name, "shape": "one_buffer_one_lane", "bytes": int(base.size),
                          "one_lane_ms": round(ms1, 3), "one_lane_GBps": round(base.size / (ms1 * 1e-3) / 1e9, 4),
                          "segmented_ms": round(ms2, 3), "segmented_GBps": round(base.size / (ms2 * 1e-3) / 1e9, 3),
                          "rewalked_segments": st["rewalks"], "rewalked_bytes": st["rewalk_bytes"],
                          "matches": int(one.size), "matches_equal": same}), flush=True)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card, "matches_equal": bool(ok)}))


if __name__ == "__main__":
    main()
