#!/usr/bin/env python
"""Literals AND regular expressions in one database (a literal matcher beside one engine run as an outfix,
DESIGN.md section 10d) on a resident corpus of uniform blocks: kernel ms of the literal pass, the engine pass
and the whole scan (run on the GPU box):  python tools/mixed_bench.py [--mb 1024] [--lits 1000]

The two passes are timed as the two halves compiled alone -- the literals as a pure-literal database, the
regexes as a single-outfix one -- over the same corpus; the whole scan is the mixed database.  Each figure is
the median of --reps scans after two warm-up scans, from the library's CUDA events around the scan's kernels
(hs_b200_last_kernel_ms).  One JSON line per database, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402

REGEXES = [rb"ab+c", rb"\d+\.\d\d", rb"x.y", rb"fo{2,}ba[rz]"]


def _esc(lit):
    return b"".join(bytes([c]) if chr(c).isalnum() else b"\\x%02x" % c for c in lit)


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
    ap.add_argument("--block-len", type=int, default=1024)
    ap.add_argument("--lits", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    bl = args.block_len
    nb = (args.mb << 20) // bl
    lits, flags, ids = synth.literal_set(args.lits, seed=2)
    data, off, ln, _ = synth.block_corpus(nb, bl, lits, plant_per_kb=0.5, seed=7)
    corpus = capi.Corpus.upload(data, off, ln)
    rids = list(range(100000, 100000 + len(REGEXES)))
    dbs = {"literal_pass": capi.compile_multi([_esc(l) for l in lits], flags, ids),
           "engine_pass": capi.compile_multi(REGEXES, [0] * len(REGEXES), rids),
           "mixed": capi.compile_multi([_esc(l) for l in lits] + REGEXES, list(flags) + [0] * len(REGEXES),
                                       list(ids) + rids)}
    assert dbs["mixed"].info().runtime_impl == 0 and dbs["engine_pass"].info().runtime_impl == 2
    counts = {}
    for name, db in dbs.items():
        ms, n = _time(db, corpus, args.reps)
        counts[name] = n
        info = db.info()
        print(json.dumps({"db": name, "runtime_impl": info.runtime_impl, "engine_id": info.engine_id,
                          "blocks": nb, "block_len": bl, "kernel_ms": round(ms, 4),
                          "GBps": round(nb * bl / (ms * 1e-3) / 1e9, 1), "records": n}), flush=True)
    corpus.free()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card, "records_match": counts["mixed"] == counts["literal_pass"] + counts["engine_pass"]}))


if __name__ == "__main__":
    main()
