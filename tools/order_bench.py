"""Time the delivery of ordered matches two ways over a resident corpus:

  device  hs_b200_scan_corpus_async + hs_b200_order_matches_async on one CUDA stream, timed with CUDA events
          on that stream (the matches stay in device memory; no host synchronisation inside the window)
  host    hs_b200_scan_corpus_async, hs_b200_scan_corpus_finish, hs_b200_fetch_matches (copy to the host,
          report rules and ordering on one CPU thread), timed with a host clock

for the bench workload (1 000 short literals, FDR; 1 GiB of 1 KiB blocks) and a regular-expression database,
and checks that both paths deliver the same matches.  Prints one JSON line with the card's name and power
limit.  Needs a CUDA device.

  python tools/order_bench.py [--blocks 1048576] [--block-len 1024] [--iters 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REGEXES = [rb"ab+c", rb"[0-9]+x", rb"q[a-f]{2,5}z", rb"foo.*bar", rb"\bzz[a-c]\b", rb"k[^a]y$"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:   # the timing stands without it, but says so
        return {"name": "unknown", "power_limit": "unknown", "error": str(e)}


def run(capi, torch, name, db, corpus, iters):
    scratch = capi.Scratch(db)
    n = capi.scan_corpus(db, corpus, scratch, fetch=False)      # grows the ring to fit
    want = capi.fetch_matches(db, scratch)
    cap = want.size + 1024
    out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def device_pass():
        capi.scan_corpus_async(db, corpus, scratch, stream=s)
        capi.order_matches_async(db, scratch, out, cnt, stream=s)

    with torch.cuda.stream(stream):
        for _ in range(3):
            device_pass()
        stream.synchronize()
        capi.scan_corpus_finish(scratch)
        scan_only = []
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        for _ in range(iters):
            device_pass()
        t1.record(stream)
        stream.synchronize()
        device_ms = t0.elapsed_time(t1) / iters
        # the scan alone on the same stream, for the ordering's share
        t0.record(stream)
        for _ in range(iters):
            capi.scan_corpus_async(db, corpus, scratch, stream=s)
        t1.record(stream)
        stream.synchronize()
        scan_ms = t0.elapsed_time(t1) / iters
        capi.scan_corpus_finish(scratch)
        device_pass()
        stream.synchronize()
    got_n = int(cnt.item())
    got = out[: 16 * min(got_n, cap)].cpu().numpy().view(capi.MATCH_DTYPE)
    capi.scan_corpus_finish(scratch)
    for _ in range(2):
        capi.scan_corpus(db, corpus, scratch)
    t = time.perf_counter()
    for _ in range(iters):
        host = capi.scan_corpus(db, corpus, scratch)
    host_ms = (time.perf_counter() - t) * 1e3 / iters
    return {"database": name, "raw_records": int(n), "delivered": int(want.size),
            "device_scan_plus_order_ms": round(device_ms, 4), "device_scan_only_ms": round(scan_ms, 4),
            "device_order_ms": round(device_ms - scan_ms, 4),
            "host_scan_finish_fetch_ms": round(host_ms, 4),
            "identical": bool(got_n == host.size and np.array_equal(got, host) and np.array_equal(host, want))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1 << 20)
    ap.add_argument("--block-len", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("order_bench.py needs a CUDA device")
    from hyperscan_b200 import build, capi, synth
    build.build_product()
    lits, flags, ids = synth.literal_set(1000, min_len=4, max_len=8, caseless_frac=0.1, seed=2)
    data, off, ln, _ = synth.block_corpus(args.blocks, args.block_len, lits, plant_per_kb=0.01, seed=7)
    corpus = capi.Corpus.upload(data, off, ln)
    rows = [run(capi, torch, "1000 literals (FDR)", capi.compile_lit_multi(lits, flags, ids), corpus, args.iters),
            run(capi, torch, "6 regular expressions", capi.compile_multi(REGEXES), corpus, args.iters)]
    res = {"tool": "order_bench", "corpus_bytes": int(ln.sum()), "blocks": int(ln.size), "card": card(),
           "results": rows}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
