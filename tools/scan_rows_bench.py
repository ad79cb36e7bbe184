#!/usr/bin/env python
"""A column of rows already in device memory (chars + int64 offsets, rows at any byte), scanned by
hs_b200_scan_rows_async and ordered on the device, against the same rows scanned as a packed, wrapped corpus.
Run on the GPU box:
    python tools/scan_rows_bench.py [--gib 1] [--reps 5]

Workloads (DESIGN.md section 10g):
  literals  bench.py's literal set (1 000 literals of 4-8 bytes, 10 % caseless) over a column of --gib GiB whose
            rows are 20-2 000 bytes long, about one planted literal per 4 KiB
  regex5    bench.py's 5-expression database (one McClellan engine) over the same kind of column
  regex5_long  the same database over 8 rows of 16 MiB: the engine runs cut the rows into segments

Timed, alternating, after one warm-up of each (CUDA events on one CUDA stream, median of --reps):
  rows      scan_rows_async (row plan, repack, scan) and order_matches_async; the scan kernels' share is
            hs_b200_last_kernel_ms, the rest of the pass before the ordering is the plan and the repack
  packed    (a) the same rows already packed at 16-byte aligned starts and wrapped with host tables:
            scan_corpus_async and order_matches_async
  roundtrip (b) what a caller does today, host clock: the offsets to the host (a synchronisation), the packed
            table computed on the host, hs_b200_corpus_wrap of a buffer packed beforehand (the caller's own repack
            kernel is not counted), the scan and the ordering, then a synchronisation
Every pass's ordered matches must equal the packed pass's, record for record.  One JSON line per workload, then
one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402

REGEX5 = [rb"ab+c", rb"[0-9]{2,}\.[0-9]", rb"^GET\s", rb"(foo|bar)x*z", rb"q.{2,4}w$"]
REGEX5_PLANT = [b"abbbc", b"123.4", b"GET /", b"fooxxz", b"q123w"]


def column(lengths, plant, seed):
    """host chars of the rows back to back after 5 bytes, a literal of `plant` about every 4 KiB; offsets;
    the packed copy (16-byte aligned starts) and its table"""
    rng = np.random.default_rng(seed)
    lens = np.asarray(lengths, dtype=np.int64)
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 ./-", np.uint8)
    total = 5 + int(lens.sum())
    chars = np.empty(total, np.uint8)
    for c0 in range(0, total, 1 << 26):
        c1 = min(total, c0 + (1 << 26))
        chars[c0:c1] = alpha[rng.integers(0, alpha.size, size=c1 - c0)]
    for at, k in zip(rng.integers(5, total - 16, size=total // 4096), rng.integers(0, len(plant), size=total // 4096)):
        lit = plant[int(k)]
        chars[int(at):int(at) + len(lit)] = np.frombuffer(lit, np.uint8)
    off = np.concatenate([[5], 5 + np.cumsum(lens)]).astype(np.int64)
    pad = np.maximum(16, (lens + 15) // 16 * 16)
    pstart = np.concatenate([[0], np.cumsum(pad)[:-1]]).astype(np.int64)
    packed = np.zeros(int(pad.sum()) + 64, np.uint8)
    step = 1 << 16
    for r0 in range(0, lens.size, step):
        r1 = min(lens.size, r0 + step)
        n = int(lens[r0:r1].sum())
        src = np.arange(off[r0], off[r0] + n, dtype=np.int64)
        dst = np.repeat(pstart[r0:r1] - off[r0:r1], lens[r0:r1]) + src
        packed[dst] = chars[src]
    return chars, off, packed, pstart.astype(np.uint64), lens.astype(np.uint32)


def host_table(off):
    lens = np.diff(off)
    pad = np.maximum(16, (lens + 15) // 16 * 16)
    return np.concatenate([[0], np.cumsum(pad)[:-1]]).astype(np.uint64), lens.astype(np.uint32)


def read(torch, out, cnt):
    n = int(cnt.cpu().numpy().view(np.uint64)[0])
    assert n != capi.ORDER_RING_OVERFLOW
    return out[:n * 16].cpu().numpy().view(capi.MATCH_DTYPE)


def run(torch, name, db, lens, plant, reps, seed):
    lens = np.asarray(lens, dtype=np.int64)
    chars, off, packed, pstart, plen = column(lens, plant, seed)
    d_chars, d_off = torch.from_numpy(chars).cuda(), torch.from_numpy(off).cuda()
    d_packed = torch.from_numpy(packed).cuda()
    corpus = capi.Corpus.wrap(d_packed.data_ptr(), packed.size, pstart, plen, keep=d_packed)
    s_rows, s_packed, s_trip = capi.Scratch(db), capi.Scratch(db), capi.Scratch(db)
    st = torch.cuda.Stream()
    sp = st.cuda_stream
    cap = 1 << 22
    outs = {k: (torch.empty(cap * 16, dtype=torch.uint8, device="cuda"),
                torch.zeros(1, dtype=torch.int64, device="cuda")) for k in ("rows", "packed", "trip")}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    res = {"rows_pass": [], "rows_scan": [], "rows_e2e": [], "packed_e2e": [], "packed_scan": [], "trip_e2e": []}

    torch.cuda.synchronize()
    for i in range(reps + 1):
        # rows
        for _ in range(2):      # (a second pass only when the ring had to grow)
            ev[0].record(st)
            capi.scan_rows_async(db, d_chars, d_off, s_rows, stream=sp)
            ev[1].record(st)
            capi.order_matches_async(db, s_rows, *outs["rows"], stream=sp)
            ev[2].record(st)
            st.synchronize()
            rc, _, _ = capi.scan_corpus_finish(s_rows)
            if rc == capi.HS_SUCCESS:
                break
        if i:
            res["rows_pass"].append(ev[0].elapsed_time(ev[1]))
            res["rows_e2e"].append(ev[0].elapsed_time(ev[2]))
            res["rows_scan"].append(s_rows.last_kernel_ms())
        # (a) packed and wrapped
        for _ in range(2):
            ev[0].record(st)
            capi.scan_corpus_async(db, corpus, s_packed, stream=sp)
            capi.order_matches_async(db, s_packed, *outs["packed"], stream=sp)
            ev[2].record(st)
            st.synchronize()
            rc, _, _ = capi.scan_corpus_finish(s_packed)
            if rc == capi.HS_SUCCESS:
                break
        if i:
            res["packed_e2e"].append(ev[0].elapsed_time(ev[2]))
            res["packed_scan"].append(s_packed.last_kernel_ms())
        # (b) the round trip through the host
        for _ in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.cuda.stream(st):
                h_off = d_off.cpu()                               # synchronises
            ps, pl = host_table(h_off.numpy())
            c2 = capi.Corpus.wrap(d_packed.data_ptr(), packed.size, ps, pl, keep=d_packed)
            capi.scan_corpus_async(db, c2, s_trip, stream=sp)
            capi.order_matches_async(db, s_trip, *outs["trip"], stream=sp)
            st.synchronize()
            t1 = time.perf_counter()
            rc, _, _ = capi.scan_corpus_finish(s_trip)
            c2.free()
            if rc == capi.HS_SUCCESS:
                break
        if i:
            res["trip_e2e"].append((t1 - t0) * 1e3)
        a, b, c = (read(torch, *outs[k]) for k in ("rows", "packed", "trip"))
        assert np.array_equal(a, b) and np.array_equal(a, c), "the match lists differ"
    med = {k: float(np.median(v)) for k, v in res.items()}
    med["rows_plan_repack"] = float(np.median(np.array(res["rows_pass"]) - np.array(res["rows_scan"])))
    return {"workload": name, "rows": int(lens.size), "chars_bytes": int(chars.size - 5),
            "matches": int(a.size), "ms_median": med, "reps": reps,
            "gbs_rows_e2e": (chars.size - 5) / (med["rows_e2e"] * 1e-3) / 1e9, "identical": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    capi.lib()
    lits, flags, ids = synth.literal_set(1000, min_len=4, max_len=8, caseless_frac=0.1, seed=2)
    lit_db = capi.compile_lit_multi(lits, flags, ids)
    rx_db = capi.compile_multi(REGEX5, [0, 0, 0, capi.HS_FLAG_CASELESS, 0], list(range(1, len(REGEX5) + 1)))
    rng = np.random.default_rng(1)
    want = int(args.gib * (1 << 30))
    lens = rng.integers(20, 2001, size=int(want / 1010))
    for name, db, ln, plant in (("literals", lit_db, lens, lits[:200]), ("regex5", rx_db, lens, REGEX5_PLANT),
                                ("regex5_long", rx_db, [16 << 20] * 8, REGEX5_PLANT)):
        print(json.dumps(run(torch, name, db, ln, plant, args.reps, seed=3)), flush=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)


if __name__ == "__main__":
    main()
