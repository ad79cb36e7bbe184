#!/usr/bin/env python
"""The first match of every row: a first-match pass (hs_b200_scan_rows_first_async) against the mask pass
(hs_b200_scan_rows_mask_async) and the ordinary pass, the device ordering and a torch reduction to the first match
per row (hs_b200_scan_rows_async + hs_b200_order_matches_async + scatter_reduce), over a column of rows in device
memory.  Run on the GPU box:
    python tools/first_match_bench.py [--gib 1] [--dense-gib 0.25] [--reps 5]

Workloads (DESIGN.md section 10i), columns of rows of 20-2 000 bytes as tools/scan_rows_bench.py makes them -- the
workloads of tools/match_mask_bench.py, and the expression set of tools/multi_outfix_bench.py:
  literals  bench.py's literal set (1 000 literals of 4-8 bytes, 10 % caseless), --gib GiB: sparse
  regex5    bench.py's 5-expression database (one McClellan engine), --gib GiB: sparse
  dense     [0-9]+ (one McClellan engine), --dense-gib GiB: a match at every digit, about one byte in six
  outfix64  64 expressions split over several engines (section 10e), --gib GiB

Timed with CUDA events on one CUDA stream, one warm-up of each path (which also grows the candidate list and the
record ring where a pass overflows them), then --reps alternating runs, median:
  first     scan_rows_first_async with a status word
  mask      scan_rows_mask_async with a status word
  ordered   scan_rows_async + order_matches_async, the record count read back, a scatter_reduce to the first
            match per row
Every run checks that the first-match table equals the reduction of the ordered matches and that the rows it marks
are the rows the mask marks.  One JSON line per workload, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hyperscan_b200 import capi, synth  # noqa: E402
from multi_outfix_bench import expressions  # noqa: E402
from scan_rows_bench import REGEX5, REGEX5_PLANT, column  # noqa: E402

INT64_MAX = (1 << 63) - 1


def first_of(torch, out, n, nrows):
    """the first (to << 32) | id per row of n ordered records, -1 where a row has none"""
    rec = out[:n * 16].view(torch.int32).view(n, 4).long()
    key = (rec[:, 2] << 32) | (rec[:, 0] & 0xFFFFFFFF)
    first = torch.full((nrows,), INT64_MAX, dtype=torch.int64, device=out.device)
    first.scatter_reduce_(0, rec[:, 1], key, "amin")
    return first.masked_fill_(first == INT64_MAX, -1)


def _pass(capi_call, scratch, st, ev, status):
    """one pass timed, again after a candidate-list overflow (the list grown): (ms, attempts)"""
    for attempt in range(4):
        ev[0].record(st)
        capi_call()
        ev[1].record(st)
        st.synchronize()
        rc, nrec, _ = capi.scan_corpus_finish(scratch)
        assert (rc == capi.HS_SUCCESS) == (int(status.item()) == 0)
        if rc == capi.HS_SUCCESS:
            assert nrec == 0
            return ev[0].elapsed_time(ev[1]), attempt
        assert rc == capi.HS_INSUFFICIENT_SPACE
    raise AssertionError("the pass did not succeed")


def run(torch, name, db, lens, plant, reps, seed):
    chars, off, _, _, _ = column(lens, plant, seed)
    d_chars, d_off = torch.from_numpy(chars).cuda(), torch.from_numpy(off).cuda()
    nrows = off.size - 1
    wpb = (capi.report_ids(db).size + 31) // 32
    s_first, s_mask, s_ord = capi.Scratch(db), capi.Scratch(db), capi.Scratch(db)
    st = torch.cuda.Stream()
    sp = st.cuda_stream
    first = torch.empty(nrows, dtype=torch.int64, device="cuda")
    mask = torch.empty((nrows, wpb), dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    cap = 1 << 20
    out, cnt = torch.empty(cap * 16, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    res = {"first": [], "mask": [], "ordered": []}
    info = {}
    torch.cuda.synchronize()
    for i in range(reps + 1):
        ms, attempt = _pass(lambda: capi.scan_rows_first_async(db, d_chars, d_off, s_first, first, status, stream=sp),
                            s_first, st, ev, status)
        if i == 0:
            info["first_rescans_first_run"] = attempt
        else:
            res["first"].append(ms)
        ms, attempt = _pass(lambda: capi.scan_rows_mask_async(db, d_chars, d_off, s_mask, mask, wpb, status,
                                                              stream=sp), s_mask, st, ev, status)
        if i == 0:
            info["mask_rescans_first_run"] = attempt
        else:
            res["mask"].append(ms)
        # scan + device ordering + reduction (again after a ring overflow, with the ring grown)
        for attempt in range(4):
            ev[0].record(st)
            capi.scan_rows_async(db, d_chars, d_off, s_ord, stream=sp)
            capi.order_matches_async(db, s_ord, out, cnt, stream=sp)
            with torch.cuda.stream(st):
                n = int(cnt.item()) & 0xFFFFFFFFFFFFFFFF   # (a host wait: the reduction needs the count)
                ok = n != capi.ORDER_RING_OVERFLOW and n <= cap
                want = first_of(torch, out, n, nrows) if ok else None
            ev[1].record(st)
            st.synchronize()
            rc, nrec, _ = capi.scan_corpus_finish(s_ord)
            if rc == capi.HS_SUCCESS and ok:
                break
            if n != capi.ORDER_RING_OVERFLOW and n > cap:
                cap = n + n // 4
                out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
        assert rc == capi.HS_SUCCESS
        if i == 0:
            info["ordered_rescans_first_run"] = attempt
            info["records"] = int(nrec)
            info["delivered"] = n
        else:
            res["ordered"].append(ev[0].elapsed_time(ev[1]))
        assert torch.equal(first, want), "the first-match tables differ"
        assert torch.equal(first != -1, mask.ne(0).any(dim=1)), "the first-match table and the mask differ"
    info["rows_matching"] = int((first != -1).sum().item())
    med = {k: float(np.median(v)) for k, v in res.items()}
    return dict({"workload": name, "rows": int(nrows), "chars_bytes": int(chars.size - 5),
                 "engines": int(db.info().engine_count), "ms_median": med, "reps": reps,
                 "first_vs_mask": med["mask"] / med["first"], "first_vs_ordered": med["ordered"] / med["first"],
                 "identical": True}, **info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--dense-gib", type=float, default=0.25)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    capi.lib()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    lits, flags, ids = synth.literal_set(1000, min_len=4, max_len=8, caseless_frac=0.1, seed=2)
    lit_db = capi.compile_lit_multi(lits, flags, ids)
    rx_db = capi.compile_multi(REGEX5, [0, 0, 0, capi.HS_FLAG_CASELESS, 0], list(range(1, len(REGEX5) + 1)))
    dense_db = capi.compile_multi([rb"[0-9]+"], [0], [1])
    exprs, samples = expressions(64)
    multi_db = capi.compile_multi(exprs, [0] * len(exprs), list(range(len(exprs))))
    rng = np.random.default_rng(1)
    lens = rng.integers(20, 2001, size=int(args.gib * (1 << 30) / 1010))
    dense = rng.integers(20, 2001, size=int(args.dense_gib * (1 << 30) / 1010))
    for name, db, ln, plant in (("literals", lit_db, lens, lits[:200]), ("regex5", rx_db, lens, REGEX5_PLANT),
                                ("dense", dense_db, dense, [b"0"]), ("outfix64", multi_db, lens, samples)):
        print(json.dumps(run(torch, name, db, ln, plant, args.reps, seed=3)), flush=True)
    print(json.dumps({"gpu": card}), flush=True)


if __name__ == "__main__":
    main()
