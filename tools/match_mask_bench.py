#!/usr/bin/env python
"""Which rows match which ids: a match-mask pass (hs_b200_scan_rows_mask_async) against the ordinary pass and the
device ordering (hs_b200_scan_rows_async + hs_b200_order_matches_async), over a column of rows in device memory.
Run on the GPU box:
    python tools/match_mask_bench.py [--gib 1] [--dense-gib 0.25] [--reps 5]

Workloads (DESIGN.md section 10h), columns of rows of 20-2 000 bytes as tools/scan_rows_bench.py makes them:
  literals  bench.py's literal set (1 000 literals of 4-8 bytes, 10 % caseless), --gib GiB: sparse
  regex5    bench.py's 5-expression database (one McClellan engine), --gib GiB: sparse
  dense     [0-9]+ (one McClellan engine), --dense-gib GiB: a match at every digit, about one byte in six

Timed with CUDA events on one CUDA stream, one warm-up of each path (which also grows the record ring where the
ordinary pass overflows it), then --reps alternating runs, median:
  mask      scan_rows_mask_async with a status word
  ordered   scan_rows_async + order_matches_async
Every run checks that the mask equals the one built from the ordered matches.  One JSON line per workload, then
one with the card's name and power limit."""
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
from scan_rows_bench import REGEX5, REGEX5_PLANT, column  # noqa: E402


def mask_of(ids, recs, nrows, wpb):
    rank = np.searchsorted(ids, recs["id"])
    m = np.zeros(nrows * wpb, np.uint32)
    np.bitwise_or.at(m, recs["block"].astype(np.int64) * wpb + rank // 32, (1 << (rank % 32)).astype(np.uint32))
    return m.reshape(nrows, wpb)


def run(torch, name, db, lens, plant, reps, seed):
    chars, off, _, _, _ = column(lens, plant, seed)
    d_chars, d_off = torch.from_numpy(chars).cuda(), torch.from_numpy(off).cuda()
    nrows = off.size - 1
    ids = capi.report_ids(db)
    wpb = (ids.size + 31) // 32
    s_mask, s_ord = capi.Scratch(db), capi.Scratch(db)
    st = torch.cuda.Stream()
    sp = st.cuda_stream
    mask = torch.empty((nrows, wpb), dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    cap = 1 << 20
    out, cnt = torch.empty(cap * 16, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    res = {"mask": [], "ordered": []}
    info = {}
    torch.cuda.synchronize()
    for i in range(reps + 1):
        # mask (again after a candidate-list overflow, with the list grown)
        for attempt in range(4):
            ev[0].record(st)
            capi.scan_rows_mask_async(db, d_chars, d_off, s_mask, mask, wpb, status, stream=sp)
            ev[1].record(st)
            st.synchronize()
            rc, nrec, _ = capi.scan_corpus_finish(s_mask)
            assert (rc == capi.HS_SUCCESS) == (int(status.item()) == 0)
            if rc == capi.HS_SUCCESS:
                break
            assert rc == capi.HS_INSUFFICIENT_SPACE
        assert rc == capi.HS_SUCCESS and nrec == 0
        if i == 0:
            info["mask_rescans_first_run"] = attempt
        else:
            res["mask"].append(ev[0].elapsed_time(ev[1]))
        # scan + device ordering (again after a ring overflow, with the ring grown)
        for attempt in range(4):
            ev[0].record(st)
            capi.scan_rows_async(db, d_chars, d_off, s_ord, stream=sp)
            capi.order_matches_async(db, s_ord, out, cnt, stream=sp)
            ev[1].record(st)
            st.synchronize()
            rc, nrec, _ = capi.scan_corpus_finish(s_ord)
            n = int(cnt.cpu().numpy().view(np.uint64)[0])
            if rc == capi.HS_SUCCESS and n <= cap:
                break
            if n != capi.ORDER_RING_OVERFLOW and n > cap:
                cap = n + n // 4
                out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
        assert rc == capi.HS_SUCCESS
        if i == 0:
            info["ordered_rescans_first_run"] = attempt
            info["records"] = int(nrec)
        else:
            res["ordered"].append(ev[0].elapsed_time(ev[1]))
        recs = out[:n * 16].cpu().numpy().view(capi.MATCH_DTYPE)
        want = mask_of(ids, recs, nrows, wpb)
        assert np.array_equal(mask.cpu().numpy().view(np.uint32), want), "the masks differ"
        info["delivered"] = int(n)
    med = {k: float(np.median(v)) for k, v in res.items()}
    return dict({"workload": name, "rows": int(nrows), "chars_bytes": int(chars.size - 5), "ids": int(ids.size),
                 "ms_median": med, "reps": reps, "mask_speedup": med["ordered"] / med["mask"],
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
    rng = np.random.default_rng(1)
    lens = rng.integers(20, 2001, size=int(args.gib * (1 << 30) / 1010))
    dense = rng.integers(20, 2001, size=int(args.dense_gib * (1 << 30) / 1010))
    for name, db, ln, plant in (("literals", lit_db, lens, lits[:200]), ("regex5", rx_db, lens, REGEX5_PLANT),
                                ("dense", dense_db, dense, [b"0"])):
        print(json.dumps(run(torch, name, db, ln, plant, args.reps, seed=3)), flush=True)
    print(json.dumps({"gpu": card}), flush=True)


if __name__ == "__main__":
    main()
