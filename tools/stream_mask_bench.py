#!/usr/bin/env python
"""Which streams or batch rows fire which report ids in a stream-set pass: a mask pass
(hs_b200_streams_scan_mask_async / hs_b200_streams_scan_rows_mask_async) against the ordinary pass, the device
ordering and a torch reduction of the ordered matches to the same mask (DESIGN.md section 9c).  Run on an H100:
    python tools/stream_mask_bench.py [--reps 5] [--sparse-streams 20] [--dense-streams 14] [--rows 20]

Workloads, each on two stream sets fed the same passes (one per path), both reset before every run:
  sparse   (section 9a) 2^sparse-streams streams of 1 KiB writes with about one planted literal each, the config-4
           literal set of bench.py (5 000 literals of 4-8 bytes): tools/stream_set_device_bench.py's writes
  dense    (section 9a) 2^dense-streams streams of 1 KiB writes over the letters a-d, with 32 literals of 3 bytes over
           the same letters: a match at about every second byte
  rows     (section 9b) tools/stream_rows_bench.py's batch: 2^rows rows of 64-1 500 bytes over 2^16 Zipf-skewed flows
           of a 2^16-stream set, the config-4 literal set

Timed with CUDA events on one CUDA stream, one warm-up of each path (which grows the record ring and the candidate
list where a pass overflows them, and sizes the ordering's output), then --reps alternating runs, median:
  mask      the mask pass with a status word (the mask clear included)
  ordered   the ordinary pass + hs_b200_order_matches_async + the torch reduction (unique (row, id) keys, one
            index_add of their bits)
Every run checks that the two masks are equal.  One JSON line per workload, then one with the card's name and
power limit."""
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
from stream_rows_bench import make_batch  # noqa: E402
from stream_set_device_bench import PITCH, WRITE, make_writes  # noqa: E402


def dense_writes(torch, nstreams, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    alpha = torch.tensor(list(b"abcd"), dtype=torch.uint8, device="cuda")
    buf = torch.zeros((nstreams, PITCH), dtype=torch.uint8, device="cuda")
    buf[:, 16:] = alpha[torch.randint(0, 4, (nstreams, WRITE), device="cuda", generator=g)]
    return buf


def reduce_to_mask(torch, out, n, d_ids, nblocks, wpb):
    """the mask of n ordered matches in `out` (16-byte records): a bit per distinct (block, id rank)"""
    rec = out[: n * 16].view(torch.int32).view(n, 4).long()
    rank = torch.searchsorted(d_ids, rec[:, 0] & 0xffffffff)
    key = torch.unique((rec[:, 1] & 0xffffffff) * (wpb * 32) + rank)
    m = torch.zeros(nblocks * wpb, dtype=torch.int64, device="cuda")
    m.index_add_(0, key // 32, torch.ones_like(key) << (key % 32))
    return (m - (m >= (1 << 31)).long() * (1 << 32)).to(torch.int32).view(nblocks, wpb)


def run(torch, name, db, nstreams, nblocks, enqueue_mask, enqueue_pass, reps):
    """enqueue_mask(set, scratch, mask, wpb, status, stream), enqueue_pass(set, scratch, stream): one pass each"""
    ids = capi.report_ids(db)
    wpb = (ids.size + 31) // 32
    d_ids = torch.from_numpy(ids.astype(np.int64)).cuda()
    s_mask, s_ord = capi.Scratch(db), capi.Scratch(db)
    set_mask, set_ord = capi.StreamSet(db, nstreams, out_cap=1), capi.StreamSet(db, nstreams, out_cap=1)
    st = torch.cuda.Stream()
    sp = st.cuda_stream
    mask = torch.empty((nblocks, wpb), dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    cap = 1 << 20
    out, cnt = torch.empty(cap * 16, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    res = {"mask": [], "ordered": []}
    info = {}
    torch.cuda.synchronize()
    for i in range(reps + 1):
        # mask (again after a candidate-list overflow, with the list grown: the set is then marked, and the reset
        # enqueued after finish, in the next epoch, commits)
        for attempt in range(4):
            set_mask.reset_async(None, stream=sp)
            ev[0].record(st)
            enqueue_mask(set_mask, s_mask, mask, wpb, status, sp)
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
        # ordinary pass + device ordering + torch reduction; the warm-up grows the ring (again after an overflow)
        # and the output, and finds the count, which every run then reduces and checks
        for attempt in range(4 if i == 0 else 1):
            set_ord.reset_async(None, stream=sp)
            ev[0].record(st)
            enqueue_pass(set_ord, s_ord, sp)
            capi.order_matches_async(db, s_ord, out, cnt, stream=sp)
            if i:
                with torch.cuda.stream(st):
                    want = reduce_to_mask(torch, out, info["delivered"], d_ids, nblocks, wpb)
            ev[1].record(st)
            st.synchronize()
            rc, nrec, _ = capi.scan_corpus_finish(s_ord)
            n = int(cnt.cpu().numpy().view(np.uint64)[0])
            if rc == capi.HS_SUCCESS and n <= cap:
                break
            if n != capi.ORDER_RING_OVERFLOW and n > cap:
                cap = n + n // 4
                out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
        assert rc == capi.HS_SUCCESS and n <= cap
        if i == 0:
            info.update({"ordered_rescans_first_run": attempt, "records": int(nrec), "delivered": n})
            with torch.cuda.stream(st):   # the reduction's first call too is warm-up
                reduce_to_mask(torch, out, n, d_ids, nblocks, wpb)
            st.synchronize()
            continue
        assert n == info["delivered"]
        res["ordered"].append(ev[0].elapsed_time(ev[1]))
        assert torch.equal(mask, want), "the masks differ"
    set_mask.close()
    set_ord.close()
    med = {k: float(np.median(v)) for k, v in res.items()}
    return dict({"workload": name, "streams": nstreams, "mask_rows": nblocks, "ids": int(ids.size),
                 "words_per_row": wpb, "mask_bytes": nblocks * wpb * 4, "ms_median": med, "ms": res, "reps": reps,
                 "mask_speedup": med["ordered"] / med["mask"], "identical": True}, **info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sparse-streams", type=int, default=20, help="log2")
    ap.add_argument("--dense-streams", type=int, default=14, help="log2")
    ap.add_argument("--rows", type=int, default=20, help="log2 of the rows pass's batch")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    lits, flags, ids = synth.literal_set(5000, min_len=4, max_len=8, caseless_frac=0.1, seed=4)
    db = capi.compile_lit_multi(lits, flags, ids, mode=capi.HS_MODE_STREAM)

    def pitched(buf):
        return (lambda s, scr, m, w, stat, sp: s.scan_mask_async(buf, PITCH, WRITE, scr, m, w, stat, stream=sp),
                lambda s, scr, sp: s.scan_async(buf, PITCH, WRITE, scr, stream=sp))

    n = 1 << args.sparse_streams
    buf = make_writes(torch, lits, n, seed=args.sparse_streams)
    print(json.dumps(run(torch, "sparse", db, n, n, *pitched(buf), args.reps)), flush=True)
    del buf
    rng = np.random.default_rng(5)
    dense = sorted({bytes(rng.choice(list(b"abcd"), size=3).astype(np.uint8)) for _ in range(200)})[:32]
    dense_db = capi.compile_lit_multi(dense, [0] * len(dense), list(range(len(dense))), mode=capi.HS_MODE_STREAM)
    n = 1 << args.dense_streams
    buf = dense_writes(torch, n, seed=args.dense_streams)
    print(json.dumps(run(torch, "dense", dense_db, n, n, *pitched(buf), args.reps)), flush=True)
    del buf
    nrows, nflows, nstreams = 1 << args.rows, 1 << 16, 1 << 16
    chars, d_off, sids, _ = make_batch(torch, lits, nrows, nflows, nstreams, 0.7, seed=16)
    d_sids = torch.from_numpy(sids.astype(np.int32)).cuda()
    print(json.dumps(run(torch, "rows", db, nstreams, nrows,
                         lambda s, scr, m, w, stat, sp: s.scan_rows_mask_async(chars, d_off, d_sids, scr, m, w, stat,
                                                                               stream=sp),
                         lambda s, scr, sp: s.scan_rows_async(chars, d_off, d_sids, scr, stream=sp), args.reps)),
          flush=True)
    print(json.dumps({"gpu": card}), flush=True)


if __name__ == "__main__":
    main()
