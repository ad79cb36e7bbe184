#!/usr/bin/env python
"""A stream-set pass over a batch of rows as traffic arrives (hs_b200_streams_scan_rows_async +
hs_b200_order_matches_async) against the same batch split into one-write-per-stream ticks through
hs_b200_streams_scan_async (DESIGN.md section 9b).  Run on the GPU box:
    python tools/stream_rows_bench.py [--rows 20] [--flows 16] [--streams 16,24] [--zipf 0.7] [--repeats 3]

Workload: the config-4 literal set of bench.py (5 000 literals of 4-8 bytes); a batch of 2^rows rows of 64-1 500 bytes
(random letters, about one planted literal per row) over 2^flows active flows whose ids are Zipf-skewed (P(rank k)
proportional to k^-zipf), scattered over a set of 2^streams streams.  The batch is generated on the device.

  rows pass   CUDA events on one CUDA stream around the pass and its ordering into device memory; then around the
              pass alone, of which the scan and confirm kernels take hs_b200_last_kernel_ms and the rest is the
              group, pack, rewrite and advance kernels.  Median of `repeats` runs after a warm-up, each on a freshly
              reset set.
  ticks       (sets that fit, and only the smaller set by default) tick k gives every flow its k-th row: as many
              ticks as the busiest flow has rows.  Each tick's pitched buffer is assembled on the device outside the
              timed window; CUDA events time each tick's scan_async + order_matches_async, summed over the ticks.

Both paths' ordered matches are compared: the ticks' (stream, to, id) mapped back to rows must equal the rows pass's
(row, to, id), record for record.  One JSON line per set size, then one with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402

MIN_ROW, MAX_ROW = 64, 1500


def make_batch(torch, lits, nrows, nflows, nstreams, zipf, seed):
    """chars (device), offsets (device int64, nrows + 1), stream ids (host and device), row lengths (host)"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(MIN_ROW, MAX_ROW + 1, size=nrows).astype(np.int64)
    p = np.arange(1, nflows + 1, dtype=np.float64) ** -zipf
    rank = rng.choice(nflows, size=nrows, p=p / p.sum())
    flows = rng.choice(nstreams, size=nflows, replace=False)
    sids = flows[rank].astype(np.int64)
    off = np.zeros(nrows + 1, dtype=np.int64)
    off[1:] = np.cumsum(lens)
    total = int(off[-1])
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    alpha = torch.tensor(list(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 ./-"),
                         dtype=torch.uint8, device="cuda")
    chars = torch.empty(total, dtype=torch.uint8, device="cuda")
    for s in range(0, total, 1 << 28):
        e = min(total, s + (1 << 28))
        chars[s:e] = alpha[torch.randint(0, alpha.numel(), (e - s,), device="cuda", generator=g)]
    table = torch.zeros(len(lits), 8, dtype=torch.uint8)
    for i, x in enumerate(lits):
        table[i, :len(x)] = torch.tensor(list(x), dtype=torch.uint8)
    table = table.cuda()
    llen = torch.tensor([len(x) for x in lits], dtype=torch.int64, device="cuda")
    which = torch.randint(0, len(lits), (nrows,), device="cuda", generator=g)
    d_off = torch.from_numpy(off).cuda()
    d_len = torch.from_numpy(lens).cuda()
    at = d_off[:-1] + (torch.rand(nrows, device="cuda", generator=g) * (d_len - 8).double()).long()
    for b in range(8):
        keep = llen[which] > b
        chars[at[keep] + b] = table[which[keep], b]
    return chars, d_off, sids, lens


def rows_pass(torch, db, sset, scratch, chars, d_off, d_ids, out, cnt, stream, ev):
    sset.reset_async(None, stream=stream.cuda_stream)
    for _ in range(3):
        ev[0].record(stream)
        sset.scan_rows_async(chars, d_off, d_ids, scratch, stream=stream.cuda_stream)
        capi.order_matches_async(db, scratch, out, cnt, stream=stream.cuda_stream)
        ev[1].record(stream)
        ev[1].synchronize()
        rc, _, _ = capi.scan_corpus_finish(scratch)
        if rc != capi.HS_INSUFFICIENT_SPACE:
            break
        sset.reset_async(None, stream=stream.cuda_stream)
    assert rc == capi.HS_SUCCESS, rc
    return ev[0].elapsed_time(ev[1])


def pass_only(torch, sset, scratch, chars, d_off, d_ids, stream, ev):
    """the pass alone, and of it the scan and confirm kernels (hs_b200_last_kernel_ms): the rest is the group, pack,
    rewrite and advance kernels"""
    sset.reset_async(None, stream=stream.cuda_stream)
    ev[0].record(stream)
    sset.scan_rows_async(chars, d_off, d_ids, scratch, stream=stream.cuda_stream)
    ev[1].record(stream)
    ev[1].synchronize()
    assert capi.scan_corpus_finish(scratch)[0] == capi.HS_SUCCESS
    return ev[0].elapsed_time(ev[1]), scratch.last_kernel_ms()


def ticks(torch, db, sset, scratch, chars, d_off, sids, lens, nstreams, stream, check):
    """the batch as one-write-per-stream ticks; returns (summed tick ms, ordered matches as (row, to, id) or None)"""
    nrows = sids.size
    order = np.argsort(sids, kind="stable")
    first = np.r_[0, np.flatnonzero(np.diff(sids[order])) + 1]
    rank = np.empty(nrows, dtype=np.int64)
    grp = np.repeat(np.arange(first.size), np.diff(np.r_[first, nrows]))
    rank[order] = np.arange(nrows) - first[grp]
    nticks = int(rank.max()) + 1
    pitch = 16 + (MAX_ROW + 15) // 16 * 16
    buf = torch.empty(nstreams * pitch, dtype=torch.uint8, device="cuda")
    d_lens = torch.zeros(nstreams, dtype=torch.int32, device="cuda")
    by_tick = np.argsort(rank, kind="stable")
    tick_start = np.searchsorted(rank[by_tick], np.arange(nticks + 1))
    d_by_tick = torch.from_numpy(by_tick).cuda()
    d_sids = torch.from_numpy(sids).cuda()
    d_lens_all = torch.from_numpy(lens).cuda()
    cap = 1 << 20
    out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sset.reset_async(None, stream=stream.cuda_stream)
    total_ms, got = 0.0, []
    for k in range(nticks):
        rows = d_by_tick[tick_start[k]:tick_start[k + 1]]
        with torch.cuda.stream(stream):
            d_lens.zero_()
            d_lens[d_sids[rows]] = d_lens_all[rows].int()
            rl = d_lens_all[rows]
            row_of = torch.repeat_interleave(rows, rl)
            start = torch.cumsum(rl, 0) - rl
            within = torch.arange(row_of.numel(), device="cuda") - torch.repeat_interleave(start, rl)
            buf[d_sids[row_of] * pitch + 16 + within] = chars[d_off[row_of] + within]
        ev0.record(stream)
        sset.scan_async(buf, pitch, d_lens, scratch, stream=stream.cuda_stream)
        capi.order_matches_async(db, scratch, out, cnt, stream=stream.cuda_stream)
        ev1.record(stream)
        ev1.synchronize()
        rc, _, _ = capi.scan_corpus_finish(scratch)
        assert rc == capi.HS_SUCCESS, (k, rc)
        total_ms += ev0.elapsed_time(ev1)
        if check:
            n = int(cnt.cpu().numpy().view(np.uint64)[0])
            m = out[: n * 16].cpu().numpy().view(capi.MATCH_DTYPE).copy()
            row_of_stream = np.full(nstreams, -1, dtype=np.int64)
            tr = by_tick[tick_start[k]:tick_start[k + 1]]
            row_of_stream[sids[tr]] = tr
            m["block"] = row_of_stream[m["block"]]
            got.append(m)
    if not check:
        return total_ms, nticks, None
    allm = np.concatenate(got) if got else np.zeros(0, capi.MATCH_DTYPE)
    return total_ms, nticks, np.sort(allm, order=["block", "to", "id"])


def run(torch, db, lits, args, log2s):
    nstreams = 1 << log2s
    nrows, nflows = 1 << args.rows, 1 << args.flows
    chars, d_off, sids, lens = make_batch(torch, lits, nrows, nflows, nstreams, args.zipf, seed=log2s)
    d_ids = torch.from_numpy(sids.astype(np.int32)).cuda()
    scratch = capi.Scratch(db)
    sset = capi.StreamSet(db, nstreams, out_cap=1)
    cap = 1 << 22
    out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    rows_pass(torch, db, sset, scratch, chars, d_off, d_ids, out, cnt, stream, ev)          # warm-up
    pass_ms, only_ms, scan_ms = [], [], []
    for _ in range(args.repeats):
        pass_ms.append(rows_pass(torch, db, sset, scratch, chars, d_off, d_ids, out, cnt, stream, ev))
        a, b = pass_only(torch, sset, scratch, chars, d_off, d_ids, stream, ev)
        only_ms.append(a)
        scan_ms.append(b)
    sset.reset_async(None, stream=stream.cuda_stream)
    rows_pass(torch, db, sset, scratch, chars, d_off, d_ids, out, cnt, stream, ev)
    n = int(cnt.cpu().numpy().view(np.uint64)[0])
    assert n <= cap
    mine = out[: n * 16].cpu().numpy().view(capi.MATCH_DTYPE).copy()
    nbytes = int(lens.sum())
    res = {"streams": nstreams, "rows": nrows, "flows": nflows, "zipf": args.zipf, "batch_bytes": nbytes,
           "busiest_flow_rows": int(np.bincount(sids).max()), "matches": int(n),
           "rows_pass_ms_median": float(np.median(pass_ms)), "rows_pass_ms": pass_ms,
           "rows_pass_gb_s": nbytes / float(np.median(pass_ms)) / 1e6,
           "pass_only_ms_median": float(np.median(only_ms)), "scan_kernels_ms_median": float(np.median(scan_ms)),
           "group_pack_rewrite_advance_ms_median": float(np.median(np.array(only_ms) - np.array(scan_ms)))}
    if log2s in [int(x) for x in args.tick_streams.split(",") if x]:
        t_ms, nticks, theirs = ticks(torch, db, sset, scratch, chars, d_off, sids, lens, nstreams, stream, True)
        res.update({"ticks": nticks, "ticks_ms": t_ms, "ticks_gb_s": nbytes / t_ms / 1e6,
                    "matches_equal": bool(np.array_equal(mine, theirs))})
    sset.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=20, help="log2 of the rows in a batch")
    ap.add_argument("--flows", type=int, default=16, help="log2 of the active flows")
    ap.add_argument("--streams", default="16,24", help="log2 of the set sizes")
    ap.add_argument("--tick-streams", default="16", help="log2 of the set sizes the tick split also runs on")
    ap.add_argument("--zipf", type=float, default=0.7)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    lits, flags, ids = synth.literal_set(5000, min_len=4, max_len=8, caseless_frac=0.1, seed=4)
    db = capi.compile_lit_multi(lits, flags, ids, mode=capi.HS_MODE_STREAM)
    for e in args.streams.split(","):
        print(json.dumps(run(torch, db, lits, args, int(e))), flush=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)


if __name__ == "__main__":
    main()
