#!/usr/bin/env python
"""One stream-set tick from writes already in HBM (hs_b200_streams_scan_async + hs_b200_order_matches_async) against
the same writes from pinned host memory (hs_b200_streams_scan_collect), for the config-4 shape of bench.py: 5 000
literals of 4-8 bytes, 1 KiB writes, one write per stream per tick (DESIGN.md section 9a).  Run on the GPU box:
    python tools/stream_set_device_bench.py [--streams 20,24] [--ticks 4]

The writes are random bytes of a 64-letter alphabet with about one planted literal per stream, generated on the
device at pitch 1 040 (16 bytes of headroom in front of each write).  Two stream sets take the same writes every
tick, and the two paths alternate tick by tick after one warm-up tick each:
  device  CUDA events around the tick on one CUDA stream (assemble, scan, confirm, advance, ordering into device
          memory); no host wait inside the window.
  host    host clock around hs_b200_streams_scan_collect from pinned memory (copy in, scan, records to the host,
          ordering there, advance), which returns when all is done.
Both report the scan kernels' time (hs_b200_last_kernel_ms, CUDA events around scan and confirm).  Every tick the
device path's ordered matches must equal the host path's, record for record.  One JSON line per stream count, then
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

WRITE, PITCH = 1024, 1040


def make_writes(torch, lits, nstreams, seed):
    """[nstreams, PITCH] bytes on the device: random headroom, a random write with about one literal planted"""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    alpha = torch.tensor(list(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 ./-"),
                         dtype=torch.uint8, device="cuda")
    buf = torch.randint(0, 256, (nstreams, PITCH), dtype=torch.uint8, device="cuda", generator=g)
    for s in range(0, nstreams, 1 << 18):   # (the int64 indices of 2^24 writes would not fit)
        e = min(nstreams, s + (1 << 18))
        buf[s:e, 16:] = alpha[torch.randint(0, alpha.numel(), (e - s, WRITE), device="cuda", generator=g)]
    table = torch.zeros(len(lits), 8, dtype=torch.uint8)
    for i, x in enumerate(lits):
        table[i, :len(x)] = torch.tensor(list(x), dtype=torch.uint8)
    table = table.cuda()
    lens = torch.tensor([len(x) for x in lits], dtype=torch.int64, device="cuda")
    which = torch.randint(0, len(lits), (nstreams,), device="cuda", generator=g)
    at = 16 + torch.randint(0, WRITE - 8, (nstreams,), device="cuda", generator=g)
    rows = torch.arange(nstreams, device="cuda")
    for b in range(8):
        keep = lens[which] > b
        buf[rows[keep], at[keep] + b] = table[which[keep], b]
    return buf


def run(torch, db, lits, nstreams, ticks, seed):
    scratch_d, scratch_h = capi.Scratch(db), capi.Scratch(db)
    dev_set = capi.StreamSet(db, nstreams, out_cap=1)
    cap = nstreams * 4
    host_set = capi.StreamSet(db, nstreams, out_cap=cap)
    out = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    off = np.arange(nstreams, dtype=np.uint64) * np.uint64(WRITE)
    ln = np.full(nstreams, WRITE, dtype=np.uint32)
    stream = torch.cuda.Stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms, dev_kms, host_ms, host_kms, matches, equal = [], [], [], [], [], True
    pinned = torch.empty(nstreams * WRITE, dtype=torch.uint8, pin_memory=True)
    for t in range(ticks + 1):
        buf = make_writes(torch, lits, nstreams, seed + t)
        pinned.view(nstreams, WRITE).copy_(buf[:, 16:])
        torch.cuda.synchronize()
        # device path: writes already in HBM (the warm-up tick grows the record ring: the pass that
        # overflowed it committed nothing and is enqueued again)
        for _ in range(3):
            ev0.record(stream)
            dev_set.scan_async(buf, PITCH, WRITE, scratch_d, stream=stream.cuda_stream)
            capi.order_matches_async(db, scratch_d, out, cnt, stream=stream.cuda_stream)
            ev1.record(stream)
            ev1.synchronize()
            rc, _, _ = capi.scan_corpus_finish(scratch_d)
            if rc != capi.HS_INSUFFICIENT_SPACE:
                break
            assert t == 0, "the ring overflowed after the warm-up tick"
        assert rc == capi.HS_SUCCESS, rc
        n = int(cnt.cpu().numpy().view(np.uint64)[0])
        assert n <= cap
        got = out[: n * 16].cpu().numpy().view(capi.MATCH_DTYPE)
        kd = scratch_d.last_kernel_ms()
        # host path: the same writes from pinned host memory
        t0 = time.perf_counter()
        want = host_set.scan(pinned.numpy(), off, ln, scratch_h)
        th = (time.perf_counter() - t0) * 1e3
        kh = scratch_h.last_kernel_ms()
        equal = equal and np.array_equal(got, want)
        if t:
            dev_ms.append(ev0.elapsed_time(ev1))
            dev_kms.append(kd)
            host_ms.append(th)
            host_kms.append(kh)
            matches.append(int(n))
        del buf
    dev_set.close()
    host_set.close()
    write_bytes = nstreams * WRITE
    return {"streams": nstreams, "write_bytes": WRITE, "pitch": PITCH, "ticks": ticks,
            "device_tick_ms_median": float(np.median(dev_ms)), "device_tick_ms": dev_ms,
            "device_scan_kernel_ms_median": float(np.median(dev_kms)),
            "device_write_gb_s": write_bytes / float(np.median(dev_ms)) / 1e6,
            "host_tick_ms_median": float(np.median(host_ms)), "host_tick_ms": host_ms,
            "host_scan_kernel_ms_median": float(np.median(host_kms)),
            "host_write_gb_s": write_bytes / float(np.median(host_ms)) / 1e6,
            "matches_per_tick": matches, "matches_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="20,24", help="log2 of the stream counts")
    ap.add_argument("--ticks", type=int, default=4)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    lits, flags, ids = synth.literal_set(5000, min_len=4, max_len=8, caseless_frac=0.1, seed=4)
    db = capi.compile_lit_multi(lits, flags, ids, mode=capi.HS_MODE_STREAM)
    for e in args.streams.split(","):
        print(json.dumps(run(torch, db, lits, 1 << int(e), args.ticks, seed=int(e))), flush=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)


if __name__ == "__main__":
    main()
