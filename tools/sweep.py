#!/usr/bin/env python
"""Kernel tuning sweep (run on the GPU box): one resident corpus, many runtime
configurations; prints kernel time, GB/s and the first/second stage counters.

  python tools/sweep.py [--mb 512] [--lits 1000] [--block-len 1024] [--configs "k=v,k=v;k=v,..."]
"""
import argparse
import json
import os
import sys
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperscan_b200 import capi, synth  # noqa: E402

DEFAULT = ("pf_dist=4;pf_dist=2;pf_dist=8;pf_dist=16;warps=24;warps=32;tile_bytes=4096;heavy=0;heavy=2;"
           "gram=0;gram=2")
BASE = {"warps": 0, "tile_bytes": 1024, "pf_dist": -1, "heavy": 1, "gram": 1}  # the library defaults


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=512)
    ap.add_argument("--lits", type=int, default=1000)
    ap.add_argument("--min-len", type=int, default=4)
    ap.add_argument("--max-len", type=int, default=8)
    ap.add_argument("--block-len", type=int, default=1024)
    ap.add_argument("--configs", default=DEFAULT)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--alphabet", default="")
    ap.add_argument("--lib", default="", help="A/B: another build of libhs_b200.so (same ABI)")
    ap.add_argument("--avx2", action="store_true", help="compile for an AVX2 platform (49..96 literals: fat Teddy)")
    args = ap.parse_args()
    if args.lib:
        capi.LIB_PATH = os.path.abspath(args.lib)
    lits, flags, ids = synth.literal_set(args.lits, min_len=args.min_len, max_len=args.max_len)
    nblocks = (args.mb << 20) // args.block_len
    data, off, ln, _ = synth.block_corpus(nblocks, args.block_len, lits, plant_per_kb=0.01)
    if args.alphabet:
        al = np.frombuffer(args.alphabet.encode(), dtype=np.uint8)
        data = al[np.random.default_rng(5).integers(0, al.size, size=data.size)]
    plat = None
    if args.avx2:
        import ctypes as C
        plat = C.byref(capi.PlatformInfo(0, capi.HS_CPU_FEATURES_AVX2, 0, 0))
    db = capi.compile_lit_multi(lits, flags, ids, platform=plat)
    info = db.info()
    print("engine", info.engine_id, "domain", info.fdr_domain, "stride", info.fdr_stride, flush=True)
    corpus = capi.Corpus.upload(data, off, ln)
    nbytes = int(ln.sum())
    base_matches = None
    base_digest = None
    for spec in args.configs.split(";"):
        cfg = dict(BASE)
        for kv in spec.split(","):
            if kv.strip():
                k, v = kv.split("=")
                cfg[k.strip()] = int(v)
        for k, v in cfg.items():
            try:
                capi.set_runtime_option(k, v)
            except capi.HsError:
                pass  # an older build of the library (--lib) without this option
        scratch = capi.Scratch(db)
        ms = []
        try:
            for i in range(3 + args.reps):
                capi.scan_corpus_async(db, corpus, scratch)
                rc, n, _ = capi.scan_corpus_finish(scratch)
                if rc == capi.HS_INSUFFICIENT_SPACE:
                    continue
                assert rc == 0, rc
                if i >= 3:
                    ms.append(scratch.last_kernel_ms())
            c = scratch.counters()
            recs = np.sort(capi.fetch_matches(db, scratch), order=["block", "to", "id"])
            digest = zlib.crc32(recs.tobytes())
            if base_matches is None:
                base_matches = c[0]
                base_digest = digest
            t = float(np.median(ms))
            print(json.dumps({"cfg": spec, "ms": round(t, 4), "GBps": round(nbytes / t / 1e6, 1),
                              "records": c[0], "same_records": c[0] == base_matches and digest == base_digest, "cand": c[2],
                              "prefilter_pass": c[4], "confirmed": c[3],
                              "cand_per_kb": round(c[2] / (nbytes / 1024), 3)}), flush=True)
        except Exception as e:  # keep sweeping
            print(json.dumps({"cfg": spec, "error": str(e)}), flush=True)
        scratch.free()


if __name__ == "__main__":
    main()
