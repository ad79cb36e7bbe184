#!/usr/bin/env python
"""Randomised parity fuzzing of the kernels on the SIMT emulator (tests/emu) against the
unmodified reference runtime: random literal sets, block layouts and runtime options
(scan geometry and the switches that force either side of the library's own choices).  Not collected by pytest; run by hand:

  python tests/fuzz_emu.py [--seconds 300] [--seed 1]
"""
import argparse
import faulthandler
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from hyperscan_b200 import capi, synth  # noqa: E402
import build_emu  # noqa: E402
import oracle.ref as ref  # noqa: E402

DEFAULTS = {"warps": 0, "tile_bytes": 1024, "pf_dist": 4, "heavy": 1, "gram": 1, "initial_ring": 1 << 20}


def fuzz_streams(args, rng):
    """Streaming API, vectored mode and stream sets against the reference stream runtime."""
    t0, n = time.time(), 0
    while time.time() - t0 < args.seconds:
        n += 1
        nl = int(rng.choice([1, 3, 8, 40, 100, 400]))
        al = [b"abcdef", b"abcdefghijklmnopqrstuvwxyz", bytes(range(0x20, 0x7f))][int(rng.integers(0, 3))]
        single = float(rng.choice([0, 0.2]))
        lits, flags, ids = synth.literal_set(nl, min_len=1 if nl < 10 else 2, max_len=8, seed=int(rng.integers(1 << 30)),
                                             caseless_frac=float(rng.choice([0, 0.3])), singlematch_frac=single,
                                             alphabet=al)
        for k, v in DEFAULTS.items():
            capi.set_runtime_option(k, v)
        capi.set_runtime_option("warps", int(rng.choice([1, 2, 5])))
        total = int(rng.choice([50, 700, 5000]))
        data, _, _ = synth.ragged_corpus([total], lits, seed=int(rng.integers(1 << 30)), plant_per_kb=20, alphabet=al)
        data = data[:total]
        cuts = np.sort(rng.integers(0, total + 1, size=int(rng.integers(1, 20))))
        wl = np.diff(np.concatenate([[0], cuts, [total]])).astype(np.uint32)
        # 1. hs_open_stream / hs_scan_stream / compress + expand half way
        db = capi.compile_lit_multi(lits, flags, ids, mode=capi.HS_MODE_STREAM)
        scratch = capi.Scratch(db)
        want, err = ref.stream_collect(db.ptr, data, wl)
        st = capi.Stream(db)
        got, pos = [], 0
        for i, w in enumerate(wl):
            if i == len(wl) // 2:
                twin = capi.Stream.expand(db, st.compress())
                st.close(scratch)
                st = twin
            rc, out = st.scan(data[pos:pos + int(w)], scratch)
            assert rc == 0
            got += [(i, a, b) for (a, b) in out]
            pos += int(w)
        st.close(scratch)
        exp = sorted((int(r["block"]), int(r["id"]), int(r["to"])) for r in want)
        if err != 0 or sorted(got) != exp:
            print("STREAM MISMATCH case", n, nl, len(al), wl.tolist()[:10], len(got), len(exp))
            return 1
        # 2. stream set (no single-match ids): every stream gets the same cuts of its own data
        if single == 0:
            ns = int(rng.choice([1, 33, 130]))
            sset = capi.StreamSet(db, ns)
            datas = [synth.ragged_corpus([total], lits, seed=int(rng.integers(1 << 30)), plant_per_kb=20, alphabet=al)[0][:total]
                     for _ in range(ns)]
            recs_all, pos = [], 0
            for i, w in enumerate(wl):
                w = int(w)
                buf = np.concatenate([d[pos:pos + w] for d in datas]) if w else np.zeros(0, np.uint8)
                off = (np.arange(ns, dtype=np.uint64) * np.uint64(w))
                recs_all.append(sset.scan(buf, off, np.full(ns, w, dtype=np.uint32), scratch))
                pos += w
            sset.close()
            for sidx in {0, ns - 1, int(rng.integers(0, ns))}:
                w2, _ = ref.stream_collect(db.ptr, datas[sidx], wl)
                exp2 = sorted((int(r["block"]), int(r["id"]), int(r["to"])) for r in w2)
                mine = []
                for i, recs in enumerate(recs_all):
                    mine += [(i, int(r["id"]), int(r["to"])) for r in recs[recs["block"] == sidx]]
                if sorted(mine) != exp2:
                    print("STREAM SET MISMATCH case", n, nl, ns, sidx, len(mine), len(exp2))
                    return 1
        scratch.free()
        # 3. vectored mode
        vdb = capi.compile_lit_multi(lits, flags, ids, mode=capi.HS_MODE_VECTORED)
        vs = capi.Scratch(vdb)
        wantv, errv = ref.vector_collect(vdb.ptr, data, wl)
        bufs, pos = [], 0
        for w in wl:
            bufs.append(data[pos:pos + int(w)])
            pos += int(w)
        rc, gotv = capi.scan_vector(vdb, bufs, vs)
        vs.free()
        if rc != 0 or errv != 0 or sorted(gotv) != sorted((int(r["id"]), int(r["to"])) for r in wantv):
            print("VECTORED MISMATCH case", n, nl, wl.tolist()[:10], len(gotv), len(wantv))
            return 1
    print("fuzz streams: %d cases, all equal to the reference stream runtime (%.0f s)" % (n, time.time() - t0))
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=300)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--dump", default="", help="write every case here before running it (post-mortem)")
    ap.add_argument("--replay", default="", help="run the one case of a --dump file")
    ap.add_argument("--mode", default="blocks", choices=["blocks", "streams"],
                    help="blocks: block-mode scans; streams: hs_*_stream, hs_scan_vector and stream sets")
    ap.add_argument("--cases", default="", help="comma list: execute only these case numbers (the others only advance the RNG)")
    args = ap.parse_args()
    capi.LIB_PATH = build_emu.build()
    if args.replay:
        import pickle
        with open(args.replay, "rb") as f:
            c = pickle.load(f)
        for k, v in c["opts"].items():
            capi.set_runtime_option(k, v)
        db = capi.compile_lit_multi(c["lits"], c["flags"], c["ids"])
        scratch = capi.Scratch(db)
        want = ref.scan_sorted(db.ptr, c["data"], c["off"], c["ln"])
        got = np.sort(capi.scan_blocks(db, c["data"], c["off"], c["ln"], scratch), order=["block", "to", "id"])
        print("replay host blocks:", len(got), len(want), np.array_equal(got, want), flush=True)
        corpus = capi.Corpus.upload(c["data"], c["off"], c["ln"])
        got2 = np.sort(capi.scan_corpus(db, corpus, scratch), order=["block", "to", "id"])
        print("replay resident corpus:", len(got2), np.array_equal(got2, want))
        return 0
    rng = np.random.default_rng(args.seed)
    if args.mode == "streams":
        return fuzz_streams(args, rng)
    t0, n, skipped = time.time(), 0, 0
    alphabets = [b"ab", b"abcd", b"abcdefgh", b"abcdefghijklmnopqrstuvwxyz", bytes(range(0x20, 0x7f)), bytes(range(256))]
    while time.time() - t0 < args.seconds:
        n += 1
        nl = int(rng.choice([1, 2, 5, 8, 20, 48, 60, 96, 200, 700, 2000]))
        al = alphabets[int(rng.integers(0, len(alphabets)))]
        lo = int(rng.integers(1, 6))
        hi = lo + int(rng.integers(0, 14))
        while len(al) ** hi < nl * 8:   # enough distinct strings for literal_set to terminate
            hi += 1
            lo = max(lo, hi - 6)
        lits, flags, ids = synth.literal_set(nl, min_len=lo, max_len=hi, seed=int(rng.integers(1 << 30)),
                                             caseless_frac=float(rng.choice([0, 0.2, 1.0])),
                                             singlematch_frac=float(rng.choice([0, 0.1])), alphabet=al)
        if rng.random() < 0.3:
            ids = [i // 3 for i in ids]
            fm = {}
            for k in range(nl):
                fm.setdefault(ids[k], flags[k] & 8)
                flags[k] = (flags[k] & ~8) | fm[ids[k]]
        opts = dict(DEFAULTS)
        opts["warps"] = int(rng.choice([1, 2, 3, 5, 8]))
        mode = rng.integers(0, 4)
        if mode == 0:     # scan geometry
            opts.update(tile_bytes=int(rng.choice([512, 1024, 2048, 4096])))
        elif mode == 1:   # candidate list and record ring overflow -> grow and rescan
            opts.update(initial_ring=int(rng.choice([16, 256])))
        elif mode == 2:   # class-pair candidate paths, class 4-gram first stage
            opts.update(heavy=int(rng.choice([0, 1, 2])), gram=int(rng.choice([0, 1, 2, 2])),
                        tile_bytes=int(rng.choice([512, 1024, 4096])))
        # mode 3: the defaults
        # 16 buckets: fat Teddy, through the class-pair kernel with folded buckets
        fat = 48 < nl <= 96 and rng.random() < 0.5 and ref.best_isa() != "corei7"
        for k, v in opts.items():
            capi.set_runtime_option(k, v)
        lens = [int(x) for x in rng.choice([0, 1, 2, 3, 15, 16, 17, 31, 32, 33, 63, 511, 512, 513, 1023, 1024, 1025, 3000, 9000],
                                           size=int(rng.integers(1, 12)))]
        data, off, ln = synth.ragged_corpus(lens, lits, seed=int(rng.integers(1 << 30)),
                                            plant_per_kb=float(rng.choice([0.5, 5, 30])), alphabet=al)
        if args.verbose:
            print("case", n, "nl", nl, "alphabet", len(al), "len", lo, hi,
                  {k: v for k, v in opts.items() if DEFAULTS[k] != v}, "lens", lens, flush=True)
        if args.cases and str(n) not in args.cases.split(","):
            continue
        faulthandler.dump_traceback_later(120, exit=True)  # a case takes seconds: anything longer is a hang
        if args.dump:
            import pickle
            with open(args.dump, "wb") as f:
                pickle.dump({"lits": lits, "flags": flags, "ids": ids, "data": data, "off": off, "ln": ln,
                             "opts": opts}, f)
        try:
            import ctypes as C
            plat = C.byref(capi.PlatformInfo(0, capi.HS_CPU_FEATURES_AVX2, 0, 0)) if fat else None
            db = capi.compile_lit_multi(lits, flags, ids, platform=plat)
        except capi.HsError:
            skipped += 1
            continue
        scratch = capi.Scratch(db)
        want = ref.scan_sorted(db.ptr, data, off, ln)
        got = np.sort(capi.scan_blocks(db, data, off, ln, scratch), order=["block", "to", "id"])
        corpus = capi.Corpus.upload(data, off, ln)
        got2 = np.sort(capi.scan_corpus(db, corpus, scratch), order=["block", "to", "id"])
        corpus.free()
        scratch.free()
        faulthandler.cancel_dump_traceback_later()
        if not (np.array_equal(got, want) and np.array_equal(got2, want)):
            print("MISMATCH case", n, "nl", nl, "alphabet", len(al), "len", lo, hi, "opts",
                  {k: v for k, v in opts.items() if DEFAULTS[k] != v}, "lens", lens, len(got), len(got2), len(want))
            return 1
    print("fuzz: %d cases (%d refused by the compiler), all bit-exact vs the reference runtime (%.0f s)"
          % (n - skipped, skipped, time.time() - t0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
