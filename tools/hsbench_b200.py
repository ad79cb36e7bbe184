#!/usr/bin/env python
"""hsbench for the H100 runtime: the reference benchmark's command line, inputs and report
(tools/hsbench/main.cpp:190-240 options, :503-527 scan loops, :721-725 Mbit/s, :773-860 the
report) over this library's C ABI.

Inputs are hsbench's own: a signature file of `ID:/regex/flags` lines (util/ExpressionParser.rl;
`-e FILE|DIR`, optionally restricted by `-s FILE` / `-z ID`) and a corpus in its sqlite schema
(`CREATE TABLE chunk(id integer primary key, stream_id integer not null, data blob)`,
tools/hsbench/data_corpus.cpp:60-125, tools/hsbench/scripts/CorpusBuilder.py).

  -N   block mode: every chunk is one block.  All blocks of the corpus go through ONE
       hs_b200_scan_blocks call per repeat (the batched form of the reference's loop of
       hs_scan calls, INTEGRATION.md section 2) from host memory: H2D copy, kernels, D2H of the
       records and the report rules are inside the timed region, as hsbench times hs_scan.
       `--per-call` uses the stock hs_scan once per block instead.
  default (streaming): the chunks of one stream_id are one stream, scanned in id order; write k of
       every stream goes through one hs_b200_streams_scan call (state resident in HBM).
`--resident` adds a second figure with the corpus already in device memory (block mode).

The report has hsbench's lines, so scripts that read "Mean throughput (overall)" keep working."""
import argparse
import os
import re
import sqlite3
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FLAG_LETTERS = {"i": 1, "s": 2, "m": 4, "H": 8, "V": 16, "8": 32, "W": 64, "P": 128, "L": 256, "C": 512, "Q": 1024}
# (HS_FLAG_* values: src/hs_compile.h:951-1060; the letters: util/ExpressionParser.rl:60-85)


def parse_signature_line(line):
    """`ID:/regex/flags{ext}` -> (id, regex bytes, flags, ext dict or None) or None for blanks / comments"""
    line = line.rstrip(b"\r\n")
    if not line.strip() or line.lstrip().startswith(b"#"):
        return None
    m = re.match(rb"^\s*(\d+):/(.*)/([A-Za-z0-9]*)(\{[^}]*\})?\s*$", line)
    if not m:
        raise ValueError("cannot parse signature line %r" % line[:80])
    ext = None
    if m.group(4):      # {min_offset=..,max_offset=..,min_length=..,edit_distance=..,hamming_distance=..}
        try:
            ext = {k.strip(): int(v) for k, v in (kv.split("=") for kv in m.group(4).decode()[1:-1].split(",") if kv.strip())}
        except ValueError:
            raise ValueError("cannot parse the extended parameters of %r" % line[:80])
        if set(ext) - {"min_offset", "max_offset", "min_length", "edit_distance", "hamming_distance"}:
            raise ValueError("unknown extended parameter in %r" % line[:80])
    flags = 0
    for c in m.group(3).decode():
        if c == "O":        # hscollider's "no prefilter conversion" marker: no flag
            continue
        if c not in FLAG_LETTERS:
            raise ValueError("unknown flag letter %r in %r" % (c, line[:80]))
        flags |= FLAG_LETTERS[c]
    return int(m.group(1)), m.group(2), flags, ext


def load_signatures(path, only_ids=None):
    files = [path] if os.path.isfile(path) else sorted(
        os.path.join(path, f) for f in os.listdir(path) if os.path.isfile(os.path.join(path, f)))
    out = {}
    for f in files:
        with open(f, "rb") as fh:
            for line in fh:
                sig = parse_signature_line(line)
                if sig and (only_ids is None or sig[0] in only_ids):
                    out[sig[0]] = sig
    return [out[k] for k in sorted(out)]


def load_id_list(path):
    ids = set()
    with open(path) as fh:
        for line in fh:
            line = line.split("#")[0].strip()
            if line:
                ids.add(int(line))
    return ids


def load_corpus(path):
    """[(stream_id, bytes)] in chunk id order"""
    con = sqlite3.connect("file:%s?mode=ro" % path, uri=True)
    try:
        rows = con.execute("SELECT stream_id, data FROM chunk ORDER BY id").fetchall()
    finally:
        con.close()
    return [(int(s), bytes(d) if d is not None else b"") for s, d in rows]


def write_corpus(path, chunks):
    """chunks: iterable of (stream_id, bytes) -- hsbench's schema (CorpusBuilder.py)"""
    if os.path.exists(path):
        os.unlink(path)
    con = sqlite3.connect(path)
    con.execute("CREATE TABLE chunk(id integer primary key, stream_id integer not null, data blob)")
    con.executemany("INSERT INTO chunk(stream_id, data) VALUES (?, ?)", ((int(s), sqlite3.Binary(d)) for s, d in chunks))
    con.commit()
    con.close()


def pack_blocks(blocks, align=16):
    """bytes list -> (data uint8, offsets u64, lengths u32), every block 16-byte aligned"""
    ln = np.array([len(b) for b in blocks], dtype=np.uint32)
    pitch = (ln.astype(np.uint64) + np.uint64(align - 1)) // np.uint64(align) * np.uint64(align)
    off = np.zeros(len(blocks), dtype=np.uint64)
    if len(blocks) > 1:
        off[1:] = np.cumsum(pitch[:-1])
    total = int(off[-1] + pitch[-1]) if len(blocks) else 0
    data = np.zeros(max(total, 16), dtype=np.uint8)
    for b, o in zip(blocks, off.tolist()):
        if b:
            data[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return data, off, ln


def mbps(seconds, nbytes):
    return nbytes / (seconds * 125000.0) if seconds > 0 else 0.0


def main(argv=None):
    ap = argparse.ArgumentParser(description="hsbench over the H100 runtime", add_help=True)
    ap.add_argument("-e", dest="expr", required=True, help="signature file or directory")
    ap.add_argument("-s", dest="sigfile", help="file with the signature IDs to use")
    ap.add_argument("-z", dest="sigid", type=int, help="one signature ID to use")
    ap.add_argument("-c", dest="corpus", required=True, help="corpus (sqlite, hsbench schema)")
    ap.add_argument("-n", dest="repeats", type=int, default=20)
    ap.add_argument("-N", dest="block", action="store_true", help="block mode (default: streaming)")
    ap.add_argument("-V", dest="vectored", action="store_true", help="vectored mode")
    ap.add_argument("-T", dest="threads", help="accepted for compatibility; the scan runs on the GPU")
    ap.add_argument("-w", dest="save", help="after compiling, save the database to DIR")
    ap.add_argument("-i", dest="load", help="don't compile, load the database from DIR")
    ap.add_argument("--per-scan", action="store_true")
    ap.add_argument("--echo-matches", action="store_true")
    ap.add_argument("--literal-on", action="store_true", help="hs_compile_lit_multi: the patterns are literals")
    ap.add_argument("--per-call", action="store_true", help="block mode: one stock hs_scan per block")
    ap.add_argument("--resident", action="store_true", help="block mode: also time the corpus resident in HBM")
    args = ap.parse_args(argv)
    if args.vectored:
        print("Error: vectored mode is not benchmarked by this tool (hs_scan_vector exists; see INTEGRATION.md).")
        return 1
    from hyperscan_b200 import capi

    only = None
    if args.sigfile:
        only = load_id_list(args.sigfile)
    if args.sigid is not None:
        only = {args.sigid}
    sigs = load_signatures(args.expr, only)
    if not sigs:
        print("Error: no signatures.")
        return 1
    mode = capi.HS_MODE_BLOCK if args.block else capi.HS_MODE_STREAM
    name = os.path.basename(args.expr.rstrip("/"))
    dbfile = None
    if args.load or args.save:
        dbfile = os.path.join(args.load or args.save, "%s_%s.db" % (name, "block" if args.block else "streaming"))
    t0 = time.perf_counter()
    if args.load:
        with open(dbfile, "rb") as fh:
            db = capi.Database.deserialize(fh.read())
    else:
        ids = [s[0] for s in sigs]
        pats = [s[1] for s in sigs]
        flags = [s[2] for s in sigs]
        try:
            if args.literal_on:
                db = capi.compile_lit_multi(pats, flags, ids, mode=mode)
            else:
                db = capi.compile_ext_multi(pats, flags, ids, [s[3] for s in sigs], mode=mode)
        except capi.HsError as e:
            print("Error: compile failed: %s" % e)
            return 1
    compile_s = time.perf_counter() - t0
    if args.save:
        os.makedirs(args.save, exist_ok=True)
        with open(dbfile, "wb") as fh:
            fh.write(db.serialize())
    info = db.info()
    chunks = load_corpus(args.corpus)
    if not chunks:
        print("Error: the corpus has no chunks.")
        return 1
    total_bytes = sum(len(d) for _, d in chunks)
    scratch = capi.Scratch(db)

    print("Signatures:        %s" % args.expr)
    print("Hyperscan info:    H100 runtime (hs-b200), reference-format database; %s"
          % ("pure literal" if info.runtime_impl == 1 else "single outfix" if info.runtime_impl == 2 else "rose"))
    print("Expression count:  %d" % len(sigs))
    print("Bytecode size:     %d bytes" % info.bytecode_len)
    print("Database CRC:      n/a")
    print("Scratch size:      %d bytes" % scratch.size())
    print("Compile time:      %0.3f seconds" % compile_s)
    print("Scan mode:         %s%s" % ("block" if args.block else "streaming",
                                       " (one hs_scan per block)" if args.per_call else ""))
    print()

    times, matches_per_run = [], None
    echo = []

    def record(n):
        nonlocal matches_per_run
        if matches_per_run is None:
            matches_per_run = n
        elif matches_per_run != n:
            matches_per_run = -1

    if args.block:
        blocks = [d for _, d in chunks]
        data, off, ln = pack_blocks(blocks)
        for r in range(args.repeats):
            t = time.perf_counter()
            if args.per_call:
                n = 0
                for b in blocks:
                    hits = []
                    capi.scan(db, b, scratch, on_event=lambda i, frm, to, fl: hits.append((i, to)) or 0)
                    n += len(hits)
                    if args.echo_matches and r == 0:
                        echo.extend(hits)
            elif args.echo_matches and r == 0:
                recs = capi.scan_blocks(db, data, off, ln, scratch)
                n = int(recs.size)
                echo.extend((int(x["id"]), int(x["to"])) for x in recs)
            else:
                n = capi.scan_blocks(db, data, off, ln, scratch, collect=False)
            times.append(time.perf_counter() - t)
            record(n)
        nstreams = None
    else:
        order, per_stream = [], {}
        for s, d in chunks:
            if s not in per_stream:
                per_stream[s] = []
                order.append(s)
            per_stream[s].append(d)
        nstreams = len(order)
        rounds = max(len(v) for v in per_stream.values())
        writes = [pack_blocks([per_stream[s][k] if k < len(per_stream[s]) else b"" for s in order]) for k in range(rounds)]
        for r in range(args.repeats):
            t = time.perf_counter()
            ss = capi.StreamSet(db, nstreams)
            n = 0
            for data, off, ln in writes:
                if args.echo_matches and r == 0:
                    recs = ss.scan(data, off, ln, scratch)
                    n += int(recs.size)
                    echo.extend((int(x["id"]), int(x["to"])) for x in recs)
                else:
                    n += ss.scan(data, off, ln, scratch, collect=False)
            ss.close()
            times.append(time.perf_counter() - t)
            record(n)

    for i, to in echo:
        print("Match @%d:%d" % (i, to))
    total_secs = sum(times)
    if matches_per_run == -1:
        print("\nWARNING: PER-SCAN MATCH COUNTS ARE INCONSISTENT!\n")
        matches_per_run = 0
    print("Time spent scanning:       %0.3f seconds" % total_secs)
    if args.block:
        print("Corpus size:               %d bytes (%d blocks)" % (total_bytes, len(chunks)))
    else:
        print("Corpus size:               %d bytes (%d blocks in %d streams)" % (total_bytes, len(chunks), nstreams))
    print("Matches per iteration:     %d (%0.3f matches/kilobyte)"
          % (matches_per_run, matches_per_run * 1024.0 / max(total_bytes, 1)))
    print("Overall block rate:        %0.2f blocks/sec" % (len(chunks) * args.repeats / total_secs))
    print("Mean throughput (overall): %0.2f Mbit/sec" % mbps(total_secs, total_bytes * args.repeats))
    print("Max throughput (per core): %0.2f Mbit/sec" % mbps(min(times), total_bytes))
    if args.block and args.resident:
        corpus = capi.Corpus.upload(data, off, ln)
        rt = []
        for r in range(args.repeats):
            t = time.perf_counter()
            capi.scan_corpus_async(db, corpus, scratch)
            rc, n, _ = capi.scan_corpus_finish(scratch)
            while rc == capi.HS_INSUFFICIENT_SPACE:      # the record ring grew: scan again
                capi.scan_corpus_async(db, corpus, scratch)
                rc, n, _ = capi.scan_corpus_finish(scratch)
            capi._check(rc, "scan_corpus")
            rt.append(time.perf_counter() - t)
        corpus.free()
        print("Device-resident corpus:    %0.2f Mbit/sec mean, %0.2f best (hs_b200_scan_corpus_async + _finish, %d records)"
              % (mbps(sum(rt), total_bytes * args.repeats), mbps(min(rt), total_bytes), n))
    print()
    if args.per_scan:
        for r, t in enumerate(times):
            print("Scan %3d: %0.2f Mbit/sec" % (r, mbps(t, total_bytes)))
    scratch.free()
    return 0


if __name__ == "__main__":
    sys.exit(main())
