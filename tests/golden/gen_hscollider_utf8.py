#!/usr/bin/env python
"""Generate tests/golden/hscollider_utf8.json from the reference's own recorded regression
vectors (tools/hscollider/test_cases/{pcre,corpora}/*.txt) for expressions in UTF-8 mode.

The pattern lines kept are those with flag `8` (HS_FLAG_UTF8), optionally with `i s m H O` and
without `W` (HS_FLAG_UCP), that this library's hs_compile compiles -- through the literal route or
the regex route -- together with the corpora lines that carry recorded match offsets (formats as in
gen_hscollider_regex.py).  The others are skipped, and the summary counts each reason: Unicode
properties, non-ASCII case folding, too many positions, anything else this compiler refuses, or no
recorded corpus.  The pattern TEXT and the recorded offsets are data of the reference's test-suite,
not code; they are stored here because the tests run where no reference checkout exists.

Each kept entry is also run through the unmodified reference runtime (oracle/_ref) on the database
compiled here: the recorded offsets and the reference runtime must agree, or the generator aborts."""
import base64
import collections
import glob
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hyperscan_b200 import capi  # noqa: E402
import oracle.ref as ref  # noqa: E402
from gen_hscollider_regex import BASE, FLAG, decode_corpus  # noqa: E402


def skip_reason(msg):
    if "Unicode properties" in msg:
        return "Unicode properties (\\p, \\P)"
    if "case folding" in msg:
        return "non-ASCII case folding"
    if "too large" in msg:
        return "too many positions"
    return "refused: " + msg.split(" (expression")[0]


def main():
    pats, skipped, lines = {}, collections.Counter(), 0
    for f in sorted(glob.glob(BASE + "/pcre/*.txt")):
        for line in open(f, "rb"):
            m = re.match(rb"^(\d+):/(.*)/([a-zA-Z8]*)(\{[a-z_0-9=,]*\})?\s*$", line.rstrip(b"\n"))
            if not m:
                continue
            pid, pat, fl = int(m.group(1)), m.group(2), m.group(3).decode()
            if "8" not in fl or set(fl) - set(FLAG) - {"8"}:
                continue
            lines += 1
            ext = None
            if m.group(4):
                ext = {k: int(v) for k, v in (kv.split("=") for kv in m.group(4).decode()[1:-1].split(",") if kv)}
            flags = capi.HS_FLAG_UTF8
            for c in fl.replace("8", ""):
                flags |= FLAG[c]
            try:
                capi.compile_ext_multi([pat], [flags], [pid], [ext])
            except capi.HsError as e:
                skipped[skip_reason(str(e))] += 1
                continue
            pats[pid] = (pat, fl, flags, os.path.basename(f), ext)
    cases = {}
    for f in sorted(glob.glob(BASE + "/corpora/*.txt")):
        for line in open(f, "rb"):
            m = re.match(rb'^(\d+)="(.*)":\s*([\d, ]*)\s*$', line.rstrip(b"\n"))
            if not m or int(m.group(1)) not in pats:
                continue
            pid = int(m.group(1))
            ends = sorted(int(x) for x in m.group(3).replace(b" ", b"").split(b",") if x)
            cases.setdefault(pid, []).append((decode_corpus(m.group(2)), ends, os.path.basename(f)))
    skipped["no recorded corpus"] += len(set(pats) - set(cases))
    out = []
    for pid in sorted(cases):
        pat, fl, flags, pfile, ext = pats[pid]
        db = capi.compile_ext_multi([pat], [flags], [pid], [ext])
        corp = []
        for data, ends, cfile in cases[pid]:
            arr = np.frombuffer(data, dtype=np.uint8)
            got = ref.scan_sorted(db.ptr, arr, np.array([0], dtype=np.uint64),
                                  np.array([len(data)], dtype=np.uint32))
            tos = [int(r["to"]) for r in got]
            if "H" in fl:
                # tools/hscollider/main.cpp:522-537: in single-match mode the scanner must
                # return exactly one of the recorded matches (when there are any)
                assert (len(tos) == 1 and tos[0] in ends) if ends else not tos, (pid, pat, ends, tos)
            else:
                assert tos == ends, (pid, pat, data, ends, got)
            corp.append({"data": base64.b64encode(data).decode(), "ends": ends, "file": cfile})
        out.append({"id": pid, "pattern": base64.b64encode(pat).decode(), "flag_letters": fl,
                    "hs_flags": flags, "ext": ext, "file": pfile, "runtime_impl": db.info().runtime_impl,
                    "corpora": corp})
        print(pid, pat, fl, len(corp), "corpora")
    with open(os.path.join(ROOT, "tests", "golden", "hscollider_utf8.json"), "w") as f:
        json.dump({"generator": "tests/golden/gen_hscollider_utf8.py",
                   "source": "intel/hyperscan 5.4.2 tools/hscollider/test_cases (recorded offsets)",
                   "lines": lines, "kept": len(out), "skipped": dict(sorted(skipped.items())),
                   "cases": out}, f, indent=0)
    print("%d UTF-8 pattern lines: %d kept (%d corpora)" % (lines, len(out), sum(len(c["corpora"]) for c in out)))
    for why, k in sorted(skipped.items()):
        print("  skipped %3d: %s" % (k, why))


if __name__ == "__main__":
    main()
