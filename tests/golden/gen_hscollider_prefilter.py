#!/usr/bin/env python
"""Generate tests/golden/hscollider_prefilter.json from the reference's own recorded regression vectors
(tools/hscollider/test_cases/{pcre,corpora}/*.txt): PCRE's match offsets for the expressions that only prefilter
mode (HS_FLAG_PREFILTER) compiles here.

The pattern lines taken are those with flags among `i s m O P` and no extended parameters (formats as in
gen_hscollider_regex.py) that are prefilter cases: the reference's own, flagged `P` (HS_FLAG_PREFILTER; all of
prefilter.txt: back-references, look-around, atomic groups, possessive quantifiers, conditionals), and the others
that this library's hs_compile refuses without the flag (long counted repeats, numeric escapes).  They are kept
when they compile with the flag and have corpora lines with recorded offsets; the summary counts why the others
are skipped.  Lines with other flags (`H` single-match, `8` UTF-8, `W` UCP, ...) or extended parameters are not
taken.  The pattern TEXT and the recorded offsets are data of the reference's test-suite, not code; they are
stored here because the tests run where no reference checkout exists.

Each kept entry is also run through the unmodified reference runtime (oracle/_ref) on the prefiltered database
compiled here: every recorded offset must be among the reference runtime's, or the generator aborts."""
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
from gen_hscollider_regex import BASE, decode_corpus  # noqa: E402

FLAG = {"i": capi.HS_FLAG_CASELESS, "s": 2, "m": 4, "O": 0, "P": 128}
PREFILTER = 128


def main():
    pats, skipped, lines, counts = {}, collections.Counter(), 0, collections.Counter()
    for f in sorted(glob.glob(BASE + "/pcre/*.txt")):
        for line in open(f, "rb"):
            m = re.match(rb"^(\d+):/(.*)/([a-zA-Z8]*)(\{[a-z_0-9=,]*\})?\s*$", line.rstrip(b"\n"))
            if not m:
                continue
            pid, pat, fl = int(m.group(1)), m.group(2), m.group(3).decode()
            if set(fl) - set(FLAG) or m.group(4):
                continue
            flags = 0
            for c in fl:
                flags |= FLAG[c]
            if not flags & PREFILTER:
                try:
                    capi.compile_multi([pat], [flags], [pid])
                    continue             # the exact route compiles it
                except capi.HsError:
                    pass
            lines += 1
            counts["P" if flags & PREFILTER else "refused"] += 1
            try:
                capi.compile_multi([pat], [flags | PREFILTER], [pid])
            except capi.HsError as e:
                skipped["refused with the flag too: " + e.message] += 1
                continue
            pats[pid] = (pat, fl, flags | PREFILTER, os.path.basename(f))
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
        pat, fl, flags, pfile = pats[pid]
        db = capi.compile_multi([pat], [flags], [pid])
        corp = []
        for data, ends, cfile in cases[pid]:
            arr = np.frombuffer(data, dtype=np.uint8)
            got = ref.scan_sorted(db.ptr, arr, np.array([0], dtype=np.uint64), np.array([len(data)], dtype=np.uint32))
            tos = {int(r["to"]) for r in got}
            assert set(ends) <= tos, (pid, pat, data, ends, sorted(tos))
            corp.append({"data": base64.b64encode(data).decode(), "ends": ends, "file": cfile})
        out.append({"id": pid, "pattern": base64.b64encode(pat).decode(), "flag_letters": fl, "hs_flags": flags,
                    "file": pfile, "corpora": corp})
        print(pid, pat, fl, len(corp), "corpora")
    with open(os.path.join(ROOT, "tests", "golden", "hscollider_prefilter.json"), "w") as f:
        json.dump({"generator": "tests/golden/gen_hscollider_prefilter.py",
                   "source": "intel/hyperscan 5.4.2 tools/hscollider/test_cases (recorded PCRE offsets)",
                   "lines": lines, "flagged_P": counts["P"], "refused_without_the_flag": counts["refused"],
                   "kept": len(out), "kept_flagged_P": sum("P" in c["flag_letters"] for c in out),
                   "skipped": dict(sorted(skipped.items())),
                   "cases": out}, f, indent=0)
    print("%d pattern lines (%d flagged P, %d refused without the flag): %d kept, %d of them flagged P (%d corpora)"
          % (lines, counts["P"], counts["refused"], len(out), sum("P" in c["flag_letters"] for c in out),
             sum(len(c["corpora"]) for c in out)))
    for why, k in sorted(skipped.items()):
        print("  skipped %3d: %s" % (k, why))


if __name__ == "__main__":
    main()
