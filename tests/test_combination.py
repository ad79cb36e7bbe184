"""Logical combinations of expressions (HS_FLAG_COMBINATION, HS_FLAG_QUIET) in block mode.

The reference's unit tests (unit/hyperscan/logical_combination.cpp, kept as data in
golden/logical_combination.json) give every callback in order.  Our databases keep the
reference's bytecode format, so the unmodified reference hs_scan runs them too: on the CPU
it checks the compiler against those answers and against a definition-level evaluator; on
the GPU the device scan is checked against the reference.  The reference's one streaming
test (MultiCombStream1) has no counterpart: combinations, like regular expressions that
need an engine, are compiled for block mode only here, and HS_MODE_STREAM is refused.
"""
import base64
import json
import os
import random
import re

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "logical_combination.json")) as _f:
    CASES = json.load(_f)["cases"]
with open(os.path.join(HERE, "golden", "bad_patterns.json")) as _f:
    BAD = [c for c in json.load(_f)["cases"] if c["hs_flags"] & 512]

MAX_OFFSET = (1 << 64) - 1


def _flags(hs, names):
    return sum(getattr(hs, n) for n in names)


def _compile(hs, case):
    return hs.compile_multi([e.encode() for e in case["expressions"]], [_flags(hs, f) for f in case["flags"]],
                            case["ids"])


def _ref_order(ref, db, data, stop_after=0):
    recs, err = ref.scan_collect(db.ptr, data, [0], [len(data)], stop_after=stop_after)
    return [(int(r["to"]), int(r["id"])) for r in recs]


# ---- a definition-level evaluator ---------------------------------------------------------------

def _ends(expr, data):
    """Every end offset of a match of `expr` (a Python-compatible regex) in data."""
    rx = re.compile(expr.encode(), re.S)
    return sorted({e for s in range(len(data)) for e in range(s + 1, len(data) + 1) if rx.fullmatch(data, s, e)})


class Comb:
    """A combination as text plus its meaning: a tree of ('id', n) / ('!', t) / ('&'|'|', l, r)."""

    def __init__(self, tree):
        self.tree = tree

    def text(self):
        t = self.tree
        if t[0] == "id":
            return str(t[1])
        if t[0] == "!":
            return "!" + Comb(t[1]).atom()
        return "(%s %s %s)" % (Comb(t[1]).text(), t[0], Comb(t[2]).text())

    def atom(self):
        return self.text() if self.tree[0] == "id" else "(%s)" % self.text()

    def leaves(self, t=None):
        t = self.tree if t is None else t
        return [t[1]] if t[0] == "id" else sum((self.leaves(c) for c in t[1:]), [])

    def value(self, seen, t=None):
        t = self.tree if t is None else t
        if t[0] == "id":
            return t[1] in seen
        if t[0] == "!":
            return not self.value(seen, t[1])
        a, b = self.value(seen, t[1]), self.value(seen, t[2])
        return (a and b) if t[0] == "&" else (a or b)


def evaluate(subs, combs, data, min_width):
    """What hs_scan delivers, from the definition: subs = [(id, regex, quiet, single)], combs = [(id, Comb,
    single, min_offset, max_offset)].  A sub-expression's match sets its id for the rest of the block (a
    single-match one only at its first match); at each offset, after the reports of that offset, every
    combination that names an id set there is evaluated and reports at that offset if true; at the end of
    the block a combination that is true with none of its sub-expressions matched reports at the end.  A
    block shorter than the shortest match is not scanned."""
    if len(data) < min_width:
        return []
    events = {}
    for sid, rx, quiet, single in subs:
        for e in _ends(rx, data):
            events.setdefault(e, []).append((sid, quiet, single))
    out, seen, first = [], set(), {}

    def bounded(lo, hi, t):
        return (lo == 0 or t >= lo) and (hi == MAX_OFFSET or t <= hi)

    for t in sorted(events):
        touched = set()
        for sid, quiet, single in sorted(events[t]):
            if single and first.setdefault(sid, t) != t:
                continue
            if not quiet:
                out.append((t, sid))
            seen.add(sid)
            touched.add(sid)
        for cid, c, single, lo, hi in combs:
            if touched & set(c.leaves()) and bounded(lo, hi, t) and not (single and cid in first) and c.value(seen):
                out.append((t, cid))
                first[cid] = t
    end = len(data)
    for cid, c, single, lo, hi in combs:
        if not (set(c.leaves()) & seen) and bounded(lo, hi, end) and not (single and cid in first) \
                and c.value(seen):
            out.append((end, cid))
            first[cid] = end
    return out


WORDS = ["abc", "bcd", "xyz", "zz", "qa", "abq", "cab", "yzx"]
REGEXES = ["ab[cq]", "x.{0,3}z", "q+a", "c(ab|zz)", "b.*d"]


def _random_tree(rng, ids, depth=0):
    if depth > 2 or rng.random() < 0.35:
        return ("id", rng.choice(ids))
    op = rng.choice(["!", "&", "|", "&", "|"])
    if op == "!":
        return ("!", _random_tree(rng, ids, depth + 1))
    return (op, _random_tree(rng, ids, depth + 1), _random_tree(rng, ids, depth + 1))


def fuzz_case(seed, literal_only):
    """A random set: 2-5 sub-expressions (literals, or regexes too), 1-3 combinations over them, with quiet
    flags, single-match combinations and offset bounds; and a corpus."""
    rng = random.Random(seed)
    pool = WORDS if literal_only else WORDS + REGEXES
    n = rng.randint(2, 5)
    subs = [(100 + i, rng.choice(pool), rng.random() < 0.3, (not literal_only) and rng.random() < 0.15)
            for i in range(n)]
    subs = [(i, rx, q and not s, s) for i, rx, q, s in subs]        # quiet + single-match is refused
    ids = [s[0] for s in subs]
    combs = []
    for k in range(rng.randint(1, 3)):
        t = _random_tree(rng, ids)
        if t[0] == "id":
            t = ("!", t) if rng.random() < 0.5 else ("|", t, ("id", rng.choice(ids)))
        lo = rng.choice([0, 0, 0, 5, 20])
        hi = rng.choice([MAX_OFFSET, MAX_OFFSET, 30, 60])
        combs.append((1000 + k, Comb(t), rng.random() < 0.25, lo, max(lo, hi)))
    data = bytes(rng.choice(b"abcdqxyz") for _ in range(rng.randint(0, 70)))
    return subs, combs, data


def compile_fuzz(hs, subs, combs):
    exprs = [rx.encode() for _, rx, _, _ in subs] + [c.text().encode() for _, c, _, _, _ in combs]
    flags = [(hs.HS_FLAG_QUIET if q else 0) | (hs.HS_FLAG_SINGLEMATCH if s else 0) for _, _, q, s in subs]
    flags += [hs.HS_FLAG_COMBINATION | (hs.HS_FLAG_SINGLEMATCH if s else 0) for _, _, s, _, _ in combs]
    ids = [s[0] for s in subs] + [c[0] for c in combs]
    ext = [None] * len(subs)
    for _, _, _, lo, hi in combs:
        e = {}
        if lo:
            e["min_offset"] = lo
        if hi != MAX_OFFSET:
            e["max_offset"] = hi
        ext.append(e or None)
    return hs.compile_ext_multi(exprs, flags, ids, ext)


def _min_width(subs):
    return min(min(len(m) for m in _expand(rx)) for _, rx, _, _ in subs)


def _expand(rx):
    """the shortest strings of a fuzz regex, enough for its minimum width"""
    return {"ab[cq]": ["abc"], "x.{0,3}z": ["xz"], "q+a": ["qa"], "c(ab|zz)": ["cab"], "b.*d": ["bd"]}.get(rx, [rx])


def _raw_records(subs, combs, data, block):
    """The raw records a scan writes for one block, from the definition: the reports of the non-quiet
    sub-expressions and a logical-key record (bit 63 of `to`) per sub-expression match, with lkeys in
    order of first mention in the combinations."""
    lkeys = {}
    for _, c, _, _, _ in combs:
        for leaf in _leaf_order(c.text()):
            lkeys.setdefault(leaf, len(lkeys))
    recs = []
    for sid, rx, quiet, _ in subs:
        for e in _ends(rx, data):
            if not quiet:
                recs.append((sid, block, e))
            if sid in lkeys:
                recs.append((lkeys[sid], block, e | (1 << 63)))
    return recs


def _leaf_order(text):
    return [int(x) for x in re.findall(r"\d+", text)]


# ---- CPU ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("regex_dfa", [1, 0])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_reference_scans_our_database(hs, ref, case, regex_dfa):
    """unit/hyperscan/logical_combination.cpp: the unmodified reference hs_scan on our database
    delivers the expected callbacks in order (single-outfix databases, McClellan and LimEx)"""
    hs.set_build_option("regex_dfa", regex_dfa)
    db = _compile(hs, case)
    assert _ref_order(ref, db, case["data"].encode()) == [tuple(m) for m in case["matches"]]


def test_reference_scans_our_pure_literal_database(hs, ref):
    """the same rules on the literal route (a pure-literal database): SingleComb1 with its regular
    expressions replaced by literals, with and without quiet sub-expressions"""
    data = b"abcdefxxfoobarrrghabcxdefxteakettleeeeexxxxijklmxxdef"
    for quiet in (False, True):
        subs = [(101, "abc", quiet, False), (102, "def", quiet, False), (103, "rrgh", quiet, False),
                (104, "teakettle", quiet, False), (105, "ijklm", False, False)]
        combs = [(1001, Comb(("|", ("&", ("&", ("id", 101), ("id", 102)), ("id", 103)),
                                   ("&", ("id", 104), ("!", ("id", 105))))), False, 0, MAX_OFFSET),
                 (1002, Comb(("&", ("!", ("id", 101)), ("id", 102))), True, 0, MAX_OFFSET)]
        db = compile_fuzz(hs, subs, combs)
        want = evaluate(subs, combs, data, 3)
        assert (1001 in [i for _, i in want]) and _ref_order(ref, db, data) == want


@pytest.mark.parametrize("case", BAD, ids=[str(c["id"]) for c in BAD])
def test_combination_parse_errors(hs, case):
    """unit/hyperscan/bad_patterns.txt rows 151-163: the reference's words and character index"""
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi([base64.b64decode(case["pattern"])], [hs.HS_FLAG_COMBINATION], [1])
    assert e.value.message == case["message"]


def test_combination_set_errors(hs):
    C, Q, S = hs.HS_FLAG_COMBINATION, hs.HS_FLAG_QUIET, hs.HS_FLAG_SINGLEMATCH

    def err(exprs, flags, ids, ext=None, mode=None):
        with pytest.raises(hs.HsError) as e:
            if mode is not None:
                hs.compile_multi(exprs, flags, ids, mode=mode)
            else:
                hs.compile_ext_multi(exprs, flags, ids, ext or [None] * len(exprs))
        return e.value.message

    assert err([b"abc", b"1 & !2"], [0, C | hs.HS_FLAG_CASELESS], [1, 9]).startswith(
        "only HS_FLAG_QUIET and HS_FLAG_SINGLEMATCH")
    assert err([b"abc", b"1 & !2"], [0, C], [1, 9], [None, {"min_length": 3}]).startswith(
        "only HS_EXT_FLAG_MIN_OFFSET and HS_EXT_FLAG_MAX_OFFSET")
    assert err([b"abc", b"def", b"1 & 2"], [0, 0, C], [1, 3, 9]) == "Unknown sub-expression id."
    assert err([b"abc", b"def", b"1 & !2", b"1 | 8"], [0, 0, C, C], [1, 2, 8, 9]) == \
        "Have combination of combination."
    # (SOM is refused for any expression in this build, before the set is looked at)
    assert err([b"abc", b"def", b"1 & 2"], [hs.HS_FLAG_SOM_LEFTMOST, 0, C], [1, 2, 9])
    assert err([b"abc", b"def", b"1 & 2"], [hs.HS_FLAG_PREFILTER, 0, C], [1, 2, 9]) == \
        "Have PREFILTER flag in sub-expression."
    # streaming / vectored: the stream state would have to carry the combination state
    for mode in (hs.HS_MODE_STREAM, hs.HS_MODE_VECTORED):
        assert "block mode" in err([b"abc", b"def", b"1 & 2"], [0, 0, C], [1, 2, 9], mode=mode)
    # quiet + single-match on an expression that is not a combination (SET_EXHAUST)
    assert "HS_FLAG_QUIET together with HS_FLAG_SINGLEMATCH" in err([b"abc", b"def", b"1 & 2"], [Q | S, 0, C],
                                                                     [1, 2, 9])
    # a quiet combination is dropped unparsed, as in the reference; quiet alone compiles
    hs.compile_multi([b"abc", b"((("], [Q, C | Q], [1, 2])


FUZZ = [(seed, seed % 3 == 0) for seed in range(300)]


@pytest.mark.parametrize("seed,literal_only", FUZZ, ids=[str(s) for s, _ in FUZZ])
def test_fuzz_against_definition_and_reference(hs, ref, seed, literal_only):
    subs, combs, data = fuzz_case(seed, literal_only)
    db = compile_fuzz(hs, subs, combs)
    want = evaluate(subs, combs, data, _min_width(subs))
    assert _ref_order(ref, db, data) == want


@pytest.mark.parametrize("seed", range(0, 300, 6))
def test_postprocess_blocks_orders_shuffled_raw_records(hs, seed):
    """hs_b200_postprocess_blocks: the raw records of many blocks, logical-key records included,
    shuffled and duplicated, give the delivered sequence of every block; no device needed.  (Pure-literal
    databases: the raw records of a single-outfix database name report programs.)"""
    subs, combs, _ = fuzz_case(seed, True)
    db = compile_fuzz(hs, subs, combs)
    rng = random.Random(seed)
    blocks = [fuzz_case(seed * 1000 + b, True)[2] for b in range(12)] + [b"", b"x" * 40]
    raw, want = [], []
    for b, data in enumerate(blocks):
        raw += _raw_records(subs, combs, data, b)
        want += [(b, t, i) for t, i in evaluate(subs, combs, data, _min_width(subs))]
    raw += raw[: len(raw) // 3]
    rng.shuffle(raw)
    recs = np.array(raw, dtype=hs.MATCH_DTYPE) if raw else np.zeros(0, dtype=hs.MATCH_DTYPE)
    got = hs.postprocess_blocks(db, recs, [len(d) for d in blocks])
    assert [(int(r["block"]), int(r["to"]), int(r["id"])) for r in got] == want
    with pytest.raises(hs.HsError):
        hs.postprocess_matches(db, recs)         # needs the block lengths


def test_database_without_combinations_unchanged(hs):
    """no combination: the bytecode has no combination tables and postprocess_matches still works"""
    db = hs.compile_multi([b"abc", b"def"], [0, 0], [1, 2])
    raw = np.array([(1, 0, 3), (2, 0, 9), (1, 0, 3)], dtype=hs.MATCH_DTYPE)
    assert hs.postprocess_matches(db, raw).size == 2
    assert hs.postprocess_blocks(db, raw, [10]).size == 2


# ---- GPU ---------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("regex_dfa", [1, 0])
def test_device_fixture_cases(hs, regex_dfa):
    """every reference test through hs_scan on the device: callbacks compared in order"""
    hs.set_build_option("regex_dfa", regex_dfa)
    for case in CASES:
        db = _compile(hs, case)
        scratch = hs.Scratch(db)
        rc, out = hs.scan(db, case["data"].encode(), scratch)
        assert rc == 0 and [(t, i) for i, t in out] == [tuple(m) for m in case["matches"]], case["name"]
        scratch.free()


@pytest.mark.gpu
def test_device_fuzz_hs_scan(hs, ref):
    for seed in range(0, 300, 3):
        subs, combs, data = fuzz_case(seed, seed % 3 == 0)
        db = compile_fuzz(hs, subs, combs)
        scratch = hs.Scratch(db)
        rc, out = hs.scan(db, data, scratch)
        assert rc == 0 and [(t, i) for i, t in out] == _ref_order(ref, db, data), seed
        scratch.free()


def _many_blocks(seed, n):
    rng = random.Random(seed)
    blocks = []
    for b in range(n):
        k = rng.random()
        if k < 0.05:
            blocks.append(b"")
        elif k < 0.15:
            blocks.append(b"x" * rng.randint(1, 80))           # nothing but negated sub-expressions hold
        else:
            blocks.append(bytes(rng.choice(b"abcdqxyz") for _ in range(rng.randint(1, 90))))
    pitch = 96
    data = np.zeros(n * pitch, dtype=np.uint8)
    for b, d in enumerate(blocks):
        data[b * pitch: b * pitch + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return blocks, data, np.arange(n, dtype=np.uint64) * pitch, np.array([len(d) for d in blocks], np.uint32)


def _ref_blocks(ref, db, data, off, ln):
    recs, _ = ref.scan_collect(db.ptr, data, off, ln)
    return [(int(r["block"]), int(r["to"]), int(r["id"])) for r in recs]


def _as_list(recs):
    return [(int(r["block"]), int(r["to"]), int(r["id"])) for r in recs]


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 5, 9, 12, 33])
def test_device_blocks_collect_and_resident(hs, ref, seed):
    """thousands of blocks through hs_b200_scan_blocks_collect, hs_b200_scan_blocks and a resident corpus
    with hs_b200_fetch_matches: combination state is per block; some blocks are empty, some hold only
    bytes that match nothing (purely negative combinations report at their end)"""
    subs, combs, _ = fuzz_case(seed, seed % 3 == 0)
    db = compile_fuzz(hs, subs, combs)
    blocks, data, off, ln = _many_blocks(seed, 3000)
    want = _ref_blocks(ref, db, data, off, ln)
    scratch = hs.Scratch(db)
    out = np.zeros(len(want) + 16, dtype=hs.MATCH_DTYPE)
    n = hs.scan_blocks_collect(db, data, off, ln, scratch, out)
    assert _as_list(out[:n]) == want
    assert _as_list(hs.scan_blocks(db, data, off, ln, scratch)) == want
    assert hs.scan_blocks(db, data, off, ln, scratch, collect=False) == len(want)
    corpus = hs.Corpus.upload(data, off, ln)
    assert _as_list(hs.scan_corpus(db, corpus, scratch)) == want
    corpus.free()
    scratch.free()


@pytest.mark.gpu
def test_device_small_ring_rescan(hs, ref):
    """a 16-record ring: the records, logical-key records included, overflow it and the scan runs again"""
    subs = [(1, "a", False, False), (2, "b", True, False)]
    combs = [(9, Comb(("&", ("id", 1), ("!", ("id", 2)))), False, 0, MAX_OFFSET)]
    db = compile_fuzz(hs, subs, combs)
    blocks, data, off, ln = _many_blocks(77, 400)
    want = _ref_blocks(ref, db, data, off, ln)
    hs.set_runtime_option("initial_ring", 16)
    try:
        scratch = hs.Scratch(db)
        assert _as_list(hs.scan_blocks(db, data, off, ln, scratch)) == want and len(want) > 1000
        scratch.free()
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)


@pytest.mark.gpu
def test_device_termination_on_a_combination_report(hs, ref):
    """a callback that stops the scan at a combination report: nothing after it is delivered"""
    case = CASES[0]
    db = _compile(hs, case)
    data = case["data"].encode()
    scratch = hs.Scratch(db)
    for stop in (4, 6, 16):
        rc, out = hs.scan(db, data, scratch, stop_after=stop)
        assert rc == hs.HS_SCAN_TERMINATED and [(t, i) for i, t in out] == _ref_order(ref, db, data, stop_after=stop)
        assert out[-1][0] == 1001
    scratch.free()


LIT_SETS = {"noodle": [b"abcq"], "teddy": [b"ab", b"bcd", b"xyz", b"qa"],
            "fdr": [b"w%03dz" % i for i in range(200)] + [b"abc", b"xyz", b"qa"]}


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["noodle", "teddy", "fdr", "mcclellan8", "limex32"])
def test_device_literal_engines(hs, ref, engine):
    """the literal matchers (noodle, Teddy, FDR) and single-outfix engines (McClellan, LimEx) all carry the
    logical-key records"""
    lits = LIT_SETS.get(engine, LIT_SETS["teddy"])
    if engine in ("mcclellan8", "limex32"):
        hs.set_build_option("outfix_engine", 2 if engine == "mcclellan8" else 5)
    n = len(lits)
    ids = list(range(1, n + 1))
    a, b = ids[-1], ids[-2] if n > 1 else ids[-1]
    exprs = [re.escape(l.decode()).encode() for l in lits] + [b"%d & !%d" % (a, b), b"!%d" % ids[0],
                                                                b"(%d | %d) & !%d" % (a, ids[0], b)]
    flags = [0] * n + [hs.HS_FLAG_COMBINATION] * 3
    flags[0] |= hs.HS_FLAG_QUIET
    db = hs.compile_multi(exprs, flags, ids + [900, 901, 902])
    blocks, data, off, ln = _many_blocks(3, 2000)
    for b in range(0, 2000, 5):
        lit = lits[b % n]
        p = int(off[b]) + (b * 7) % max(1, int(ln[b]) - len(lit) + 1)
        if int(ln[b]) >= len(lit):
            data[p:p + len(lit)] = np.frombuffer(lit, dtype=np.uint8)
    want = _ref_blocks(ref, db, data, off, ln)
    scratch = hs.Scratch(db)
    assert _as_list(hs.scan_blocks(db, data, off, ln, scratch)) == want and len(want) > 500
    scratch.free()
