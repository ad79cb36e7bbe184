"""Regular-expression sets too large for one automaton: several engines (McClellan-8 / 16, LimEx), each run as an
outfix on its own queue, in one FULL_ROSE database without a literal matcher (rose_build.cpp
buildMultiOutfixRose; DESIGN.md section 10e).  A set takes this route only where its one automaton raised the
set-level "Pattern set is too large" error, no expression of it expands to literals, it has no combination and the
mode is block.

CPU half: the UNMODIFIED reference hs_scan on our databases equals the definition -- every end offset of a match
(test_regex._ends, or re.fullmatch over every start and end for expressions without anchors or word boundaries),
one report per (id, offset), and for HS_FLAG_SINGLEMATCH ids only the first per block -- and reproduces the
recorded hscollider vectors of groups of 30-60 expressions.  GPU half: the device, through every scan entry point
and the device ordering, equals the reference per block."""
import base64
import re

import numpy as np
import pytest

from test_golden import COLLIDER_REGEX
from test_mixed_rose import MixedSet, _blocks, _device_all_entries, _pack, _per_block, _ref_per_block
from test_regex import _ends, _ends_ext

CASELESS, DOTALL, SINGLE = 1, 2, 8
SET_TOO_LARGE = "Pattern set is too large: its character positions exceed the 512-state NFA model."
ALPHA = b"abcdqrstxyz0123 "
ENGINE_KIND = {6: "mcclellan8", 7: "mcclellan16", 0: "limex", 1: "limex", 2: "limex", 3: "limex", 4: "limex",
               5: "limex"}   # enum NFAEngineType of a single-outfix database


def _plain(pat):
    """no anchor or word boundary: the definition is re.fullmatch over [start, end)"""
    return not re.search(rb"\$|\^|\\[zZbBA]", pat)


def _def_ends(pat, fl, block):
    if not _plain(pat):
        return _ends(pat, fl, block)
    rx = re.compile(pat, (re.I if fl & CASELESS else 0) | (re.S if fl & DOTALL else 0))
    return sorted({e for s in range(len(block)) for e in range(s + 1, len(block) + 1) if rx.fullmatch(block, s, e)})


class RegexSet(MixedSet):
    """a set of regular expressions only: (pattern, flags, id, ext or None)"""

    def __init__(self, regexes):
        super().__init__([], [], [], regexes)

    def definition(self, block):
        got, single = set(), set()
        for pat, fl, rid, ext in self.regexes:
            ends = _ends_ext(pat, fl, block, **ext) if ext else _def_ends(pat, fl, block)
            got.update((e, rid) for e in ends)
            if fl & SINGLE:
                single.add(rid)
        out, seen = [], set()
        for to, rid in sorted(got):
            if rid in single:
                if rid in seen:
                    continue
                seen.add(rid)
            out.append((to, rid))
        return out


# ---- seeded sets that overflow one automaton ------------------------------------------------------------------------

def _seeded(seed, n):
    """n expressions of 5-60 positions: a prefix, a counted class, a repeated suffix; and a sample match of each"""
    rng = np.random.default_rng(seed)
    regexes, samples = [], []
    for i in range(n):
        pre = bytes(rng.choice(list(b"qrst"), size=int(rng.integers(2, 4))).tolist())
        cls, chars = [(b"[a-d]", b"abcd"), (b"[0-3]", b"0123"), (b"[a-dx]", b"abcdx")][int(rng.integers(0, 3))]
        lo = int(rng.integers(2, 12))
        hi = lo + int(rng.integers(0, 45))
        suf = bytes([int(rng.choice(list(b"xyz")))])
        fl = CASELESS if rng.random() < 0.15 else 0
        regexes.append((pre + cls + b"{%d,%d}" % (lo, hi) + suf + b"+", fl, 100 + i, None))   # (not a finite set)
        samples.append(pre + bytes(rng.choice(list(chars), size=int(rng.integers(lo, hi + 1))).tolist()) + suf)
    return RegexSet(regexes), samples


SEEDED = [(1, 30), (2, 60), (3, 110), (4, 170)]   # (seed, expressions): 2, 5, 8 and 12 engines


def _seeded_blocks(samples, seed, n=12):
    return _blocks(seed, n, max_len=72, plant=samples, alphabet=ALPHA, empty_every=5) + [b"", b"q", b"qa"]


@pytest.mark.parametrize("seed,n", SEEDED)
def test_reference_scans_split_sets_as_defined(hs, ref, seed, n):
    rs, samples = _seeded(seed, n)
    db = rs.compile(hs)
    info = db.info()
    assert info.runtime_impl == 0 and info.hwlm_type == 0 and 2 <= info.engine_count <= 12
    blocks = _seeded_blocks(samples, seed)
    got = _ref_per_block(ref, db, blocks)
    assert got == [rs.definition(b) for b in blocks]
    assert sum(map(len, got)) >= 8


# ---- engines of every kind in one database ----------------------------------------------------------------------

# Greedy packing in expression order: each row is one group -- its first expression does not fit beside the
# group before.  Alone, the groups compile to McClellan-16 (a counter of 300), LimEx (a set whose determinised
# automaton passes 1 024 states) and McClellan-8 (a counter of 200 on other bytes, and a small expression).
KIND_GROUPS = [[(rb"q[a-d]{300}z", 0, 1, None)],
               [(rb"r[0-3]{300}s", 0, 2, None), (rb"x[ab]*a[ab]{10}y", 0, 3, None)],
               [(rb"t[0-3]{200}u", 0, 4, None), (rb"xy+z", CASELESS, 5, None)]]


def _kind_blocks(seed):
    plant = [b"q" + b"abcd" * 75 + b"z", b"r" + b"0123" * 75 + b"s", b"t" + b"30" * 100 + b"u",
             b"xba" + b"ab" * 5 + b"y", b"xbbbba" + b"ba" * 5 + b"y", b"xYYz"]
    blocks = _blocks(seed, 6, max_len=360, plant=plant, alphabet=b"abcd0123xyz", empty_every=4)
    return blocks + plant


@pytest.mark.parametrize("dfa", [1, 0])
def test_reference_scans_engines_of_every_kind(hs, ref, dfa):
    hs.set_build_option("regex_dfa", dfa)
    kinds = []
    for g in KIND_GROUPS:
        alone = RegexSet(g).compile(hs).info()
        assert alone.runtime_impl == 2 and alone.engine_count == 1
        kinds.append(ENGINE_KIND[alone.engine_id])
    assert kinds == (["mcclellan16", "limex", "mcclellan8"] if dfa else ["limex"] * 3)
    rs = RegexSet([r for g in KIND_GROUPS for r in g])
    db = rs.compile(hs)
    assert db.info().engine_count == len(KIND_GROUPS) and db.info().min_width == 3   # "xy+z"
    blocks = _kind_blocks(3)
    got = _ref_per_block(ref, db, blocks)
    assert got == [rs.definition(b) for b in blocks]
    assert {i for g in got for _, i in g} == {1, 2, 3, 4, 5}


# ---- the report rules across engines ----------------------------------------------------------------------------

FILLER = [(rb"q[a-d]{300}z", 0, 90, None), (rb"r[a-d]{300}s", 0, 91, None), (rb"t[a-d]{300}u", 0, 92, None)]


def _rules_set(single):
    """(no expression is a finite set of literals) ids raised by expressions in different engines (7 and 9 at the same offsets), a single-match id across
    engines, hs_expr_ext bounds and min_length, and $ / \\z / \\b accepts at the end of data in every engine"""
    s = SINGLE if single else 0
    a = [(rb"ab+c", 0, 7, None), (rb"\d\.\d+", s, 9, None), (rb"d+q", 0, 20, {"min_offset": 6, "max_offset": 40}),
         (rb"zq?$", 0, 22, None), (rb"y\z", 0, 23, None)]
    b = [(rb"a[bc]+c", 0, 7, None), (rb"[0-9]+\.[0-9]", s, 9, None), (rb"a[bc]+", 0, 21, {"min_length": 4}),
         (rb"\bdd", 0, 10, None), (rb"\w+y\b", 0, 24, None), (rb"c$", 0, 25, None)]
    c = [(rb"bc+", 0, 7, None), (rb"x.y\z", 0, 26, None), (rb"\d+\.", s, 9, None)]
    return RegexSet(a + FILLER[:1] + FILLER[1:2] + b + FILLER[2:] + c)


def _rules_blocks(seed, n=40):
    return _blocks(seed, n, max_len=48, plant=[b"abbc", b"xay", b"0.12", b"ddq", b" dd", b"abcbc", b"3.4 5.6"],
                   alphabet=b"abcdqxyz.012 ", empty_every=7) + [b"", b"z", b"dd", b"abbc", b"y", b"1.2", b"xzy"]


@pytest.mark.parametrize("single", [0, 1])
@pytest.mark.parametrize("dfa", [1, 0])
def test_reference_applies_report_rules_across_engines(hs, ref, single, dfa):
    hs.set_build_option("regex_dfa", dfa)
    rs = _rules_set(single)
    db = rs.compile(hs)
    assert db.info().engine_count == 3 and db.info().min_width == 1
    blocks = _rules_blocks(3)
    got = _ref_per_block(ref, db, blocks)
    assert got == [rs.definition(b) for b in blocks]
    assert got[-4] == [(4, 7), (4, 21), (4, 25)]        # "abbc": three engines raise id 7 at 4, one report
    if single:
        assert all(sum(i == 9 for _, i in g) <= 1 for g in got)
    flat = [i for g in got for _, i in g]
    assert all(i in flat for i in (7, 9, 10, 20, 21, 22, 23, 24, 25, 26))


# ---- recorded hscollider vectors, 30-60 expressions per database --------------------------------------------------

def _collider_groups(n_groups=8, seed=9):
    rng = np.random.default_rng(seed)
    cases = [c for c in COLLIDER_REGEX if not c.get("ext")]
    return [[cases[i] for i in rng.choice(len(cases), size=int(rng.integers(30, 61)), replace=False)]
            for _ in range(n_groups)]


def _collider_corpus(group):
    """every corpus of every member as one block, 16-byte aligned; (member, its corpus index) per block"""
    buf, off, ln, who = bytearray(), [], [], []
    for k, c in enumerate(group):
        for j, cp in enumerate(c["corpora"]):
            d = base64.b64decode(cp["data"])
            while len(buf) % 16:
                buf.append(0)
            off.append(len(buf))
            ln.append(len(d))
            who.append((k, j))
            buf += d
    data = np.frombuffer(bytes(buf) + b"\0" * 16, dtype=np.uint8)
    return data, np.array(off, np.uint64), np.array(ln, np.uint32), who


COLLIDER_GROUPS = _collider_groups()


@pytest.mark.parametrize("gi", range(len(COLLIDER_GROUPS)))
def test_reference_reproduces_recorded_vectors_of_split_groups(hs, ref, gi):
    group = COLLIDER_GROUPS[gi]
    try:
        db = hs.compile_multi([base64.b64decode(c["pattern"]) for c in group], [c["hs_flags"] for c in group],
                              [1000 + k for k in range(len(group))])
    except hs.HsError as e:
        assert str(e).startswith("Pattern set is too large")   # more engines than a database holds
        return
    data, off, ln, who = _collider_corpus(group)
    got = ref.scan_sorted(db.ptr, data, off, ln)
    for b, (k, j) in enumerate(who):
        tos = [int(r["to"]) for r in got[(got["block"] == b) & (got["id"] == 1000 + k)]]
        want = group[k]["corpora"][j]["ends"]
        if "H" in group[k]["flag_letters"]:
            assert (len(tos) == 1 and tos[0] in want) if want else not tos, (gi, k, j, tos, want)
        else:
            assert tos == want, (gi, k, j, tos, want)
    assert not np.any(got["id"] >= 1000 + len(group))


def test_most_recorded_groups_overflow_one_automaton(hs):
    counts = []
    for group in COLLIDER_GROUPS:
        try:
            counts.append(hs.compile_multi([base64.b64decode(c["pattern"]) for c in group],
                                           [c["hs_flags"] for c in group], list(range(len(group)))).info().engine_count)
        except hs.HsError:
            counts.append(None)
    assert sum(1 for n in counts if n and n >= 2) > len(counts) // 2, counts


# ---- which sets take the route ----------------------------------------------------------------------------------

def _error(hs, exprs, flags=None, ids=None, **kw):
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi(exprs, flags, ids, **kw)
    return e.value.message, e.value.expression


def test_which_sets_take_the_route(hs):
    assert hs.compile_multi([rb"ab+c", rb"x.y"]).info().engine_count == 1            # fits one automaton: as before
    assert hs.compile_multi([rb"ab+c", rb"x.y"]).info().runtime_impl == 2
    rs, _ = _seeded(1, 30)
    info = rs.compile(hs).info()
    assert (info.runtime_impl, info.engine_count) == (0, 2)
    # the same set always compiles to the same bytes
    assert rs.compile(hs).serialize() == rs.compile(hs).serialize()


def test_errors_stay_as_before(hs):
    fill = [r[0] for r in FILLER]
    # literals plus oversized regexes: the literal-matcher route's error, message and index unchanged
    lits = [b"abcd%d" % i for i in range(1000)]
    msg, idx = _error(hs, lits + [rb"q[a-d]{300}z", rb"r[a-d]{300}z"])
    assert msg == SET_TOO_LARGE and idx < 1000
    # one expression alone does not fit an engine (its min_length levels): the one automaton's error, which was
    # raised at the second filler
    alone = {"min_length": 200}
    with pytest.raises(hs.HsError) as e:
        hs.compile_ext_multi(fill[:2] + [rb"ab[a-d]+"], [0] * 3, [0, 1, 2], [None, None, alone])
    assert (e.value.message, e.value.expression) == (SET_TOO_LARGE, 1)
    # a combination, streaming and vectored mode keep their errors
    msg, _ = _error(hs, fill + [b"0 & 1"], [0, 0, 0, hs.HS_FLAG_COMBINATION], [0, 1, 2, 3])
    assert msg == SET_TOO_LARGE
    for mode in (hs.HS_MODE_STREAM, hs.HS_MODE_VECTORED):
        assert "block mode only" in _error(hs, fill, mode=mode)[0]
    # a single expression beyond the 510 positions: its own error
    assert _error(hs, fill[:1] + [rb"q[a-d]{600}z"])[0].startswith("Pattern is too large")


def test_host_postprocess_entries_refuse(hs):
    db = _rules_set(0).compile(hs)
    recs = np.zeros(2, dtype=hs.MATCH_DTYPE)
    with pytest.raises(hs.HsError):
        hs.postprocess_matches(db, recs)
    with pytest.raises(hs.HsError):
        hs.postprocess_blocks(db, recs, np.array([10], np.uint32))


# ---- the device ---------------------------------------------------------------------------------------------------

def _device_order_equals_fetch(hs, db, blocks, pitch=None):
    from test_gpu_device_order import _order_last, _scan
    data, off, ln = _pack(blocks, pitch)
    scratch = hs.Scratch(db)
    corpus = hs.Corpus.upload(data, off, ln)
    _scan(hs, db, scratch, corpus)
    want = hs.fetch_matches(db, scratch)
    got, n = _order_last(hs, db, scratch)
    assert n == want.size and np.array_equal(got, want)
    corpus.free()
    scratch.free()
    return _per_block(want, len(blocks))


@pytest.mark.gpu
@pytest.mark.parametrize("seed,n", SEEDED)
def test_device_equals_reference(hs, ref, seed, n):
    rs, samples = _seeded(seed, n)
    db = rs.compile(hs)
    blocks = _seeded_blocks(samples, seed, n=150)
    want = _device_all_entries(hs, ref, db, blocks)
    assert _device_order_equals_fetch(hs, db, blocks) == want
    assert sum(map(len, want)) > 100


@pytest.mark.gpu
@pytest.mark.parametrize("dfa", [1, 0])
def test_device_engines_of_every_kind(hs, ref, dfa):
    hs.set_build_option("regex_dfa", dfa)
    db = RegexSet([r for g in KIND_GROUPS for r in g]).compile(hs)
    blocks = _kind_blocks(5) * 8
    want = _device_all_entries(hs, ref, db, blocks)
    assert _device_order_equals_fetch(hs, db, blocks) == want


@pytest.mark.gpu
@pytest.mark.parametrize("single", [0, 1])
@pytest.mark.parametrize("dfa", [1, 0])
def test_device_report_rules_across_engines(hs, ref, single, dfa):
    hs.set_build_option("regex_dfa", dfa)
    db = _rules_set(single).compile(hs)
    blocks = _rules_blocks(4, 500)
    want = _device_all_entries(hs, ref, db, blocks)
    assert _device_order_equals_fetch(hs, db, blocks) == want


@pytest.mark.gpu
def test_device_small_ring_and_chunked_upload(hs, ref):
    """a 16-record initial ring (overflow, grow, rescan with every engine), then chunk_mb=1"""
    rs, samples = _seeded(3, 110)
    db = rs.compile(hs)
    blocks = _seeded_blocks(samples, 21, n=300)
    hs.set_runtime_option("initial_ring", 16)
    try:
        want = _device_all_entries(hs, ref, db, blocks)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)
    assert len({i for g in want for _, i in g}) > 20
    big = _blocks(22, 2500, max_len=1200, plant=samples, alphabet=ALPHA)
    hs.set_runtime_option("chunk_mb", 1)
    try:
        want = _device_all_entries(hs, ref, db, big)
    finally:
        hs.set_runtime_option("chunk_mb", 128)
    assert sum(map(len, want)) > 1000


@pytest.mark.gpu
def test_device_callback_termination(hs, ref):
    """a callback that stops the scan: HS_SCAN_TERMINATED, and what was delivered is a prefix of (block, to, id)
    over every engine's records"""
    rs = _rules_set(0)
    db = rs.compile(hs)
    data = b"abbc 1.23 dd ddq xay abcbc zq"
    scratch = hs.Scratch(db)
    rc, full = hs.scan(db, data, scratch)
    assert rc == 0 and len(full) >= 8
    assert sorted((to, i) for i, to in full) == [tuple(x) for x in _ref_per_block(ref, db, [data])[0]]
    assert [(to, i) for i, to in full] == sorted((to, i) for i, to in full)
    for stop in (1, 2, 5):
        rc, got = hs.scan(db, data, scratch, stop_after=stop)
        assert rc == hs.HS_SCAN_TERMINATED and got == full[:stop]
    scratch.free()


@pytest.mark.gpu
@pytest.mark.parametrize("nblocks", [4096, 7])
def test_device_uniform_blocks(hs, ref, nblocks):
    """4 096 uniform 1 KiB blocks, and a corpus of fewer blocks than one warp"""
    rs, samples = _seeded(2, 60)
    db = rs.compile(hs)
    blocks = _blocks(31, nblocks, max_len=1024, plant=samples * 4, alphabet=ALPHA)
    blocks = [b.ljust(1024, b" ") for b in blocks]
    want = _device_all_entries(hs, ref, db, blocks, pitch=1024)
    assert _device_order_equals_fetch(hs, db, blocks, pitch=1024) == want
    assert sum(map(len, want)) >= nblocks // 8
