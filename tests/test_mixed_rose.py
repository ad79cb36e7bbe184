"""Sets of literals AND regular expressions: a literal matcher (noodle, Teddy, FDR, the 4-gram stage) beside ONE
engine (McClellan-8 / 16, LimEx) run as the outfix on queue 0 -- a FULL_ROSE database (rose_build.cpp
buildMixedRose; DESIGN.md section 10d).  Such a set takes this route where the expressions' one automaton would
be too large, or always under the build option mixed_rose=1.

CPU half: the UNMODIFIED reference hs_scan on our databases equals the definition -- every literal occurrence
(oracle/brute.py) and every end offset of a regex match (test_regex._ends), one report per (id, offset), and
for HS_FLAG_SINGLEMATCH ids only the first per block -- which pins the bytecode.  GPU half: the device, through
every scan entry point, equals the reference per block."""
import base64
import ctypes as C
import io
import os
import re
import importlib.util
from contextlib import redirect_stdout

import numpy as np
import pytest

import oracle.brute as brute
from hyperscan_b200 import synth
from test_golden import COLLIDER_REGEX, _check_collider, _collider_blocks
from test_regex import _ends, _ends_ext

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASELESS, DOTALL, MULTILINE, SINGLE = 1, 2, 4, 8
ALPHA = b"abcdxyz.0123 qA"


def _esc(lit):
    return b"".join(bytes([c]) if chr(c).isalnum() else b"\\x%02x" % c for c in lit)


def _lits(n, seed, caseless_frac=0.0, min_len=4, max_len=8, alphabet=b"abcdefghijklmnopqrstuvwxyz"):
    lits, flags, _ = synth.literal_set(n, min_len=min_len, max_len=max_len, caseless_frac=caseless_frac, seed=seed,
                                       alphabet=alphabet)
    return lits, flags


class MixedSet:
    """lits (with flags and ids) and regexes: (pattern, flags, id, ext dict or None)"""

    def __init__(self, lits, lflags, lids, regexes):
        self.lits, self.lflags, self.lids, self.regexes = lits, lflags, lids, regexes

    def compile(self, hs, platform=None):
        exprs = [_esc(l) for l in self.lits] + [r[0] for r in self.regexes]
        flags = list(self.lflags) + [r[1] for r in self.regexes]
        ids = list(self.lids) + [r[2] for r in self.regexes]
        ext = [None] * len(self.lits) + [r[3] for r in self.regexes]
        return hs.compile_ext_multi(exprs, flags, ids, ext, platform=platform)

    def definition(self, block):
        """sorted (to, id) of one block"""
        plain = [f & ~SINGLE for f in self.lflags]
        got = set((to, rid) for rid, to in brute.scan_block(self.lits, plain, self.lids, block))
        single = {i for i, f in zip(self.lids, self.lflags) if f & SINGLE}
        for pat, fl, rid, ext in self.regexes:
            got.update((e, rid) for e in (_ends_ext(pat, fl, block, **ext) if ext else _ends(pat, fl, block)))
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


def _blocks(seed, n, max_len=64, plant=(), alphabet=ALPHA, empty_every=0):
    """n blocks of random bytes with literals of `plant` written in; some empty and some short"""
    rng = np.random.default_rng(seed)
    a = np.frombuffer(alphabet, dtype=np.uint8)
    blocks = []
    for b in range(n):
        if empty_every and b % empty_every == 0:
            blocks.append(b"")
            continue
        ln = int(rng.integers(1, max_len + 1)) if b % 3 == 0 else max_len
        d = bytearray(a[rng.integers(0, a.size, size=ln)].tobytes())
        for _ in range(2):
            if plant:
                lit = plant[int(rng.integers(0, len(plant)))]
                if len(lit) <= ln:
                    p = int(rng.integers(0, ln - len(lit) + 1))
                    d[p:p + len(lit)] = lit
        blocks.append(bytes(d))
    return blocks


def _pack(blocks, pitch=None):
    pitch = pitch or max(16, (max(len(b) for b in blocks) + 15) // 16 * 16)
    data = np.zeros(len(blocks) * pitch + 16, dtype=np.uint8)
    for i, d in enumerate(blocks):
        data[i * pitch:i * pitch + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return data, np.arange(len(blocks), dtype=np.uint64) * pitch, np.array([len(d) for d in blocks], np.uint32)


def _per_block(recs, n):
    out = [[] for _ in range(n)]
    for r in recs:
        out[int(r["block"])].append((int(r["to"]), int(r["id"])))
    return [sorted(x) for x in out]


def _ref_per_block(ref, db, blocks):
    data, off, ln = _pack(blocks)
    return _per_block(ref.scan_sorted(db.ptr, data, off, ln), len(blocks))


# ---- the databases: each literal matcher crossed with each engine ------------------------------------------------

REGEX_SMALL = [(rb"ab+c", 0, 5001, None), (rb"\d+\.\d\d", 0, 5002, None), (rb"x.y", 0, 5003, None)]
REGEX_WIDE = [(rb"a[ab]*a[ab]{7}c", 0, 5004, None), (rb"q[0-3]+z", CASELESS, 5005, None)]   # McClellan-16
REGEX_HUGE = [(rb"q[a-d0-3]{270}z", 0, 5006, None), (rb"ab+c", 0, 5001, None)]         # > 256 positions: LimEx-512
LITERAL_KINDS = {  # name -> (count, route): small sets need mixed_rose=1, large ones overflow the automaton
    "noodle": (1, 1), "teddy": (12, 1), "fat_teddy": (60, 1), "fdr": (1000, 0), "gram4": (10000, 0)}
ENGINES = {"mcclellan8": (REGEX_SMALL, 1), "mcclellan16": (REGEX_WIDE, 1), "limex": (REGEX_SMALL, 0),
           "limex512": (REGEX_HUGE, 0)}
ENGINE_IDS = {"mcclellan8": 6, "mcclellan16": 7, "limex": 0, "limex512": 5}   # enum NFAEngineType


def _platform(hs, kind):
    if kind != "fat_teddy":
        return None
    return C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0))   # 16-bucket Teddy is allowed


def _kind_set(hs, kind, engine, seed=1):
    n, route = LITERAL_KINDS[kind]
    regexes, dfa = ENGINES[engine]
    lits, flags = _lits(n, seed, caseless_frac=0.1, min_len=4 if n > 1 else 5)
    hs.set_build_option("mixed_rose", route)
    hs.set_build_option("regex_dfa", dfa)
    ms = MixedSet(lits, flags, list(range(len(lits))), regexes)
    db = ms.compile(hs, _platform(hs, kind))
    return ms, db


def _expect_hwlm(hs, db, kind):
    info = db.info()
    assert info.runtime_impl == 0
    if kind == "noodle":
        assert info.hwlm_type == 16
    elif kind == "teddy":
        assert info.hwlm_type == 12 and 11 <= info.engine_id <= 18
    elif kind == "fat_teddy":
        assert info.hwlm_type == 12 and 3 <= info.engine_id <= 10
    else:
        assert info.hwlm_type == 12 and info.engine_id == 0


def _kind_blocks(ms, seed, n=24):
    plant = list(ms.lits[:40]) + [b"abbbc", b"12.345", b"xay", b"aababbabc", b"q0123Z"]
    huge = any(r[2] == 5006 for r in ms.regexes)
    blocks = _blocks(seed, n, max_len=300 if huge else 64, plant=plant,
                     alphabet=b"abcdxyz.0123 qA" + bytes(sorted(set(b"".join(ms.lits[:40])))), empty_every=11)
    return blocks + ([b"xx q" + b"a0" * 135 + b"z abbc", b"q" + b"b3" * 135 + b"zq" + b"a" * 270 + b"z"] if huge else [])


KIND_X_ENGINE = [(k, e) for k in LITERAL_KINDS for e in ENGINES]


@pytest.mark.parametrize("kind,engine", KIND_X_ENGINE)
def test_reference_scans_mixed_database_as_defined(hs, ref, kind, engine):
    ms, db = _kind_set(hs, kind, engine)
    _expect_hwlm(hs, db, kind)
    # the engine half is the automaton the regexes alone compile to
    alone = hs.compile_ext_multi([r[0] for r in ms.regexes], [r[1] for r in ms.regexes], [r[2] for r in ms.regexes])
    assert alone.info().runtime_impl == 2 and alone.info().engine_id == ENGINE_IDS[engine]
    blocks = _kind_blocks(ms, 7, n=8 if engine == "limex512" else 24)   # (300-byte blocks: a slow definition)
    got = _ref_per_block(ref, db, blocks)
    assert got == [ms.definition(b) for b in blocks]
    assert sum(map(len, got)) > 10 or engine == "limex512" and sum(i == 5006 for g in got for _, i in g) >= 2


# ---- the report rules across both halves ------------------------------------------------------------------------

def _rules_set():
    """ids shared by literals and regexes (one at the same offset as a regex match), a shared SINGLEMATCH id,
    caseless literals, hs_expr_ext bounds and min_length, end anchors and word boundaries"""
    lits = [b"abbc", b"xay", b"0.12", b"dd", b"QQq", b"zz"]
    lflags = [0, 0, SINGLE, 0, CASELESS, 0]
    lids = [7, 8, 9, 10, 11, 12]
    regexes = [(rb"ab+c", 0, 7, None),                      # abbc: both halves at one offset, one report
               (rb"x.y", 0, 8, None),
               (rb"\d\.\d+", SINGLE, 9, None),              # single-match across both halves
               (rb"d+q", 0, 20, {"min_offset": 6, "max_offset": 40}),
               (rb"a[bc]+", 0, 21, {"min_length": 4}),
               (rb"zq?$", 0, 22, None), (rb"y\z", 0, 23, None), (rb"\bdd", 0, 10, None), (rb"\w+y\b", 0, 24, None)]
    return MixedSet(lits, lflags, lids, regexes)


def _rules_blocks(seed, n=40):
    return _blocks(seed, n, max_len=48, plant=[b"abbc", b"xay", b"0.12", b"ddq", b"qqQ", b"zz", b" dd", b"abcbc"],
                   alphabet=b"abcdqxyz.012 ", empty_every=7)


@pytest.mark.parametrize("dfa", [1, 0])
@pytest.mark.parametrize("route", [1, 0])
def test_reference_applies_report_rules_across_both_halves(hs, ref, dfa, route):
    ms = _rules_set()
    hs.set_build_option("regex_dfa", dfa)
    if route:
        hs.set_build_option("mixed_rose", 1)
    else:   # the same rules where the literals overflow the automaton
        extra, _ = _lits(1000, 4, alphabet=b"EFGHIJKLMNOP")
        ms.lits = list(ms.lits) + extra
        ms.lflags = list(ms.lflags) + [0] * len(extra)
        ms.lids = list(ms.lids) + list(range(100, 100 + len(extra)))
    db = ms.compile(hs)
    assert db.info().runtime_impl == 0
    assert db.info().min_width == 1   # \bdd, zq?$ ... the shortest match of either half; "zz" and "dd" are longer
    blocks = _rules_blocks(3) + [b"", b"z", b"dd", b"abbc", b"y"]
    got = _ref_per_block(ref, db, blocks)
    assert got == [ms.definition(b) for b in blocks]
    assert got[-2] == [(4, 7), (4, 21)]                          # "abbc": literal and regex of id 7, one report
    assert all(sum(i == 9 for _, i in g) <= 1 for g in got)      # single-match across both halves
    flat = [i for g in got for _, i in g]
    assert all(i in flat for i in (9, 10, 11, 20, 21, 22, 23))


def test_min_width_covers_both_halves(hs, ref):
    """blocks shorter than minWidth are not scanned: the shortest match is the regex half's here"""
    hs.set_build_option("mixed_rose", 1)
    ms = MixedSet([b"abcdefgh"], [0], [1], [(rb"xy+z", 0, 2, None)])
    db = ms.compile(hs)
    assert db.info().min_width == 3
    blocks = [b"", b"xy", b"xyz", b"abcdefgh", b"xyyz abcdefgh"]
    assert _ref_per_block(ref, db, blocks) == [ms.definition(b) for b in blocks] == [[], [], [(3, 2)], [(8, 1)],
                                                                                    [(4, 2), (13, 1)]]


# ---- the reference's recorded vectors beside 1 000 literals ------------------------------------------------------

FILLER, _ = _lits(1000, 11, alphabet=bytes(range(0xc0, 0xd0)))   # bytes no recorded corpus holds
SAMPLE = COLLIDER_REGEX[::23]


def _with_filler(hs, case):
    exprs = [base64.b64decode(case["pattern"])] + [_esc(l) for l in FILLER]
    return hs.compile_ext_multi(exprs, [case["hs_flags"]] + [0] * len(FILLER),
                                [case["id"]] + list(range(20000, 20000 + len(FILLER))),
                                [case.get("ext")] + [None] * len(FILLER))


@pytest.mark.parametrize("case", SAMPLE, ids=[str(c["id"]) for c in SAMPLE])
def test_reference_reproduces_recorded_vectors_beside_literals(hs, ref, case):
    try:
        db = _with_filler(hs, case)
    except hs.HsError:
        pytest.skip("the expression's automaton alone is too large here")
    data, off, ln, ends = _collider_blocks(case)
    got = ref.scan_sorted(db.ptr, data, off, ln)
    _check_collider(case, got[got["id"] == case["id"]], ends)
    assert not np.any(got["id"] != case["id"])


# ---- compile rules ---------------------------------------------------------------------------------------------

def test_which_sets_take_the_route(hs):
    lits, _ = _lits(20, 5)
    exprs = [_esc(l) for l in lits] + [rb"ab+c"]
    assert hs.compile_multi(exprs).info().runtime_impl == 2          # fits one automaton: as before
    assert hs.compile_multi([rb"ab+c", rb"x.y"]).info().runtime_impl == 2
    big, _ = _lits(1000, 6)
    exprs = [_esc(l) for l in big] + [rb"ab+c", rb"\d+\.\d\d", rb"x.y"]
    assert hs.compile_multi(exprs).info().runtime_impl == 0          # too large for one: split
    hs.set_build_option("mixed_rose", 1)
    assert hs.compile_multi([_esc(l) for l in lits] + [rb"ab+c"]).info().runtime_impl == 0
    assert hs.compile_multi([_esc(l) for l in lits]).info().runtime_impl == 1   # no regex: pure literal
    assert hs.compile_multi([rb"ab+c"]).info().runtime_impl == 2                # no literal: single outfix


def _error(hs, *args, **kw):
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi(*args, **kw)
    return e.value.message


def test_errors_stay_as_before(hs):
    big, _ = _lits(1000, 6)
    lits = [_esc(l) for l in big]
    # the regex half alone does not fit: today's set-level error, message and index unchanged
    huge = [rb"q[a-d]{300}z", rb"r[a-d]{300}z"]
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi(lits + huge)
    assert e.value.message == "Pattern set is too large: its character positions exceed the 512-state NFA model."
    assert e.value.expression < 1000   # where the one automaton overflowed, not where the engine half alone does
    # a set with a combination, and streaming mode, keep their errors
    msg = _error(hs, lits + [rb"ab+c", b"0 & 1000"], [0] * 1001 + [hs.HS_FLAG_COMBINATION], list(range(1002)))
    assert msg.startswith("Pattern set is too large")
    assert "block mode only" in _error(hs, lits + [rb"ab+c"], mode=hs.HS_MODE_STREAM)
    hs.set_build_option("mixed_rose", 1)
    assert "block mode only" in _error(hs, [b"abcd", rb"ab+c"], mode=hs.HS_MODE_STREAM)
    # combinations keep the single-outfix route even under mixed_rose=1
    assert hs.compile_multi([b"abcd", rb"ab+c", b"0 & 1"], [0, 0, hs.HS_FLAG_COMBINATION],
                            [0, 1, 2]).info().runtime_impl == 2
    assert "SINGLEMATCH" in _error(hs, [b"abcd", rb"ab+c"], [SINGLE, 0], [3, 3])


def test_host_postprocess_entries_refuse(hs):
    """as for single-outfix databases, the host-only entries have no program walk: refused, never wrong"""
    hs.set_build_option("mixed_rose", 1)
    db = MixedSet([b"abcd"], [0], [1], REGEX_SMALL).compile(hs)
    recs = np.zeros(2, dtype=hs.MATCH_DTYPE)
    with pytest.raises(hs.HsError):
        hs.postprocess_matches(db, recs)
    with pytest.raises(hs.HsError):
        hs.postprocess_blocks(db, recs, np.array([10], np.uint32))


# ---- tools/hsbench_b200.py on a mixed signature file -----------------------------------------------------------

def _cli():
    spec = importlib.util.spec_from_file_location("hsbench_b200", os.path.join(ROOT, "tools", "hsbench_b200.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    return cli


def _cli_inputs(tmp_path, cli):
    lits, _ = _lits(800, 9)
    sig = tmp_path / "sigs"
    sig.write_bytes(b"".join(b"%d:/%s/\n" % (i, l) for i, l in enumerate(lits)) +
                    b"900:/ab+c/\n901:/\\d+\\.\\d\\d/\n902:/x.y/s\n")
    blocks = _blocks(5, 300, max_len=200, plant=lits[:50] + [b"abbc", b"3.14", b"x\ny"], alphabet=b"abcdefxyz.0123\n ")
    path = str(tmp_path / "corpus.db")
    cli.write_corpus(path, [(i % 7, b) for i, b in enumerate(blocks)])
    return str(sig), path, blocks


# ---- the device ----------------------------------------------------------------------------------------------

def _device_all_entries(hs, ref, db, blocks, pitch=None):
    """hs_scan per block, scan_blocks, scan_blocks_collect, the counting path, a resident corpus with
    hs_b200_fetch_matches: each equals the reference per block"""
    want = _ref_per_block(ref, db, blocks)
    data, off, ln = _pack(blocks, pitch)
    scratch = hs.Scratch(db)
    assert _per_block(hs.scan_blocks(db, data, off, ln, scratch), len(blocks)) == want
    out = np.zeros(sum(map(len, want)) + 16, dtype=hs.MATCH_DTYPE)
    n = hs.scan_blocks_collect(db, data, off, ln, scratch, out)
    assert _per_block(out[:n], len(blocks)) == want
    assert hs.scan_blocks(db, data, off, ln, scratch, collect=False) == sum(map(len, want))
    corpus = hs.Corpus.upload(data, off, ln)
    assert _per_block(hs.scan_corpus(db, corpus, scratch), len(blocks)) == want
    corpus.free()
    for b in range(0, len(blocks), max(1, len(blocks) // 12)):
        rc, got = hs.scan(db, blocks[b], scratch)
        assert rc == 0 and sorted((to, i) for i, to in got) == want[b]
    scratch.free()
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("kind,engine", KIND_X_ENGINE)
def test_device_equals_reference(hs, ref, kind, engine):
    ms, db = _kind_set(hs, kind, engine)
    want = _device_all_entries(hs, ref, db, _kind_blocks(ms, 7, n=200))
    assert sum(map(len, want)) > 50


@pytest.mark.gpu
@pytest.mark.parametrize("dfa", [1, 0])
@pytest.mark.parametrize("route", [1, 0])
def test_device_report_rules_across_both_halves(hs, ref, dfa, route):
    ms = _rules_set()
    hs.set_build_option("regex_dfa", dfa)
    hs.set_build_option("mixed_rose", route)
    if not route:
        extra, _ = _lits(1000, 4, alphabet=b"EFGHIJKLMNOP")
        ms.lits = list(ms.lits) + extra
        ms.lflags = list(ms.lflags) + [0] * len(extra)
        ms.lids = list(ms.lids) + list(range(100, 100 + len(extra)))
    db = ms.compile(hs)
    _device_all_entries(hs, ref, db, _rules_blocks(3, 600) + [b"", b"z", b"dd", b"abbc", b"y"])


def _issue_set():
    """1 000 literals of 4-8 bytes with ab+c, \\d+\\.\\d\\d and x.y: too large for one automaton"""
    big, _ = _lits(1000, 6)
    return MixedSet(big, [0] * 1000, list(range(1000)), REGEX_SMALL)


@pytest.mark.gpu
def test_device_small_ring_overflows_both_sources(hs, ref):
    """a 16-record initial ring: literal and engine records both overflow it, and the rescan holds them all"""
    ms = _issue_set()
    db = ms.compile(hs)
    blocks = _blocks(21, 400, max_len=200, plant=list(ms.lits[:30]) + [b"abbbc", b"9.99", b"xqy"])
    hs.set_runtime_option("initial_ring", 16)
    try:
        want = _device_all_entries(hs, ref, db, blocks)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)
    flat = [i for g in want for _, i in g]
    assert sum(i < 1000 for i in flat) > 100 and sum(i >= 5000 for i in flat) > 100


@pytest.mark.gpu
def test_device_chunked_upload(hs, ref):
    """chunk_mb=1: the literal ranges run per upload chunk, the engine once the whole corpus is there"""
    ms = _issue_set()
    db = ms.compile(hs)
    blocks = _blocks(22, 3000, max_len=1500, plant=list(ms.lits[:30]) + [b"abbbc", b"9.99", b"xqy"])
    hs.set_runtime_option("chunk_mb", 1)
    try:
        want = _device_all_entries(hs, ref, db, blocks)
    finally:
        hs.set_runtime_option("chunk_mb", 128)
    assert sum(map(len, want)) > 1000


@pytest.mark.gpu
def test_device_callback_termination(hs, ref):
    """a callback that stops the scan: HS_SCAN_TERMINATED, and what was delivered is a prefix of the library's
    order (block, to, id) over both halves' records"""
    ms = _issue_set()
    db = ms.compile(hs)
    data = b" ".join([ms.lits[0], b"abbc", ms.lits[1], b"1.23 xzy", ms.lits[2], b"abc"])
    scratch = hs.Scratch(db)
    rc, full = hs.scan(db, data, scratch)
    assert rc == 0 and len(full) >= 7
    assert [(to, i) for i, to in full] == sorted((to, i) for i, to in full)
    assert sorted((to, i) for i, to in full) == [tuple(x) for x in _ref_per_block(ref, db, [data])[0]]
    for stop in (1, 2, 4):
        rc, got = hs.scan(db, data, scratch, stop_after=stop)
        assert rc == hs.HS_SCAN_TERMINATED and got == full[:stop]
    scratch.free()


@pytest.mark.gpu
def test_device_thousands_of_uniform_blocks(hs, ref):
    ms = _issue_set()
    db = ms.compile(hs)
    data, off, ln, _ = synth.block_corpus(4096, 1024, list(ms.lits), plant_per_kb=2.0, seed=3)
    blocks = [data[int(o):int(o) + int(n)].tobytes() for o, n in zip(off, ln)]
    want = _device_all_entries(hs, ref, db, blocks, pitch=1024)
    assert sum(map(len, want)) > 4096


@pytest.mark.gpu
def test_device_recorded_vectors_beside_literals(hs):
    for case in SAMPLE:
        try:
            db = _with_filler(hs, case)
        except hs.HsError:
            continue
        data, off, ln, ends = _collider_blocks(case)
        scratch = hs.Scratch(db)
        got = np.sort(hs.scan_blocks(db, data, off, ln, scratch), order=["block", "to", "id"])
        _check_collider(case, got, ends)
        scratch.free()


@pytest.mark.gpu
def test_hsbench_cli_runs_a_mixed_signature_file(hs, ref, tmp_path):
    cli = _cli()
    sig, corpus, blocks = _cli_inputs(tmp_path, cli)
    exprs, flags, ids = [], [], []
    for line in open(sig, "rb"):
        rid, pat, fl, ext = cli.parse_signature_line(line)
        exprs.append(pat)
        flags.append(fl)
        ids.append(rid)
    db = hs.compile_multi(exprs, flags, ids)
    assert db.info().runtime_impl == 0
    want = sum(map(len, _ref_per_block(ref, db, blocks)))
    out = io.StringIO()
    with redirect_stdout(out):
        rc = cli.main(["-e", sig, "-c", corpus, "-N", "-n", "2"])
    assert rc == 0, out.getvalue()
    assert int(re.search(r"Matches per iteration:\s+(\d+)", out.getvalue()).group(1)) == want and want > 100
