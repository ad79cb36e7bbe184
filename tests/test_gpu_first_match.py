"""First-match passes (hs_b200_scan_corpus_first_async / hs_b200_scan_rows_first_async).  Entry b of the table is
(to << 32) | id of the first match block b delivers in (block, to, id) order, ~0 when it delivers none: the table
equals the first match per block of an ordinary pass (fetched and ordered on the device), the smallest (to, id) per
block of the reference runtime's matches, and the mask pass's "does block b match", for every database shape and
first stage the device runs.  Covers the report rules (dedupe, single-match, min_offset / max_offset / min_length,
ties at one offset, end-of-data accepts), the engine walks' early stops (dense blocks, literals beside an outfix,
several engines, segmented runs), empty and short blocks, a column at the end of its allocation, a table pre-filled
with another value, the status word after a candidate-list overflow and a bad row table, a dense column that overflows
the record ring on the ordinary pass, the refusals, and what the record readers serve after a first pass.  They run
on the H100 and, with numpy arrays as device memory, on the SIMT emulator; every first-match instantiation of the
engine kernel that test_gpu_engine_variants reaches for records is reached here too."""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_engine_variants import (FUSED, LENS, NFA_TYPE, SEGS, _db_lens, _fused_plant, _opts, _pack,
                                      _planted_blocks, _single_outfix_db)
from test_gpu_engine_variants import _scratch as _walk_scratch
from test_gpu_scan_rows import (SHAPES, _column, _dev, _lengths, _needle_db, _out, _read, _scratch, _shape,
                                _sync)
from test_mixed_rose import _kind_set
from test_multi_outfix import KIND_GROUPS, RegexSet

pytestmark = pytest.mark.gpu

EMU = os.environ.get("HSB200_EMU") == "1"
NONE = 0xFFFFFFFFFFFFFFFF
CASELESS, MULTILINE, SINGLE = 1, 4, 8


# ---- tables ----------------------------------------------------------------------------------------------------------

def _first_of(recs, nblocks):
    """the smallest (to, id) per block of a list of matches, as table entries"""
    t = np.full(nblocks, NONE, np.uint64)
    for r in recs:
        b, key = int(r["block"]), (int(r["to"]) << 32) | int(r["id"])
        if key < int(t[b]):
            t[b] = key
    return t


def _host_u64(x):
    _sync()
    a = x if EMU else x.cpu().numpy()
    return np.ascontiguousarray(a).view(np.uint64)


def _host_u32(x):
    _sync()
    a = x if EMU else x.cpu().numpy()
    return np.ascontiguousarray(a).view(np.uint32)


def _first_buf(n):
    """a table pre-filled with a value that is not ~0 (every entry must be written) and a status word that is not 0"""
    return _dev(np.full(n, 0x0000000300000005, np.int64)), _dev(np.full(1, 7, np.int32))


def _rows_first(hs, db, scratch, d_chars, d_off, nrows):
    """one row first-match pass, then finish: (table, status, finish rc)"""
    first, status = _first_buf(nrows)
    hs.scan_rows_first_async(db, d_chars, d_off, scratch, first, status)
    t, st = _host_u64(first).copy(), int(_host_u32(status)[0])
    rc, n, _ = hs.scan_corpus_finish(scratch)
    if rc == hs.HS_SUCCESS:
        assert n == 0                       # no record was written
    return t, st, rc


def _corpus_first(hs, db, scratch, chars, off):
    corpus = hs.Corpus.upload(chars, off[:-1].astype(np.uint64), np.diff(off).astype(np.uint32))
    first, status = _first_buf(off.size - 1)
    hs.scan_corpus_first_async(db, corpus, scratch, first, status)
    t, st = _host_u64(first).copy(), int(_host_u32(status)[0])
    rc, n, _ = hs.scan_corpus_finish(scratch)
    corpus.free()
    return t, st, rc


def _ordinary(hs, db, scratch, d_chars, d_off, nrows, cap=1 << 16):
    """the first match per row of an ordinary pass: fetched, and ordered on the device.  (Under the emulator, where
    one device ordering costs about a second, the fetched matches alone: test_gpu_device_order checks there that the
    ordering equals them.)"""
    hs.scan_rows_async(db, d_chars, d_off, scratch)
    if not EMU:
        out, cnt = _out(cap)
        hs.order_matches_async(db, scratch, out, cnt)
        ordered = _read(hs, out, cnt)
    rc, _, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS
    fetched = hs.fetch_matches(db, scratch)
    if not EMU:
        assert ordered is not None and np.array_equal(fetched, ordered)
    return _first_of(fetched, nrows)


def _mask_rows(hs, db, scratch, d_chars, d_off, nrows):
    """which rows match anything, from the mask pass"""
    wpb = max(1, (hs.report_ids(db).size + 31) // 32)
    mask = _dev(np.full((nrows, wpb), -1, np.int32))
    hs.scan_rows_mask_async(db, d_chars, d_off, scratch, mask, wpb)
    m = _host_u32(mask).reshape(nrows, wpb).copy()
    rc, _, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS
    return m.any(axis=1)


def _check(hs, db, chars, off, ref=None, scratch=None):
    """the row and corpus first-match passes equal the ordinary pass's first matches, the mask pass's matching rows
    and, given ref, the reference's smallest (to, id) per block; returns the table"""
    nrows = off.size - 1
    scratch = scratch or _scratch(hs, db)
    d_chars, d_off = _dev(chars), _dev(off)
    want = _ordinary(hs, db, scratch, d_chars, d_off, nrows)
    if ref is not None:
        recs = ref.scan_sorted(db.ptr, chars, off[:-1].astype(np.uint64), np.diff(off).astype(np.uint32))
        assert np.array_equal(_first_of(recs, nrows), want)
    assert np.array_equal(_mask_rows(hs, db, scratch, d_chars, d_off, nrows), want != NONE)
    got, st, rc = _rows_first(hs, db, scratch, d_chars, d_off, nrows)
    assert rc == hs.HS_SUCCESS and st == 0
    assert np.array_equal(got, want)
    got, st, rc = _corpus_first(hs, db, scratch, chars, off)
    assert rc == hs.HS_SUCCESS and st == 0
    assert np.array_equal(got, want)
    return want


def _rows_of(rows):
    chars = np.frombuffer(b"".join(rows), np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return chars, off


def _entry(to, rid):
    return (to << 32) | rid


# ---- parity: every shape and first stage -----------------------------------------------------------------------------

@pytest.mark.parametrize("name", SHAPES)
def test_first_equals_reference_ordinary_and_mask(hs, ref, name):
    try:
        db, plant, alpha = _shape(hs, name)
        long_ = name in ("limex512", "split", "limex256")
        chars, off, _ = _column(23, _lengths(7, 40, 700 if long_ else 160), plant, alpha, lead=5)
        want = _check(hs, db, chars, off, ref)
        assert (want != NONE).any() and (want == NONE).any()
    finally:
        hs.set_runtime_option("gram", 1)


# ---- report rules ----------------------------------------------------------------------------------------------------

def _rules_db(hs, case):
    if case == "shared_id":      # three literals of id 5 end at one offset (dedupe), beside id 7
        return hs.compile_lit_multi([b"abcd", b"bcd", b"cd", b"zz"], [0, 0, 0, 0], [5, 5, 5, 7])
    if case == "single":
        return hs.compile_lit_multi([b"ab", b"ba", b"xyz"], [SINGLE, 0, SINGLE], [3, 4, 2])
    if case == "min_offset":     # the first raw matches lie before offset 20
        return hs.compile_ext_multi([rb"ab+c", rb"needle"], [0, 0], [1, 2], [{"min_offset": 20}, {"min_offset": 12}])
    if case == "max_min_length":
        return hs.compile_ext_multi([rb"x[0-9]+y", rb"q[a-c]*z", rb"pin"], [0, 0, 0], [1, 2, 3],
                                    [{"max_offset": 30}, {"min_length": 6}, {"max_offset": 9}])
    if case == "tie":            # several ids end at one offset: the smallest wins
        return hs.compile_multi([rb"ab+c", rb"b+c", rb"[a-c]c", rb"abbc"], [0, 0, 0, 0], [9, 4, 6, 2])
    return hs.compile_multi([rb"xyz$", rb"z\z", rb"[a-z]yz", rb"qq"], [0, 0, 0, 0], [3, 1, 5, 7])


RULE_ROWS = {
    "shared_id": [b"abcdzz", b"zzabcd", b"xxbcdx", b"cd", b"", b"zabcdabcd"],
    "single": [b"abababxyzxyz", b"babab", b"xyzab", b"b", b"xyab"],
    "min_offset": [b"abcneedle" + b"-" * 20 + b"abbbc", b"needle" * 5, b"abc" * 10, b"-" * 11 + b"needle",
                   b"ac" * 20],
    "max_min_length": [b"x1y" * 12, b"qz qabcz qaz", b"pin pin pin", b"-" * 29 + b"x12y", b"qabcabcz"],
    "tie": [b"xabbc", b"bc", b"abcabbc", b"cc", b"aaaa"],
    "end": [b"xyz", b"axyz", b"zz", b"xyzxyz", b"xyzq", b"qqxyz", b"ayz", b"", b"xyz\n", b"axyz\n", b"xyzxyz\n"],
}


@pytest.mark.parametrize("case", list(RULE_ROWS))
def test_report_rules(hs, ref, case):
    db = _rules_db(hs, case)
    chars, off = _rows_of(RULE_ROWS[case])
    want = _check(hs, db, chars, off, ref)
    if case == "tie":
        assert int(want[0]) == _entry(5, 2) and int(want[1]) == _entry(2, 4)
    if case == "end":
        # "xyz": xyz$ (3), z\z (1) and [a-z]yz (5) all end at 3: id 1 wins; "ayz": [a-z]yz and z\z tie at 3
        assert int(want[0]) == _entry(3, 1) and int(want[6]) == _entry(3, 1) and int(want[4]) == _entry(3, 5)
        # "xyz\n": xyz$ reports at 3, one byte before its raw end, and wins the tie with [a-z]yz (5)
        assert int(want[8]) == _entry(3, 3) and int(want[9]) == _entry(4, 3)
    if case == "min_offset":
        # row 0: "abc" (3) and "needle" (9) end before their bounds, "abbbc" at 34 is the first that passes
        assert [int(v) for v in want[[0, 1, 3]]] == [_entry(34, 1), _entry(12, 2), _entry(17, 2)]


# An engine report one byte back (offset_adjust -1: a trailing \b, `$` before a final newline, multiline `$`) ties
# with the report of the byte before it: a lane that has reported must walk on until no later byte can reach its
# entry.  The prefixes put the tie at every position of a 16-byte piece, in the last partial piece, and across a
# 128-byte tile.
ADJUSTED = {"word_boundary": (rb"ab+c\b", 0, [b"abbc x", b"abc", b"abbbc-"]),
            "dollar_newline": (rb"ab+c$", 0, [b"abc\n", b"abbc"]),
            "multiline_dollar": (rb"ab+c$", MULTILINE, [b"q abc\nq", b"abc\n", b"abbc"])}


@pytest.mark.parametrize("dfa", [1, 0])
@pytest.mark.parametrize("case", list(ADJUSTED))
def test_ties_with_reports_one_byte_back(hs, ref, case, dfa):
    pat, flags, base = ADJUSTED[case]
    hs.set_build_option("regex_dfa", dfa)
    db = hs.compile_multi([rb"ab+c", pat], [0, flags], [2, 1])
    rows = [b"-" * k + r for r in base for k in list(range(0, 21)) + list(range(120, 131))]
    chars, off = _rows_of(rows)
    want = _check(hs, db, chars, off, ref)
    assert all(int(v) & 0xFFFFFFFF == 1 for v in want)   # the smaller id wins every tie


# ---- early stops -----------------------------------------------------------------------------------------------------

def test_dense_blocks_many_matches_after_the_first(hs, ref):
    hs.set_build_option("regex_dfa", 1)
    db = hs.compile_multi([rb"[0-9]+", rb"ab+c", rb"[a-d]{3}9"], [0, 0, 0], [4, 2, 1])
    chars, off, _ = _column(31, _lengths(8, 48, 300), [b"abbc", b"cab9", b"77"], b"abcd0123456789 ", lead=3)
    want = _check(hs, db, chars, off, ref)
    assert (want != NONE).sum() > 30


def test_literals_beside_an_outfix(hs, ref):
    """a §10d set: in some rows a literal comes before the engine's first match, in others after it"""
    ms, db = _kind_set(hs, "fdr", "mcclellan8")
    lit = bytes(ms.lits[0])
    rows = [lit + b"..abbbc", b"abbbc.." + lit, b"12.345" + lit, lit, b"xay", b"..." + lit + b"12.345" + lit]
    chars, off = _rows_of(rows + [r[::-1] for r in rows])
    _check(hs, db, chars, off, ref)


def test_several_engines_report_in_different_orders(hs, ref):
    db = RegexSet([r for g in KIND_GROUPS for r in g]).compile(hs)
    q, r, t = b"q" + b"abcd" * 75 + b"z", b"r" + b"0123" * 75 + b"s", b"t" + b"30" * 100 + b"u"
    x = b"xba" + b"ab" * 5 + b"y"
    rows = [q + r + t, t + r + q, r + x + q, x + t, b"xYYz" + q, q[:-1] + b"xyz", b"abcd" * 30]
    chars, off = _rows_of(rows)
    want = _check(hs, db, chars, off, ref)
    assert [int(v) & 0xFFFFFFFF for v in want[:4]] == [1, 4, 2, 3]


def test_long_rows_cut_into_segments(hs):
    """a segmented engine run gives the table of an unsegmented one"""
    db, plant, alpha = _shape(hs, "limex128")
    big = 20000 if EMU else 3 << 20
    rng = np.random.default_rng(6)
    chars, off, _ = _column(9, [big, 100, big + 7] + [60] * 40 + [big // 2 + 3], alphabet=alpha, lead=1)
    for p in rng.integers(big // 2, chars.size - 500, size=200):   # the long rows' first halves stay empty
        lit = plant[int(p) % len(plant)]
        chars[int(p):int(p) + len(lit)] = np.frombuffer(lit, np.uint8)
    scratch = _scratch(hs, db)
    before = scratch.segment_stats()
    want = _check(hs, db, chars, off, scratch=scratch)
    assert (want != NONE).any() and scratch.segment_stats()["runs"] > before["runs"]
    hs.set_runtime_option("engine_segment", -1)
    try:
        runs = scratch.segment_stats()["runs"]
        t, st, rc = _rows_first(hs, db, scratch, _dev(chars), _dev(off), off.size - 1)
        assert scratch.segment_stats()["runs"] == runs
    finally:
        hs.set_runtime_option("engine_segment", 0)
    assert rc == hs.HS_SUCCESS and st == 0 and np.array_equal(t, want)


# Every first-match walk of the engine kernel, on the databases and blocks test_gpu_engine_variants runs: one block
# per lane and segmented (engine_segment=16 / 64) for every engine kind, and fused launches of several engines.

def _check_walks(hs, ref, db, blocks, seg_modes):
    data, off, ln = _pack(blocks, "ragged", 3)
    want = _first_of(ref.scan_sorted(db.ptr, data, off, ln), len(blocks))
    assert (want != NONE).sum() >= 10
    corpus = hs.Corpus.upload(data, off, ln)
    try:
        for seg in [-1] + seg_modes:
            scratch = _walk_scratch(hs, db, 1, seg)
            with _opts(hs, engine_segment=seg):
                runs = scratch.segment_stats()["runs"]
                first, status = _first_buf(len(blocks))
                hs.scan_corpus_first_async(db, corpus, scratch, first, status)
                t, st = _host_u64(first).copy(), int(_host_u32(status)[0])
                rc, n, _ = hs.scan_corpus_finish(scratch)
                assert rc == hs.HS_SUCCESS and st == 0 and n == 0, seg
                assert np.array_equal(t, want), seg
                if seg != -1:
                    assert scratch.segment_stats()["runs"] > runs, seg
            scratch.free()
    finally:
        corpus.free()


@pytest.mark.parametrize("name", list(NFA_TYPE))
def test_single_outfix_every_walk(hs, ref, name):
    db, plant, alpha = _single_outfix_db(hs, name)
    assert db.info().engine_id == NFA_TYPE[name]
    long_ = 1200 if EMU else 5000
    _check_walks(hs, ref, db, _planted_blocks(11, _db_lens(long_, 70 if EMU else 400), plant, alpha), SEGS)


@pytest.mark.parametrize("which", list(FUSED))
def test_fused_every_walk(hs, ref, which):
    groups, dfa, _ = FUSED[which]
    hs.set_build_option("regex_dfa", dfa)
    db = RegexSet([r for g in groups for r in g]).compile(hs)
    plant = _fused_plant(groups)
    lens = [600, 520, 300] + [LENS[i % len(LENS)] for i in range(30 if EMU else 130)]
    blocks = _planted_blocks(12, lens, plant, b"abcd0123qrstuvwxyz") + [b" " + p + b" " for p in plant]
    _check_walks(hs, ref, db, blocks, [])


# ---- layouts ---------------------------------------------------------------------------------------------------------

def test_empty_short_and_narrow_blocks(hs, ref):
    db = hs.compile_lit_multi([b"needle", b"pin", b"haystacks"], [0, CASELESS, 0], [1, 2, 3])
    rows = [b"", b"n", b"pin", b"PIN", b"", b"needle", b"xneedlex", b"xx", b"pi", b"needlepinneedle", b""]
    rows += [b"needle"[: k % 7] + b"pin"[: k % 4] for k in range(1, 18)]
    chars, off = _rows_of(rows)
    assert (_check(hs, db, chars, off, ref) != NONE).any()
    scratch = _scratch(hs, db)   # no rows at all, and rows with no bytes
    t, st, rc = _rows_first(hs, db, scratch, _dev(np.zeros(1, np.uint8)[:0]), _dev(np.zeros(1, np.int64)), 0)
    assert rc == hs.HS_SUCCESS and st == 0 and t.size == 0
    t, st, rc = _rows_first(hs, db, scratch, _dev(np.zeros(1, np.uint8)[:0]), _dev(np.zeros(4, np.int64)), 3)
    assert rc == hs.HS_SUCCESS and st == 0 and (t == NONE).all()


def test_column_at_the_end_of_its_allocation(hs):
    db = _needle_db(hs)
    rows = [b"dle x", b"", b"needle", b"pi", b"n", b"xxneedlexxPIN"]
    body = b"".join(rows)
    front = b"needlepinneedlenee"
    whole = np.frombuffer(front + body, dtype=np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    if EMU:
        buf = np.empty(whole.size, dtype=np.uint8)
        buf[:] = whole
    else:
        import torch
        buf = torch.from_numpy(whole).cuda()
    t, st, rc = _rows_first(hs, db, _scratch(hs, db), buf[len(front):], _dev(off), len(rows))
    assert rc == hs.HS_SUCCESS and st == 0
    assert [int(v) for v in t] == [NONE, NONE, _entry(6, 1), NONE, NONE, _entry(8, 1)]


# ---- status and overflow ---------------------------------------------------------------------------------------------

def test_candidate_overflow_then_the_pass_again(hs):
    hs.set_runtime_option("initial_ring", 16)
    try:
        db = _needle_db(hs)
        scratch = hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)
    chars, off, _ = _column(4, [64] * 12, [b"needle", b"pin"], lead=9)
    d_chars, d_off = _dev(chars), _dev(off)
    t, st, rc = _rows_first(hs, db, scratch, d_chars, d_off, 12)
    assert rc == hs.HS_INSUFFICIENT_SPACE and st != 0
    t, st, rc = _rows_first(hs, db, scratch, d_chars, d_off, 12)
    assert rc == hs.HS_SUCCESS and st == 0
    assert np.array_equal(t, _ordinary(hs, db, scratch, d_chars, d_off, 12))


def test_bad_row_table_then_the_pass_again(hs):
    db = _needle_db(hs)
    chars, off, _ = _column(3, [20, 0, 33, 17, 40], [b"needle", b"PIN"], lead=2)
    scratch = _scratch(hs, db)
    want = _ordinary(hs, db, scratch, _dev(chars), _dev(off), 5)
    assert (want != NONE).any()
    o = off.copy()
    o[3] = o[2] - 1
    t, st, rc = _rows_first(hs, db, scratch, _dev(chars), _dev(o), 5)
    assert rc == hs.HS_INVALID and st != 0
    t, st, rc = _rows_first(hs, db, scratch, _dev(chars), _dev(off), 5)
    assert rc == hs.HS_SUCCESS and st == 0 and np.array_equal(t, want)


def test_dense_column_needs_no_rescan(hs):
    """[0-9]+ fires at every digit: the ordinary pass overflows the record ring, the first pass is right at once"""
    hs.set_build_option("regex_dfa", 1)
    db = hs.compile_multi([rb"[0-9]+", rb"abc"], [0, 0], [1, 2])
    scratch = _scratch(hs, db)
    nrows, ln = (64, 600) if EMU else (4096, 600)
    chars, off, rows = _column(7, [ln] * nrows, alphabet=b"0123456789 ")
    d_chars, d_off = _dev(chars), _dev(off)
    t, st, rc = _rows_first(hs, db, scratch, d_chars, d_off, nrows)
    assert rc == hs.HS_SUCCESS and st == 0
    hs.scan_rows_async(db, d_chars, d_off, scratch)
    rc, n, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_INSUFFICIENT_SPACE and n > 16000
    assert np.array_equal(t, _ordinary(hs, db, scratch, d_chars, d_off, nrows, cap=1 << 22))
    want = [_entry(next(i for i, c in enumerate(r) if c != 0x20) + 1, 1) for r in rows]
    assert [int(v) for v in t] == want


# ---- protocols -------------------------------------------------------------------------------------------------------

def test_record_readers_after_a_first_pass(hs):
    """after a first-match pass, fetch, the device ordering and the export have no records to serve"""
    db = _needle_db(hs)
    scratch = _scratch(hs, db)
    chars, off, _ = _column(3, [40] * 8, [b"needle", b"pin"])
    d_chars, d_off = _dev(chars), _dev(off)
    assert (_ordinary(hs, db, scratch, d_chars, d_off, 8) != NONE).any()
    first, status = _first_buf(8)
    hs.scan_rows_first_async(db, d_chars, d_off, scratch, first, status)
    out, cnt = _out(64)
    hs.order_matches_async(db, scratch, out, cnt)
    got = _read(hs, out, cnt)
    assert got is not None and got.size == 0
    exp_out, exp_cnt = _out(64)
    assert hs.lib().hs_b200_export_records_async(scratch.ptr, C.c_void_p(hs._dev_ptr(exp_out)), 64,
                                                 C.c_void_p(hs._dev_ptr(exp_cnt)), None) == hs.HS_SUCCESS
    _sync()
    assert int((exp_cnt if EMU else exp_cnt.cpu().numpy()).view(np.uint64)[0]) == 0
    rc, n, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS and n == 0
    assert hs.fetch_matches(db, scratch).size == 0
    assert (_host_u64(first) != NONE).any()


def test_refusals(hs):
    L = hs.lib()
    db = _needle_db(hs)
    scratch = _scratch(hs, db)
    chars, off, _ = _column(2, [10, 20], [b"needle"])
    d_chars, d_off = _dev(chars), _dev(off)
    first, status = _first_buf(3)
    pc, po = C.c_void_p(hs._dev_ptr(d_chars)), C.c_void_p(hs._dev_ptr(d_off))
    pf, ps = C.c_void_p(hs._dev_ptr(first)), C.c_void_p(hs._dev_ptr(status))
    corpus = hs.Corpus.upload(chars, off[:-1].astype(np.uint64), np.diff(off).astype(np.uint32))

    def rows(db_=db, s=scratch, f=pf, st=ps):
        return L.hs_b200_scan_rows_first_async(db_.ptr if db_ is not None else None, pc, chars.size, po, 2,
                                               s.ptr if s is not None else None, f, st, None)

    def corp(db_=db, s=scratch, f=pf, st=ps, c=corpus):
        return L.hs_b200_scan_corpus_first_async(db_.ptr if db_ is not None else None, c.ptr if c else None,
                                                 s.ptr if s is not None else None, f, st, None)

    for call in (rows, corp):
        assert call(db_=None) == hs.HS_INVALID
        assert call(s=None) == hs.HS_INVALID
        assert call(f=None) == hs.HS_INVALID                                  # (NULL only without blocks)
        assert call(f=C.c_void_p(pf.value + 4)) == hs.HS_INVALID              # 8-byte entries
        assert call(st=C.c_void_p(ps.value + 1)) == hs.HS_INVALID
        other = hs.compile_lit_multi([b"abc"], [0], [0])
        assert call(db_=other) == hs.HS_INVALID                               # no image of it in the scratch
        comb = hs.compile_multi([b"abc", b"def", b"1&2"], [0, 0, hs.HS_FLAG_COMBINATION], [1, 2, 3])
        assert call(db_=comb, s=_scratch(hs, comb)) == hs.HS_INVALID
        stream_db = hs.compile_lit_multi([b"abc"], [0], [0], mode=hs.HS_MODE_STREAM)
        assert call(db_=stream_db, s=_scratch(hs, stream_db)) == hs.HS_DB_MODE_ERROR
    assert corp(c=None) == hs.HS_INVALID
    peer, _ = _out(64)
    bases = (C.c_void_p * 1)(hs._dev_ptr(peer))
    assert L.hs_b200_set_peer_exchange(scratch.ptr, 1, 0, bases, 3, 0) == hs.HS_SUCCESS
    assert rows() == hs.HS_ARCH_ERROR and corp() == hs.HS_ARCH_ERROR
    assert L.hs_b200_set_peer_exchange(scratch.ptr, 0, 0, None, 0, 0) == hs.HS_SUCCESS
    t, st, rc = _rows_first(hs, db, scratch, d_chars, d_off, 2)
    assert rc == hs.HS_SUCCESS and st == 0
    assert [int(v) & 0xFFFFFFFF for v in t] == [1, 1]
    corpus.free()
