"""Match masks (hs_b200_scan_corpus_mask_async / hs_b200_scan_rows_mask_async) and the id table behind their columns
(hs_b200_report_ids).  A mask pass sets bit r of row b iff block b delivers a match with id report_ids(db)[r]: the
mask equals the one built from the reference runtime's matches per block and the one derived from the delivered
matches of an ordinary pass, for every database shape and first stage the device runs.  Covers several words per
block and spare words, empty and short blocks, a column at the end of its allocation, engine runs cut into segments,
a buffer pre-filled with ones, the status word after a candidate-list overflow and a bad row table, a dense workload
that overflows the record ring, the refusals, and what the record readers serve after a mask pass.  The tests marked
gpu run on the H100 and, with numpy arrays as device memory, on the SIMT emulator; report_ids needs no device."""
import ctypes as C
import os

import numpy as np
import pytest

from hyperscan_b200 import synth
from test_gpu_scan_rows import (SHAPES, _column, _dev, _lengths, _needle_db, _out, _read, _scratch, _shape,
                                _sync)
from test_mixed_rose import _kind_set
from test_multi_outfix import KIND_GROUPS, RegexSet

EMU = os.environ.get("HSB200_EMU") == "1"

CASELESS, SINGLE, QUIET, UTF8, PREFILTER = 1, 8, 1024, 32, 128


# ---- masks -----------------------------------------------------------------------------------------------------------

def _mask_of(ids, recs, nblocks, wpb):
    """the mask a list of (block, id) matches makes"""
    rank = {int(v): i for i, v in enumerate(ids)}
    m = np.zeros((nblocks, wpb), np.uint32)
    for r in recs:
        i = rank[int(r["id"])]
        m[int(r["block"]), i // 32] |= np.uint32(1 << (i % 32))
    return m


def _host_arr(x):
    _sync()
    a = x if EMU else x.cpu().numpy()
    return np.ascontiguousarray(a).view(np.uint32)


def _mask_buf(nblocks, wpb):
    """a mask buffer pre-filled with ones (the pass must write every word) and a status word that is not 0"""
    return (_dev(np.full((nblocks, wpb), -1, np.int32)), _dev(np.full(1, 7, np.int32)))


def _rows_mask(hs, db, scratch, d_chars, d_off, nrows, wpb):
    """one row mask pass, then finish: (mask, status, finish rc)"""
    mask, status = _mask_buf(nrows, wpb)
    hs.scan_rows_mask_async(db, d_chars, d_off, scratch, mask, wpb, status)
    m, st = _host_arr(mask).reshape(nrows, wpb), int(_host_arr(status)[0])
    rc, n, _ = hs.scan_corpus_finish(scratch)
    if rc == hs.HS_SUCCESS:
        assert n == 0                       # no record was written
    return m, st, rc


def _corpus_mask(hs, db, scratch, data, off, ln, wpb):
    corpus = hs.Corpus.upload(data, off, ln)
    mask, status = _mask_buf(ln.size, wpb)
    hs.scan_corpus_mask_async(db, corpus, scratch, mask, wpb, status)
    m, st = _host_arr(mask).reshape(ln.size, wpb), int(_host_arr(status)[0])
    rc, n, _ = hs.scan_corpus_finish(scratch)
    corpus.free()
    return m, st, rc


def _ordinary(hs, db, scratch, d_chars, d_off):
    hs.scan_rows_async(db, d_chars, d_off, scratch)
    rc, _, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS
    return hs.fetch_matches(db, scratch)


def _check(hs, db, chars, off, ref=None, spare=1, scratch=None):
    """the row and corpus mask passes equal the mask of the ordinary pass's delivered matches and, given ref, the
    reference's per block; returns that mask"""
    ids = hs.report_ids(db)
    nrows = off.size - 1
    wpb = (ids.size + 31) // 32 + spare
    scratch = scratch or _scratch(hs, db)
    d_chars, d_off = _dev(chars), _dev(off)
    want = _mask_of(ids, _ordinary(hs, db, scratch, d_chars, d_off), nrows, wpb)
    if ref is not None:
        ln = np.diff(off).astype(np.uint32)
        recs = ref.scan_sorted(db.ptr, chars, off[:-1].astype(np.uint64), ln)
        assert np.array_equal(_mask_of(ids, recs, nrows, wpb), want)
    got, st, rc = _rows_mask(hs, db, scratch, d_chars, d_off, nrows, wpb)
    assert rc == hs.HS_SUCCESS and st == 0
    assert np.array_equal(got, want)
    ln = np.diff(off).astype(np.uint32)
    got, st, rc = _corpus_mask(hs, db, scratch, chars, off[:-1].astype(np.uint64), ln, wpb)
    assert rc == hs.HS_SUCCESS and st == 0
    assert np.array_equal(got, want)
    return want


# ---- report ids: host only ---------------------------------------------------------------------------------------------

def _ref_ids(ref, db, blocks):
    data = b"".join(blocks)
    ln = np.array([len(b) for b in blocks], np.uint32)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    recs = ref.scan_sorted(db.ptr, np.frombuffer(data, np.uint8).copy(), off, ln)
    return sorted({int(r["id"]) for r in recs})


REGEXES = [(rb"ab+c", 0, 7), (rb"x[0-9]{3}y", CASELESS, 9), (rb"q[a-d]{5}z", 0, 7)]


def _id_cases(hs):
    """(name, database, blocks that fire every id it can deliver, the ids)"""
    lits = [b"needle", b"haystack", b"pin", b"thread"]
    yield "literal", hs.compile_lit_multi(lits, [0, SINGLE, CASELESS, 0], [3, 1, 3, 40]), lits, [1, 3, 40]
    hs.set_build_option("outfix_engine", 2)
    try:
        db = hs.compile_lit_multi([b"abcd", b"bcad", b"dab"], [0, 0, 0], [5, 6, 5])
    finally:
        hs.set_build_option("outfix_engine", 0)
    yield "outfix", db, [b"abcd", b"bcad", b"dab"], [5, 6]
    ms, db = _kind_set(hs, "fdr", "mcclellan8")
    yield "beside_outfix", db, [bytes(x) for x in ms.lits] + [b"abbbc", b"12.345", b"xay"], None
    db = RegexSet([r for g in KIND_GROUPS for r in g]).compile(hs)
    yield "outfixes", db, [b"q" + b"abcd" * 75 + b"z", b"r" + b"0123" * 75 + b"s", b"t" + b"30" * 100 + b"u",
                           b"xba" + b"ab" * 5 + b"y", b"xYYz"], [1, 2, 3, 4, 5]
    db = hs.compile_ext_multi([r[0] for r in REGEXES] + [rb"zz[0-9]+", rb"quiet"],
                              [r[1] for r in REGEXES] + [SINGLE, QUIET], [r[2] for r in REGEXES] + [11, 12],
                              [None, {"min_offset": 4}, None, {"max_offset": 100}, None])
    yield "ext_single_quiet", db, [b"xxabbc", b"__x123y", b"qabcdz", b"zz12", b"quiet"], [7, 9, 11]


def test_report_ids_are_the_ids_the_reference_delivers(hs, ref):
    for name, db, blocks, ids in _id_cases(hs):
        got = hs.report_ids(db)
        assert got.dtype == np.uint32 and np.all(np.diff(got.astype(np.int64)) > 0), name
        assert list(got) == _ref_ids(ref, db, blocks), name
        if ids is not None:
            assert list(got) == ids, name


def test_report_ids_of_combinations_and_refusals(hs):
    comb = hs.compile_multi([b"abc", b"def", b"1&2"], [QUIET, 0, hs.HS_FLAG_COMBINATION], [1, 2, 3])
    assert list(hs.report_ids(comb)) == [2, 3]   # the quiet sub-expression delivers nothing
    L = hs.lib()
    db = hs.compile_lit_multi([b"abc", b"abd"], [0, 0], [4, 2])
    n = C.c_size_t()
    assert L.hs_b200_report_ids(None, None, 0, C.byref(n)) == hs.HS_INVALID
    assert L.hs_b200_report_ids(db.ptr, None, 0, None) == hs.HS_INVALID
    assert L.hs_b200_report_ids(db.ptr, None, 2, C.byref(n)) == hs.HS_INVALID
    bad = (C.c_ubyte * 64)()
    assert L.hs_b200_report_ids(C.addressof(bad), None, 0, C.byref(n)) == hs.HS_INVALID
    one = np.zeros(1, np.uint32)
    assert L.hs_b200_report_ids(db.ptr, one.ctypes.data, 1, C.byref(n)) == hs.HS_INSUFFICIENT_SPACE
    assert n.value == 2 and one[0] == 0
    stream_db = hs.compile_lit_multi([b"abc"], [0], [9], mode=hs.HS_MODE_STREAM)
    assert list(hs.report_ids(stream_db)) == [9]


# ---- parity: every shape and first stage -------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", SHAPES)
def test_mask_equals_reference_and_ordinary_pass(hs, ref, name):
    try:
        db, plant, alpha = _shape(hs, name)
        long_ = name in ("limex512", "split", "limex256")
        chars, off, _ = _column(21, _lengths(6, 40, 700 if long_ else 160), plant, alpha, lead=5)
        want = _check(hs, db, chars, off, ref)
        assert want.any()
    finally:
        hs.set_runtime_option("gram", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["bounds", "utf8", "prefilter"])
def test_bounds_utf8_and_prefilter(hs, ref, case):
    if case == "bounds":
        # min_offset / max_offset clear bits the raw engine and the literal would set
        db = hs.compile_ext_multi([rb"ab+c", rb"x[0-9]{3}y", rb"needle", rb"pin"], [0, 0, 0, 0], [1, 2, 3, 4],
                                  [{"min_offset": 20}, {"max_offset": 30}, None, {"min_offset": 12}])
        plant, alpha = [b"abbbc", b"x123y", b"needle", b"pin"], b"abcxy0123 "
    elif case == "utf8":
        db = hs.compile_multi(["café+".encode(), "ü[a-z]ß".encode(), rb"pl[a-c]in"],
                              [UTF8, UTF8, UTF8 | CASELESS], [1, 2, 3])
        plant, alpha = ["caféé".encode(), "übß".encode(), b"PLaIN"], b"abcdefz "
    else:
        db = hs.compile_multi([rb"(a|b)c\1d", rb"(?=x)xy+z", rb"q(?>ab|a)c"], [PREFILTER] * 3, [1, 2, 3])
        plant, alpha = [b"acad", b"bcbd", b"xyyz", b"qabc"], b"abcdxyzq "
    chars, off, _ = _column(8, _lengths(2, 50, 60), plant, alpha, lead=1)
    assert _check(hs, db, chars, off, ref).any()


@pytest.mark.gpu
def test_many_ids_several_words_and_spare_words(hs, ref):
    """70 ids: three words per block, and two spare words that the pass zeroes"""
    lits, flags, _ = synth.literal_set(140, min_len=4, max_len=8, seed=3, alphabet=b"abcdefgh")
    ids = [1000 + 7 * (i % 70) for i in range(len(lits))]   # each id twice
    db = hs.compile_lit_multi(lits, flags, ids)
    assert hs.report_ids(db).size == 70
    chars, off, _ = _column(4, _lengths(9, 30, 400), lits, b"abcdefgh ")
    want = _check(hs, db, chars, off, ref, spare=2)
    assert want[:, 2].any() and not want[:, 3:].any()


# ---- layouts ---------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_empty_and_short_blocks(hs, ref):
    db = _needle_db(hs)
    rows = [b"", b"n", b"pin", b"PIN", b"", b"needle", b"xneedlex", b"xx", b"pi", b"needlepinneedle", b""]
    rows += [b"needle"[: k % 7] + b"pin"[: k % 4] for k in range(1, 18)]
    chars = np.frombuffer(b"".join(rows), np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    assert _check(hs, db, chars, off, ref).any()
    scratch = _scratch(hs, db)   # no rows at all, and blocks with no bytes
    m, st, rc = _rows_mask(hs, db, scratch, _dev(np.zeros(1, np.uint8)[:0]), _dev(np.zeros(1, np.int64)), 0, 1)
    assert rc == hs.HS_SUCCESS and st == 0 and m.size == 0
    m, st, rc = _rows_mask(hs, db, scratch, _dev(np.zeros(1, np.uint8)[:0]), _dev(np.zeros(4, np.int64)), 3, 2)
    assert rc == hs.HS_SUCCESS and st == 0 and not m.any()


@pytest.mark.gpu
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
    d_chars = buf[len(front):]
    scratch = _scratch(hs, db)
    m, st, rc = _rows_mask(hs, db, scratch, d_chars, _dev(off), len(rows), 1)
    assert rc == hs.HS_SUCCESS and st == 0
    assert [int(x) for x in m[:, 0]] == [0, 0, 1, 0, 0, 3]   # ids 1, 2 are ranks 0, 1


@pytest.mark.gpu
def test_long_rows_cut_into_segments(hs):
    """a segmented engine run sets the same bits as an unsegmented one"""
    db, plant, alpha = _shape(hs, "limex128")
    big = 20000 if EMU else 3 << 20
    n = 40
    rng = np.random.default_rng(5)
    chars, off, _ = _column(9, [big, 100, big + 7] + [60] * n + [big // 2 + 3], alphabet=alpha, lead=1)
    for p in rng.integers(0, chars.size - 500, size=200):
        lit = plant[int(p) % len(plant)]
        chars[int(p):int(p) + len(lit)] = np.frombuffer(lit, np.uint8)
    scratch = _scratch(hs, db)
    before = scratch.segment_stats()
    want = _check(hs, db, chars, off, scratch=scratch)
    assert want.any() and scratch.segment_stats()["runs"] > before["runs"]
    hs.set_runtime_option("engine_segment", -1)
    try:
        runs = scratch.segment_stats()["runs"]
        m, st, rc = _rows_mask(hs, db, scratch, _dev(chars), _dev(off), off.size - 1, want.shape[1])
        assert scratch.segment_stats()["runs"] == runs
    finally:
        hs.set_runtime_option("engine_segment", 0)
    assert rc == hs.HS_SUCCESS and st == 0 and np.array_equal(m, want)


# ---- status and overflow -----------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_candidate_overflow_then_the_pass_again(hs):
    hs.set_runtime_option("initial_ring", 16)
    try:
        db = _needle_db(hs)
        scratch = hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)
    chars, off, _ = _column(4, [64] * 12, [b"needle", b"pin"], lead=9)
    d_chars, d_off = _dev(chars), _dev(off)
    m, st, rc = _rows_mask(hs, db, scratch, d_chars, d_off, 12, 1)
    assert rc == hs.HS_INSUFFICIENT_SPACE and st != 0
    m, st, rc = _rows_mask(hs, db, scratch, d_chars, d_off, 12, 1)
    assert rc == hs.HS_SUCCESS and st == 0
    assert np.array_equal(m, _mask_of(hs.report_ids(db), _ordinary(hs, db, scratch, d_chars, d_off), 12, 1))


@pytest.mark.gpu
def test_bad_row_table_then_the_pass_again(hs):
    db = _needle_db(hs)
    chars, off, _ = _column(3, [20, 0, 33, 17, 40], [b"needle", b"PIN"], lead=2)
    scratch = _scratch(hs, db)
    want = _mask_of(hs.report_ids(db), _ordinary(hs, db, scratch, _dev(chars), _dev(off)), 5, 1)
    assert want.any()
    o = off.copy()
    o[3] = o[2] - 1
    m, st, rc = _rows_mask(hs, db, scratch, _dev(chars), _dev(o), 5, 1)
    assert rc == hs.HS_INVALID and st != 0
    m, st, rc = _rows_mask(hs, db, scratch, _dev(chars), _dev(off), 5, 1)
    assert rc == hs.HS_SUCCESS and st == 0 and np.array_equal(m, want)


@pytest.mark.gpu
def test_dense_workload_needs_no_rescan(hs):
    """[0-9]+ fires at every digit: the ordinary pass overflows the record ring, the mask pass does not"""
    hs.set_build_option("regex_dfa", 1)
    db = hs.compile_multi([rb"[0-9]+", rb"abc"], [0, 0], [1, 2])
    scratch = _scratch(hs, db)
    nrows, ln = (64, 600) if EMU else (4096, 600)
    chars, off, _ = _column(7, [ln] * nrows, alphabet=b"0123456789 ")
    d_chars, d_off = _dev(chars), _dev(off)
    m, st, rc = _rows_mask(hs, db, scratch, d_chars, d_off, nrows, 1)
    assert rc == hs.HS_SUCCESS and st == 0
    hs.scan_rows_async(db, d_chars, d_off, scratch)
    rc, n, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_INSUFFICIENT_SPACE and n > 16000
    assert np.array_equal(m, _mask_of(hs.report_ids(db), _ordinary(hs, db, scratch, d_chars, d_off), nrows, 1))
    assert (m[:, 0] == 1).all()


# ---- protocols -------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_record_readers_after_a_mask_pass(hs):
    """after a mask pass, fetch, the device ordering and the export have no records to serve"""
    db = _needle_db(hs)
    scratch = _scratch(hs, db)
    chars, off, _ = _column(3, [40] * 8, [b"needle", b"pin"])
    d_chars, d_off = _dev(chars), _dev(off)
    assert _ordinary(hs, db, scratch, d_chars, d_off).size > 0
    mask, status = _mask_buf(8, 1)
    hs.scan_rows_mask_async(db, d_chars, d_off, scratch, mask, 1, status)
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
    assert _host_arr(mask).any()


@pytest.mark.gpu
def test_refusals(hs):
    L = hs.lib()
    db = _needle_db(hs)
    scratch = _scratch(hs, db)
    chars, off, _ = _column(2, [10, 20], [b"needle"])
    d_chars, d_off = _dev(chars), _dev(off)
    mask, status = _mask_buf(2, 2)
    pc, po = C.c_void_p(hs._dev_ptr(d_chars)), C.c_void_p(hs._dev_ptr(d_off))
    pm, ps = C.c_void_p(hs._dev_ptr(mask)), C.c_void_p(hs._dev_ptr(status))
    corpus = hs.Corpus.upload(chars, off[:-1].astype(np.uint64), np.diff(off).astype(np.uint32))

    def rows(db_=db, s=scratch, m=pm, w=1, st=ps):
        return L.hs_b200_scan_rows_mask_async(db_.ptr if db_ is not None else None, pc, chars.size, po, 2,
                                              s.ptr if s is not None else None, m, w, st, None)

    def corp(db_=db, s=scratch, m=pm, w=1, st=ps, c=corpus):
        return L.hs_b200_scan_corpus_mask_async(db_.ptr if db_ is not None else None, c.ptr if c else None,
                                                s.ptr if s is not None else None, m, w, st, None)

    for call in (rows, corp):
        assert call(db_=None) == hs.HS_INVALID
        assert call(s=None) == hs.HS_INVALID
        assert call(m=None) == hs.HS_INVALID                                  # (NULL only without blocks)
        assert call(m=C.c_void_p(pm.value + 2)) == hs.HS_INVALID
        assert call(st=C.c_void_p(ps.value + 1)) == hs.HS_INVALID
        assert call(w=0) == hs.HS_INVALID                                     # below ceil(2 / 32)
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
    m, st, rc = _rows_mask(hs, db, scratch, d_chars, d_off, 2, 1)
    assert rc == hs.HS_SUCCESS and st == 0 and int(m[0, 0]) == 1 and int(m[1, 0]) == 1
    corpus.free()
