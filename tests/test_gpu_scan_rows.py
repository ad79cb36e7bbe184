"""Row scans (hs_b200_scan_rows_async): a column of rows already in device memory -- chars plus int64 offsets, the
Arrow large_string / torch jagged layout, every row at any byte -- packed and scanned on the device with no host
wait.  The delivered matches, through the device ordering and through finish + fetch, equal
hs_b200_scan_blocks_collect over the same rows from host memory and, per row, the unmodified reference runtime, for
every database shape the device scans.  Covers rows at every residue mod 16, empty rows, one row and none, a first
offset above 0, literals across row boundaries, a column at the very end of its allocation, engine runs that cut
long rows into segments, bad row tables, a ring overflow, the refusals and a pipeline on a torch stream.  Runs on
the H100 and, with numpy arrays as device memory, on the SIMT emulator."""
import ctypes as C
import os

import numpy as np
import pytest

from hyperscan_b200 import synth
from test_mixed_rose import REGEX_WIDE, _kind_set
from test_multi_outfix import KIND_GROUPS, RegexSet

EMU = os.environ.get("HSB200_EMU") == "1"

pytestmark = pytest.mark.gpu

CASELESS, SINGLE = 1, 8


# ---- device memory: torch CUDA tensors on the GPU, host arrays under the emulator ------------------------------------

def _dev(a):
    a = np.ascontiguousarray(a)
    if EMU:
        return a.copy()
    import torch
    return torch.from_numpy(a.copy()).cuda()


def _out(cap):
    if EMU:
        return np.zeros(cap * 16, dtype=np.uint8), np.zeros(1, dtype=np.uint64)
    import torch
    return (torch.empty(cap * 16, dtype=torch.uint8, device="cuda"),
            torch.zeros(1, dtype=torch.int64, device="cuda"))


def _sync():
    if not EMU:
        import torch
        torch.cuda.synchronize()


def _read(hs, out, cnt):
    _sync()
    o = out if EMU else out.cpu().numpy()
    c = int(cnt[0]) if EMU else int(cnt.cpu().numpy().view(np.uint64)[0])
    if c == hs.ORDER_RING_OVERFLOW:
        return None
    assert c * 16 <= o.size, "the test's output buffer is too small"
    return o.view(hs.MATCH_DTYPE)[:c].copy()


def _scratch(hs, db):
    """under the emulator a small ring, as the emulated shapes are: the ordering kernels' grids follow the ring's
    capacity"""
    if not EMU:
        return hs.Scratch(db)
    hs.set_runtime_option("initial_ring", 1 << 14)
    try:
        return hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)


# ---- columns ---------------------------------------------------------------------------------------------------------

def _column(seed, lengths, plant=(), alphabet=b"abcdefgh ", lead=0):
    """rows of the given lengths back to back after `lead` bytes, literals of `plant` written in; returns the chars,
    the nrows + 1 offsets (int64) and the rows"""
    rng = np.random.default_rng(seed)
    a = np.frombuffer(alphabet, dtype=np.uint8)
    rows = []
    for ln in lengths:
        d = bytearray(a[rng.integers(0, a.size, size=int(ln))].tobytes())
        for _ in range(3):
            if plant:
                lit = plant[int(rng.integers(0, len(plant)))]
                if len(lit) <= ln:
                    p = int(rng.integers(0, ln - len(lit) + 1))
                    d[p:p + len(lit)] = lit
        rows.append(bytes(d))
    head = a[rng.integers(0, a.size, size=lead)].tobytes()
    chars = np.frombuffer(head + b"".join(rows), dtype=np.uint8).copy()
    off = np.concatenate([[lead], lead + np.cumsum([len(r) for r in rows], dtype=np.int64)]).astype(np.int64)
    return chars, off, rows


def _host(hs, db, chars, off, scratch=None):
    """hs_b200_scan_blocks_collect over the same rows from host memory"""
    scratch = scratch or _scratch(hs, db)
    ln = np.diff(off).astype(np.uint32)
    out = np.zeros(max(1024, int(ln.sum())), dtype=hs.MATCH_DTYPE)
    n = hs.scan_blocks_collect(db, chars, off[:-1].astype(np.uint64), ln, scratch, out)
    return out[:n].copy()


def _rows(hs, db, scratch, d_chars, d_off, cap=1 << 16, stream=None):
    """one row pass and its device ordering, then finish + fetch: (ordered matches, finish rc, fetched matches)"""
    out, cnt = _out(cap)
    hs.scan_rows_async(db, d_chars, d_off, scratch, stream=stream)
    hs.order_matches_async(db, scratch, out, cnt, stream=stream)
    got = _read(hs, out, cnt)
    rc, _, _ = hs.scan_corpus_finish(scratch)
    fetched = hs.fetch_matches(db, scratch) if rc == hs.HS_SUCCESS else None
    return got, rc, fetched


def _check(hs, db, chars, off, ref=None, scratch=None):
    """both delivery routes of a row pass equal the host path (and, given ref, the reference per row)"""
    want = _host(hs, db, chars, off)
    scratch = scratch or _scratch(hs, db)
    got, rc, fetched = _rows(hs, db, scratch, _dev(chars), _dev(off))
    assert rc == hs.HS_SUCCESS
    assert got is not None and np.array_equal(got, want)
    assert np.array_equal(fetched, want)
    if ref is not None:
        ln = np.diff(off).astype(np.uint32)
        recs = ref.scan_sorted(db.ptr, chars, off[:-1].astype(np.uint64), ln)
        mine = sorted((int(r["block"]), int(r["to"]), int(r["id"])) for r in want)
        assert mine == sorted((int(r["block"]), int(r["to"]), int(r["id"])) for r in recs)
    return want


# ---- the database shapes ---------------------------------------------------------------------------------------------

LIT_SETS = {  # name: (count, min_len, options, AVX2 platform)
    "noodle": (1, 5, {}, False), "teddy8": (12, 3, {}, False), "fat_teddy": (64, 3, {}, True),
    "fdr_pair": (1000, 4, {}, False), "fdr_gram4": (400, 4, {"gram": 2}, False)}
OUTFIX_LITS = {"mcclellan8": 2, "mcclellan16": 3, "sheng": 4, "limex32": 5}   # build option outfix_engine
LIMEX = {"limex64": (40, 1), "limex128": (100, 2), "limex256": (200, 3), "limex512": (300, 5)}   # {n}, engine id
SHAPES = list(LIT_SETS) + list(OUTFIX_LITS) + list(LIMEX) + ["beside_outfix", "split"]


def _shape(hs, name):
    """(database, strings to plant, alphabet)"""
    if name in LIT_SETS:
        n, min_len, opts, avx2 = LIT_SETS[name]
        lits, flags, _ = synth.literal_set(n, min_len=min_len, max_len=8, caseless_frac=0.2, seed=5,
                                           alphabet=b"abcdefgh")
        ids = [i % max(1, n // 3) for i in range(n)]
        flags = [f | (SINGLE if ids[i] % 5 == 1 else 0) for i, f in enumerate(flags)]
        plat = C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0)) if avx2 else None
        for k, v in opts.items():
            hs.set_runtime_option(k, v)
        return hs.compile_lit_multi(lits, flags, ids, platform=plat), lits[:50], b"abcdefgh "
    if name in OUTFIX_LITS:
        lits = [b"abc", b"bcd"] if name == "sheng" else [b"abcd", b"bcad", b"dab", b"hgfe"]
        hs.set_build_option("outfix_engine", OUTFIX_LITS[name])
        try:
            db = hs.compile_lit_multi(lits, [0] * len(lits), list(range(len(lits))))
        finally:
            hs.set_build_option("outfix_engine", 0)
        assert db.info().runtime_impl == 2
        return db, lits, b"abcdefgh "
    if name in LIMEX:
        n, eid = LIMEX[name]
        hs.set_build_option("regex_dfa", 0)
        db = hs.compile_multi([b"q[a-d0-3]{%d}z" % n, rb"ab+c"], [0, 0], [1, 2])
        assert db.info().runtime_impl == 2 and db.info().engine_id == eid
        return db, [b"q" + b"a0b1" * (n // 4) + b"c3"[: n % 4] + b"z", b"abbbc"], b"abcd0123qz "
    if name == "beside_outfix":
        ms, db = _kind_set(hs, "fdr", "mcclellan8")
        return db, list(ms.lits[:40]) + [b"abbbc", b"12.345", b"xay"], b"abcdxyz.0123 qA"
    rs = RegexSet([r for g in KIND_GROUPS for r in g])
    db = rs.compile(hs)
    assert db.info().engine_count == len(KIND_GROUPS)
    plant = [b"q" + b"abcd" * 75 + b"z", b"r" + b"0123" * 75 + b"s", b"t" + b"30" * 100 + b"u",
             b"xba" + b"ab" * 5 + b"y", b"xYYz"]
    return db, plant, b"abcd0123xyz"


def _lengths(seed, n, max_len):
    rng = np.random.default_rng(seed)
    ln = rng.integers(0, max_len + 1, size=n)
    ln[::7] = 0
    return ln


@pytest.mark.parametrize("name", SHAPES)
def test_rows_equal_host_path_and_reference(hs, ref, name):
    try:
        db, plant, alpha = _shape(hs, name)
        long_ = name in ("limex512", "split", "limex256")
        chars, off, _ = _column(17, _lengths(3, 40, 700 if long_ else 160), plant, alpha, lead=3)
        want = _check(hs, db, chars, off, ref)
        assert want.size >= 3
        if not EMU:   # a larger column, against the host path
            chars, off, _ = _column(18, _lengths(4, 3000, 1200 if long_ else 400), plant, alpha, lead=11)
            assert _check(hs, db, chars, off).size > 100
    finally:
        hs.set_runtime_option("gram", 1)


# ---- layouts ---------------------------------------------------------------------------------------------------------

def _needle_db(hs):
    return hs.compile_lit_multi([b"needle", b"pin"], [0, CASELESS], [1, 2])


def test_every_residue_empty_rows_and_boundaries(hs):
    """rows starting at every residue mod 16, empty ones among them, the first offset above 0, chars_bytes equal to
    the last offset; a literal split across each row boundary is never matched"""
    db = _needle_db(hs)
    rows = []
    for i in range(48):
        ln = (i * 7) % 37
        body = bytearray(b"x" * ln)
        if ln >= 3:
            body[:3] = b"dle"                 # the row before ends with "nee"
            body[-3:] = b"nee"
        if ln >= 12 and i % 3 == 0:
            body[4:10] = b"needle"
        rows.append(bytes(body))
    lead = 5
    chars = np.frombuffer(b"abcde" + b"".join(rows), dtype=np.uint8).copy()
    off = np.concatenate([[lead], lead + np.cumsum([len(r) for r in rows])]).astype(np.int64)
    assert {int(o) % 16 for o in off[:-1]} == set(range(16))
    assert off[-1] == chars.size
    want = _check(hs, db, chars, off)
    assert want.size == sum(r.count(b"needle") for r in rows) > 0
    # one row, and none
    _check(hs, db, chars[7:30], np.array([0, 23], np.int64))
    scratch = _scratch(hs, db)
    got, rc, fetched = _rows(hs, db, scratch, _dev(np.zeros(1, np.uint8)[:0]), _dev(np.zeros(1, np.int64)))
    assert rc == hs.HS_SUCCESS and got.size == 0 and fetched.size == 0


def test_column_at_the_end_of_its_allocation(hs):
    """the column is the tail of its buffer and the bytes in front of it would match: nothing outside
    [chars, chars + chars_bytes) takes part (and, under the emulator's sanitizer build, is read)"""
    db = _needle_db(hs)
    rows = [b"dle x", b"", b"needle", b"pi", b"n", b"xxneedlexxPIN"]
    body = b"".join(rows)
    front = b"needlepinneedlenee"
    whole = np.frombuffer(front + body, dtype=np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    if EMU:
        buf = np.empty(whole.size, dtype=np.uint8)           # an allocation of its own, ending with the column
        buf[:] = whole
        d_chars = buf[len(front):]
    else:
        import torch
        buf = torch.from_numpy(whole).cuda()
        d_chars = buf[len(front):]
    want = _host(hs, db, np.frombuffer(body, np.uint8).copy(), off)
    assert want.size == 3
    scratch = _scratch(hs, db)
    got, rc, fetched = _rows(hs, db, scratch, d_chars, _dev(off))
    assert rc == hs.HS_SUCCESS and np.array_equal(got, want) and np.array_equal(fetched, want)


# ---- engine segments -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("engine", ["limex128", "mcclellan16"])
def test_long_rows_cut_into_segments(hs, engine):
    if engine == "limex128":
        db, plant, alpha = _shape(hs, "limex128")
    else:
        hs.set_build_option("regex_dfa", 1)
        db = hs.compile_multi([r[0] for r in REGEX_WIDE], [r[1] for r in REGEX_WIDE], [r[2] for r in REGEX_WIDE])
        assert db.info().engine_id == 7
        plant, alpha = [b"aababbabaabc", b"q0123Z", b"Q33z"], b"abcq0123zZ "
    big = 20000 if EMU else 3 << 20
    rng = np.random.default_rng(5)
    chars, off, _ = _column(9, [big, 100, big + 7, big // 2 + 3], alphabet=alpha, lead=1)
    for p in rng.integers(0, chars.size - 500, size=300 if EMU else 3000):   # plants across the whole column
        lit = plant[int(p) % len(plant)]
        chars[int(p):int(p) + len(lit)] = np.frombuffer(lit, np.uint8)
    want = _host(hs, db, chars, off)
    assert want.size > 50
    scratch = _scratch(hs, db)
    before = scratch.segment_stats()
    got, rc, fetched = _rows(hs, db, scratch, _dev(chars), _dev(off), cap=want.size + 64)
    assert rc == hs.HS_SUCCESS and np.array_equal(got, want) and np.array_equal(fetched, want)
    after = scratch.segment_stats()
    assert after["runs"] > before["runs"] and after["segments"] > before["segments"] + 4
    hs.set_runtime_option("engine_segment", -1)
    try:
        got1, rc, _ = _rows(hs, db, scratch, _dev(chars), _dev(off), cap=want.size + 64)
    finally:
        hs.set_runtime_option("engine_segment", 0)
    assert rc == hs.HS_SUCCESS and np.array_equal(got1, want)
    assert scratch.segment_stats()["runs"] == after["runs"]


# ---- protocols -------------------------------------------------------------------------------------------------------

def test_bad_tables_fail_the_pass(hs):
    db = _needle_db(hs)
    chars, off, _ = _column(3, [20, 0, 33, 17, 40], [b"needle", b"PIN"], lead=2)
    want = _host(hs, db, chars, off)
    assert want.size > 0
    scratch = _scratch(hs, db)
    for bad in (1, 2):
        o = off.copy()
        if bad == 1:
            o[3] = o[2] - 1                          # decreasing
        else:
            o[-1] = chars.size + 1                   # ends past chars_bytes
        got, rc, _ = _rows(hs, db, scratch, _dev(chars), _dev(o))
        assert got is None and rc == hs.HS_INVALID
        got, rc, fetched = _rows(hs, db, scratch, _dev(chars), _dev(off))
        assert rc == hs.HS_SUCCESS and np.array_equal(got, want) and np.array_equal(fetched, want)


def test_ring_overflow_and_the_pass_again(hs):
    hs.set_runtime_option("initial_ring", 16)
    try:
        db = _needle_db(hs)
        scratch = hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)
    chars, off, _ = _column(4, [64] * 12, [b"needle", b"pin"], lead=9)
    want = _host(hs, db, chars, off)
    assert want.size > 16
    d_chars, d_off = _dev(chars), _dev(off)
    got, rc, _ = _rows(hs, db, scratch, d_chars, d_off)
    assert got is None and rc == hs.HS_INSUFFICIENT_SPACE
    got, rc, fetched = _rows(hs, db, scratch, d_chars, d_off)
    assert rc == hs.HS_SUCCESS and np.array_equal(got, want) and np.array_equal(fetched, want)


def test_refusals(hs):
    L = hs.lib()
    db = _needle_db(hs)
    scratch = _scratch(hs, db)
    chars, off, _ = _column(2, [10, 20], [b"needle"])
    d_chars, d_off = _dev(chars), _dev(off)
    pc, po = C.c_void_p(hs._dev_ptr(d_chars)), C.c_void_p(hs._dev_ptr(d_off))

    def call(db_=db, c=pc, nbytes=chars.size, o=po, n=2, s=scratch):
        return L.hs_b200_scan_rows_async(db_.ptr if db_ is not None else None, c, nbytes, o, n,
                                         s.ptr if s is not None else None, None)

    assert call(db_=None) == hs.HS_INVALID
    assert call(s=None) == hs.HS_INVALID
    assert call(o=None) == hs.HS_INVALID
    assert call(c=None) == hs.HS_INVALID
    assert call(o=C.c_void_p(po.value + 4)) == hs.HS_INVALID
    assert call(n=0xfffffff1) == hs.HS_INVALID
    other = hs.compile_lit_multi([b"abc"], [0], [0])
    assert call(db_=other) == hs.HS_INVALID                          # no image of it in the scratch
    comb = hs.compile_multi([b"abc", b"def", b"1&2"], [0, 0, hs.HS_FLAG_COMBINATION], [1, 2, 3])
    assert call(db_=comb, s=_scratch(hs, comb)) == hs.HS_INVALID
    stream_db = hs.compile_lit_multi([b"abc"], [0], [0], mode=hs.HS_MODE_STREAM)
    assert call(db_=stream_db, s=_scratch(hs, stream_db)) == hs.HS_DB_MODE_ERROR
    peer, _ = _out(64)
    bases = (C.c_void_p * 1)(hs._dev_ptr(peer))
    assert L.hs_b200_set_peer_exchange(scratch.ptr, 1, 0, bases, 3, 0) == hs.HS_SUCCESS
    assert call() == hs.HS_ARCH_ERROR
    assert L.hs_b200_set_peer_exchange(scratch.ptr, 0, 0, None, 0, 0) == hs.HS_SUCCESS
    got, rc, _ = _rows(hs, db, scratch, d_chars, d_off)
    assert rc == hs.HS_SUCCESS and np.array_equal(got, _host(hs, db, chars, off))


def test_torch_stream_pipeline_without_host_waits(hs, real_gpu):
    """offsets made by a kernel on a torch stream, the pass and its ordering behind it on that stream; the host
    waits once, for the ordered matches"""
    import torch
    db = _needle_db(hs)
    scratch = _scratch(hs, db)
    lens = _lengths(8, 20000, 300)
    chars, off, _ = _column(12, lens, [b"needle", b"Pin"])
    want = _host(hs, db, chars, off)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_chars = torch.from_numpy(chars).to("cuda", non_blocking=True)
        d_lens = torch.from_numpy(lens.astype(np.int64)).to("cuda", non_blocking=True)
        d_off = torch.zeros(lens.size + 1, dtype=torch.int64, device="cuda")
        d_off[1:] = torch.cumsum(d_lens, 0)
        out = torch.empty((want.size + 64) * 16, dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        hs.scan_rows_async(db, d_chars, d_off, scratch, stream=s.cuda_stream)
        hs.order_matches_async(db, scratch, out, cnt, stream=s.cuda_stream)
        n_host = cnt.to("cpu", non_blocking=True)
        o_host = out.to("cpu", non_blocking=True)
    s.synchronize()
    n = int(n_host.numpy().view(np.uint64)[0])
    assert n == want.size
    assert np.array_equal(o_host.numpy().view(hs.MATCH_DTYPE)[:n], want)
    assert hs.scan_corpus_finish(scratch)[0] == hs.HS_SUCCESS
