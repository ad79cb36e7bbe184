"""The report rules on the device (hs_b200_order_matches_async / hs_b200_order_records_async): the matches
ordered, deduplicated and resolved by kernels into device memory equal, record for record and in count, what
the host delivers for the same scan (hs_b200_fetch_matches, hs_b200_postprocess_matches) -- for every database
shape the device scans, at the edges of the output capacity, after a ring overflow, for raw records of several
scans and for sort keys wider than 64 bits.  Runs on the H100 and, smaller, on the SIMT emulator."""
import ctypes as C
import os

import numpy as np
import pytest

from hyperscan_b200 import synth
from test_mixed_rose import ENGINES, _kind_blocks, _kind_set, _pack, _rules_blocks, _rules_set

EMU = os.environ.get("HSB200_EMU") == "1"

pytestmark = pytest.mark.gpu

SINGLE, CASELESS = 8, 1


# ---- device buffers: torch CUDA tensors on the GPU, host arrays under the emulator --------------------------------

def _alloc(n):
    if EMU:
        return np.zeros(max(n, 1) * 16, dtype=np.uint8), np.zeros(1, dtype=np.uint64)
    import torch
    return (torch.empty(max(n, 1) * 16, dtype=torch.uint8, device="cuda"),
            torch.zeros(1, dtype=torch.int64, device="cuda"))


def _to_dev(recs):
    recs = np.ascontiguousarray(recs, dtype=None).view(np.uint8)
    if EMU:
        return recs.copy()
    import torch
    return torch.from_numpy(recs.copy()).cuda()


def _sync():
    if not EMU:
        import torch
        torch.cuda.synchronize()


def _read(hs, out, cnt, cap):
    _sync()
    o = out if EMU else out.cpu().numpy()
    c = int(cnt[0]) if EMU else int(cnt.cpu().numpy().view(np.uint64)[0])
    recs = o.view(hs.MATCH_DTYPE)[: min(c, cap)].copy() if c != hs.ORDER_RING_OVERFLOW else None
    return recs, c


def _order_last(hs, db, scratch, cap=None, stream=None):
    """the device ordering of the last scan, into a buffer of `cap` records (default: room for all)"""
    if cap is None:
        cap = int(scratch_records(hs, scratch)) + 64
    out, cnt = _alloc(cap)
    hs.order_matches_async(db, scratch, out, cnt, stream=stream, cap=cap)
    return _read(hs, out, cnt, cap)


def _order_raw(hs, db, scratch, recs, cap=None):
    recs = np.ascontiguousarray(recs, dtype=hs.MATCH_DTYPE)
    cap = recs.size * 4 + 64 if cap is None else cap
    out, cnt = _alloc(cap)
    d = _to_dev(recs)
    hs.order_records_async(db, scratch, d, recs.size, out, cnt, cap=cap)
    return _read(hs, out, cnt, cap)


def scratch_records(hs, scratch):
    return scratch.counters()[0]


def _scan(hs, db, scratch, corpus):
    for _ in range(3):
        hs.scan_corpus_async(db, corpus, scratch)
        rc, n, _ = hs.scan_corpus_finish(scratch)
        if rc == hs.HS_INSUFFICIENT_SPACE:
            continue
        assert rc == hs.HS_SUCCESS
        return n
    raise AssertionError("ring kept overflowing")


def _raw(hs, scratch, n):
    """the raw records of the last scan, through the stream-ordered export"""
    out, cnt = _alloc(n + 1)
    C_ = hs.lib()
    rc = C_.hs_b200_export_records_async(scratch.ptr, C.c_void_p(hs._dev_ptr(out)), n, C.c_void_p(hs._dev_ptr(cnt)),
                                         None)
    assert rc == hs.HS_SUCCESS
    _sync()
    o = out if EMU else out.cpu().numpy()
    return o.view(hs.MATCH_DTYPE)[:n].copy()


def _check_scan(hs, db, blocks_or_corpus, pitch=None):
    """scan, then the device delivery equals fetch_matches; returns the matches"""
    if isinstance(blocks_or_corpus, tuple):
        data, off, ln = blocks_or_corpus
    else:
        data, off, ln = _pack(blocks_or_corpus, pitch)
    scratch = hs.Scratch(db)
    corpus = hs.Corpus.upload(data, off, ln)
    _scan(hs, db, scratch, corpus)
    want = hs.fetch_matches(db, scratch)
    got, n = _order_last(hs, db, scratch)
    assert n == want.size
    assert np.array_equal(got, want)
    return want, scratch, corpus


def _ragged(blocks):
    """blocks at 16-byte aligned, unequal offsets"""
    off, pos = [], 0
    for b in blocks:
        off.append(pos)
        pos += (len(b) + 15) // 16 * 16 + 16
    data = np.zeros(pos + 16, dtype=np.uint8)
    for o, b in zip(off, blocks):
        data[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return data, np.array(off, np.uint64), np.array([len(b) for b in blocks], np.uint32)


# ---- pure literal ---------------------------------------------------------------------------------------------------

LIT_SETS = {  # name: (count, min_len, options, AVX2 platform)
    "noodle": (1, 5, {}, False), "teddy8": (12, 3, {}, False), "fat_teddy": (64, 3, {}, True),
    "fdr1000": (1000, 4, {}, False), "gram4": (400, 4, {"gram": 2}, False)}


@pytest.mark.parametrize("name", list(LIT_SETS))
def test_pure_literal_equals_fetch(hs, name):
    n, min_len, opts, avx2 = LIT_SETS[name]
    lits, flags, _ = synth.literal_set(n, min_len=min_len, max_len=8, caseless_frac=0.2, seed=5,
                                       alphabet=b"abcdefgh")
    ids = [i % max(1, n // 3) for i in range(n)]                  # ids shared by several literals
    flags = [f | (SINGLE if ids[i] % 5 == 1 else 0) for i, f in enumerate(flags)]
    plat = C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0)) if avx2 else None
    for k, v in opts.items():
        hs.set_runtime_option(k, v)
    try:
        db = hs.compile_lit_multi(lits, flags, ids, platform=plat)
        rng = np.random.default_rng(3)
        nb = 24 if EMU else 400
        blocks = []
        for b in range(nb):
            ln = 0 if b % 9 == 0 else int(rng.integers(1, 200))
            d = bytearray(rng.choice(np.frombuffer(b"abcdefgh ", np.uint8), size=ln).tobytes())
            for _ in range(3):
                lit = lits[int(rng.integers(0, n))]
                if len(lit) <= ln:
                    p = int(rng.integers(0, ln - len(lit) + 1))
                    d[p:p + len(lit)] = lit.upper() if rng.random() < 0.3 else lit
            blocks.append(bytes(d))
        want, _, _ = _check_scan(hs, db, blocks)
        assert want.size > 20
        _check_scan(hs, db, _ragged(blocks))
    finally:
        hs.set_runtime_option("gram", 1)


# ---- single outfix and literals beside an outfix --------------------------------------------------------------------

@pytest.mark.parametrize("engine", list(ENGINES))
def test_single_outfix_equals_fetch(hs, engine):
    ms = _rules_set()
    regexes, dfa = ENGINES[engine]
    hs.set_build_option("regex_dfa", dfa)
    exprs = [r[0] for r in regexes + ms.regexes] if engine != "limex512" else [r[0] for r in regexes]
    flags = [r[1] for r in regexes + ms.regexes] if engine != "limex512" else [r[1] for r in regexes]
    ids = [r[2] for r in regexes + ms.regexes] if engine != "limex512" else [r[2] for r in regexes]
    ext = [r[3] for r in regexes + ms.regexes] if engine != "limex512" else [r[3] for r in regexes]
    db = hs.compile_ext_multi(exprs, flags, ids, ext)
    assert db.info().runtime_impl == 2
    blocks = _rules_blocks(3, n=16 if EMU else 60) + [b"", b"z", b"dd", b"abbc", b"y", b"ab" * 8 + b"c"]
    if engine == "limex512":
        blocks += [b"xx q" + b"a0" * 135 + b"z abbc"]
    want, _, _ = _check_scan(hs, db, blocks)
    assert want.size > 5


@pytest.mark.parametrize("kind", ["noodle", "teddy", "fdr"])
def test_literals_beside_outfix_equals_fetch(hs, kind):
    ms, db = _kind_set(hs, kind, "mcclellan8")
    blocks = _kind_blocks(ms, 7, n=10 if EMU else 60)
    want, _, _ = _check_scan(hs, db, blocks)
    assert want.size > 5


@pytest.mark.parametrize("route", [1, 0])
def test_rules_across_both_halves(hs, route):
    """shared ids, a SINGLEMATCH id across both halves, bounds, $ \\z \\b; mixed_rose=1 or the 1 000-literal split"""
    ms = _rules_set()
    if route:
        hs.set_build_option("mixed_rose", 1)
    else:
        extra, _, _ = synth.literal_set(1000, min_len=4, max_len=8, seed=4, alphabet=b"EFGHIJKLMNOP")
        ms.lits = list(ms.lits) + extra
        ms.lflags = list(ms.lflags) + [0] * len(extra)
        ms.lids = list(ms.lids) + list(range(100, 100 + len(extra)))
    db = ms.compile(hs)
    assert db.info().runtime_impl == 0
    blocks = _rules_blocks(3, n=16 if EMU else 80) + [b"", b"z", b"dd", b"abbc", b"y"]
    want, _, _ = _check_scan(hs, db, blocks)
    assert (want["id"] == 9).sum() >= 1


# ---- edges ----------------------------------------------------------------------------------------------------------

def _small_db(hs):
    return hs.compile_lit_multi([b"abc", b"bcd", b"cd"], [0, SINGLE, CASELESS], [3, 1, 3])


def test_no_matches_and_short_blocks(hs):
    db = _small_db(hs)
    want, _, _ = _check_scan(hs, db, [b"xyz" * 5, b"", b"c", b"zz"])
    assert want.size == 0
    hs.set_build_option("mixed_rose", 1)
    ms, db2 = _kind_set(hs, "noodle", "mcclellan8")
    _check_scan(hs, db2, [b"", b"a", b"ab", b"xyz"])


def test_capacity_zero_and_short(hs):
    db = _small_db(hs)
    blocks = [b"abcd cd abcd CD" * 3] * 6
    want, scratch, _ = _check_scan(hs, db, blocks)
    got, n = _order_last(hs, db, scratch, cap=0)
    assert n == want.size and got.size == 0
    out, cnt = _alloc(0)
    hs.order_matches_async(db, scratch, None, cnt, cap=0)
    assert _read(hs, out, cnt, 0)[1] == want.size
    got, n = _order_last(hs, db, scratch, cap=7)
    assert n == want.size and np.array_equal(got, want[:7])


def test_uniform_corpus(hs):
    db = _small_db(hs)
    _check_scan(hs, db, [b"xxabcdxx" * 4, b"cdcdcd", b"ABCD" * 8, b""] * 4, pitch=64)


def test_ring_overflow_then_rescan(hs):
    hs.set_runtime_option("initial_ring", 16)
    try:
        db = _small_db(hs)
        data, off, ln = _pack([b"abcd cd " * 8] * 8)
        scratch = hs.Scratch(db)
        corpus = hs.Corpus.upload(data, off, ln)
        hs.scan_corpus_async(db, corpus, scratch)
        out, cnt = _alloc(64)
        hs.order_matches_async(db, scratch, out, cnt, cap=64)
        _, n = _read(hs, out, cnt, 64)
        assert n == hs.ORDER_RING_OVERFLOW
        assert hs.scan_corpus_finish(scratch)[0] == hs.HS_INSUFFICIENT_SPACE
        _scan(hs, db, scratch, corpus)
        want = hs.fetch_matches(db, scratch)
        got, n = _order_last(hs, db, scratch)
        assert n == want.size and np.array_equal(got, want)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)


# ---- raw records ----------------------------------------------------------------------------------------------------

def test_raw_exported_shuffled(hs):
    db = _small_db(hs)
    blocks = [b"abcd cd abCD xx" * 4] * 10
    want, scratch, _ = _check_scan(hs, db, blocks)
    raw = _raw(hs, scratch, scratch_records(hs, scratch))
    np.random.default_rng(1).shuffle(raw)
    got, n = _order_raw(hs, db, scratch, raw)
    assert n == want.size and np.array_equal(got, want)


def test_raw_gather_pure_literal(hs):
    db = _small_db(hs)
    scratch = hs.Scratch(db)
    parts = []
    for seed, blocks in enumerate([[b"abcd cd " * 4] * 5, [b"xx cd abc bcd" * 3] * 7]):
        data, off, ln = _pack(blocks)
        corpus = hs.Corpus.upload(data, off, ln)
        n = _scan(hs, db, scratch, corpus)
        r = _raw(hs, scratch, n)
        if seed:
            r["block"] += 5                                     # the second rank's blocks follow the first's
        parts.append(r)
    both = np.concatenate(parts)
    want = hs.postprocess_matches(db, both)
    got, n = _order_raw(hs, db, scratch, both)
    assert n == want.size and np.array_equal(got, want)


def test_raw_gather_regex(hs):
    ms = _rules_set()
    hs.set_build_option("mixed_rose", 1)
    db = ms.compile(hs)
    scratch = hs.Scratch(db)
    raws, fetched = [], []
    nb = 0
    for seed in (3, 4):
        data, off, ln = _pack(_rules_blocks(seed, n=12 if EMU else 40))
        corpus = hs.Corpus.upload(data, off, ln)
        n = _scan(hs, db, scratch, corpus)
        r, f = _raw(hs, scratch, n), hs.fetch_matches(db, scratch)
        keep = r["id"] != 0xffffffff
        r["block"][keep] += nb
        f["block"] += nb
        raws.append(r)
        fetched.append(f)
        nb += ln.size
    want = np.concatenate(fetched)
    got, n = _order_raw(hs, db, scratch, np.concatenate(raws))
    assert n == want.size and np.array_equal(got, want)


def test_raw_wide_keys(hs):
    """block indices near 2^32 and end offsets near 2^32: a key of 32 + 33 + rank bits"""
    db = _small_db(hs)
    scratch = hs.Scratch(db)
    rng = np.random.default_rng(9)
    n = 3000 if EMU else 200000
    recs = np.zeros(n, dtype=hs.MATCH_DTYPE)
    recs["id"] = rng.choice([1, 3], size=n)
    recs["block"] = (2 ** 32 - 1) - rng.integers(0, 40, size=n)
    recs["to"] = 2 ** 32 - rng.integers(0, 50, size=n)
    recs[::7]["to"] = rng.integers(0, 30, size=recs[::7].size)
    want = hs.postprocess_matches(db, recs)
    got, m = _order_raw(hs, db, scratch, recs)
    assert m == want.size and np.array_equal(got, want)


# ---- stream order and refusals --------------------------------------------------------------------------------------

def test_stream_order_without_host_sync(hs, real_gpu):
    import torch
    db = _small_db(hs)
    data, off, ln = _pack([b"abcd cd abCD " * 40] * 300)
    scratch = hs.Scratch(db)
    corpus = hs.Corpus.upload(data, off, ln)
    _scan(hs, db, scratch, corpus)
    want = hs.fetch_matches(db, scratch)
    out, cnt = _alloc(want.size + 16)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out.zero_()
        hs.scan_corpus_async(db, corpus, scratch, stream=s.cuda_stream)
        hs.order_matches_async(db, scratch, out, cnt, stream=s.cuda_stream)
    torch.cuda.synchronize()
    got, n = _read(hs, out, cnt, want.size + 16)
    assert n == want.size and np.array_equal(got, want)
    assert hs.scan_corpus_finish(scratch)[0] == hs.HS_SUCCESS


def test_refusals(hs):
    L = hs.lib()
    db = _small_db(hs)
    other = hs.compile_lit_multi([b"zzz"], [0], [0])
    scratch = hs.Scratch(db)
    out, cnt = _alloc(4)
    o, c = C.c_void_p(hs._dev_ptr(out)), C.c_void_p(hs._dev_ptr(cnt))
    assert L.hs_b200_order_matches_async(other.ptr, scratch.ptr, o, 4, c, None) == hs.HS_INVALID
    assert L.hs_b200_order_matches_async(None, scratch.ptr, o, 4, c, None) == hs.HS_INVALID
    assert L.hs_b200_order_matches_async(db.ptr, None, o, 4, c, None) == hs.HS_INVALID
    assert L.hs_b200_order_matches_async(db.ptr, scratch.ptr, None, 4, c, None) == hs.HS_INVALID
    assert L.hs_b200_order_matches_async(db.ptr, scratch.ptr, o, 4, None, None) == hs.HS_INVALID
    assert L.hs_b200_order_records_async(db.ptr, scratch.ptr, None, 3, o, 4, c, None) == hs.HS_INVALID
    comb = hs.compile_multi([b"abc", b"bcd", b"1 & 2"], [0, 0, hs.HS_FLAG_COMBINATION], [1, 2, 3])
    cs = hs.Scratch(comb)
    assert L.hs_b200_order_matches_async(comb.ptr, cs.ptr, o, 4, c, None) == hs.HS_INVALID
    assert L.hs_b200_order_records_async(comb.ptr, cs.ptr, o, 0, o, 4, c, None) == hs.HS_INVALID
