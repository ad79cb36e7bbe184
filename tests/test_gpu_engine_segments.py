"""Long blocks cut into segments, each walked by its own lane, and joined by their start states (DESIGN.md section
10f; runtime option engine_segment).  Whatever the cut, the records are the ones the one-lane walk of a block
emits: the unmodified reference hs_scan agrees, and so does the device itself with engine_segment=-1, record for
record.  Seams are placed exactly with forced segment lengths; the default rule cuts the long blocks of corpora
that leave the GPU idle and leaves corpora that fill it as they were.  Runs on the H100 and on the SIMT emulator."""
import contextlib

import numpy as np
import pytest

from test_gpu_device_order import _alloc, _read
from test_limex import _emit, _random_nfa, _random_wide_nfa, _triples
from test_mixed_rose import MixedSet, _lits, _pack, _per_block, _ref_per_block

pytestmark = pytest.mark.gpu

CASELESS, SINGLE = 1, 8
SEGS = [16, 64, 1000, 4096]


@contextlib.contextmanager
def _opts(hs, **kw):
    defaults = {"engine_segment": 0, "initial_ring": 1 << 20, "chunk_mb": 128}
    for k, v in kw.items():
        hs.set_runtime_option(k, v)
    try:
        yield
    finally:
        for k in kw:
            hs.set_runtime_option(k, defaults[k])


def _planted(seed, lengths, plants, alphabet=b"abcdefgh ", at=()):
    """blocks of random bytes of `alphabet` with the byte strings of `plants` written in at random places, and
    at the (block, offset, bytes) of `at`"""
    rng = np.random.default_rng(seed)
    a = np.frombuffer(alphabet, dtype=np.uint8)
    blocks = []
    for n in lengths:
        d = bytearray(a[rng.integers(0, a.size, size=n)].tobytes())
        for _ in range(n // 200):
            lit = plants[int(rng.integers(0, len(plants)))]
            if len(lit) < n:
                p = int(rng.integers(0, n - len(lit) + 1))
                d[p:p + len(lit)] = lit
        blocks.append(d)
    for b, p, lit in at:
        blocks[b][p:p + len(lit)] = lit
    return [bytes(d) for d in blocks]


def _around_seams(blocks, lit, seg, b=0):
    """`lit` planted to end exactly at, one byte before and one byte after seams of `seg`-byte segments of block
    b, and to start in one segment and end two segments later"""
    d = bytearray(blocks[b])
    n = len(d)
    for k, delta in ((1, 0), (3, -1), (5, 1)):
        end = k * seg + delta
        if len(lit) <= end <= n:
            d[end - len(lit):end] = lit
    blocks[b] = bytes(d)
    return blocks


def _device(hs, db, blocks, seg, stats=False):
    """per-block delivered matches of a resident corpus scan (hs_b200_fetch_matches) with engine_segment=seg"""
    data, off, ln = _pack(blocks)
    with _opts(hs, engine_segment=seg):
        scratch = hs.Scratch(db)
        corpus = hs.Corpus.upload(data, off, ln)
        got = _per_block(hs.scan_corpus(db, corpus, scratch), len(blocks))
        st = scratch.segment_stats()
        corpus.free()
        scratch.free()
    return (got, st) if stats else got


def _check(hs, ref, db, blocks, segs=SEGS, min_matches=1):
    """the reference, the one-lane walk and every forced segment length agree; each forced length cuts"""
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) >= min_matches
    assert _device(hs, db, blocks, -1) == want
    for seg in segs:
        got, st = _device(hs, db, blocks, seg, stats=True)
        assert got == want, seg
        assert st["runs"] >= 1 and st["segments"] > len(blocks)
    return want


# ---- seams at chosen places, every engine kind ---------------------------------------------------------------------

REGEX_MCC8 = [(rb"ab+c", 0, 1, None), (rb"\d+\.\d\d", 0, 2, None), (rb"x.y", 0, 3, None), (rb"hed[a-h]{3}", 0, 4, None)]
REGEX_MCC16 = [(rb"a[ab]*a[ab]{7}c", 0, 11, None), (rb"q[0-3]+z", CASELESS, 12, None)]


def _db(hs, regexes, dfa=1):
    hs.set_build_option("regex_dfa", dfa)
    return MixedSet([], [], [], regexes).compile(hs)


@pytest.mark.parametrize("seg", SEGS)
def test_seams_mcclellan8(hs, ref, seg):
    db = _db(hs, REGEX_MCC8)
    blocks = _planted(1, [9000, 20000, 300, 0, 5000], [b"abbbc", b"12.34", b"xqy", b"hedabc"], b"abcdhexy0123.")
    blocks = _around_seams(blocks, b"abbbbbc", seg)
    blocks = _around_seams(blocks, b"a" + b"b" * (2 * seg + 3) + b"c", seg, b=1)   # spans three segments
    _check(hs, ref, db, blocks, segs=[seg], min_matches=20)


@pytest.mark.parametrize("which", [0, 1])
def test_seams_mcclellan16(hs, ref, which):
    """McClellan-16 (Sherman states compressed against a parent row), its successor table in shared memory"""
    regexes = [REGEX_MCC16, [(rb"q[a-d]{300}z", 0, 13, None)]][which]
    db = _db(hs, regexes)
    assert db.info().engine_id == 7
    plants = [b"abbaabababc", b"q0123z", b"Q33Z", b"q" + b"abcd" * 75 + b"z"]
    blocks = _planted(2, [12000, 7000, 64], plants, b"ab0123qz")
    blocks = _around_seams(blocks, b"ab" * 8 + b"c", 1000)
    _check(hs, ref, db, blocks, min_matches=10)


def test_seams_mcclellan16_table_in_l2(hs, ref):
    """a random McClellan-16 table of 300 states over 256 byte classes (150 KiB): too large for shared memory
    beside the tiles, read through L2"""
    rng = np.random.default_rng(14)
    n = 300
    nxt = rng.integers(1, n, size=(n, 256)).astype(np.uint16)
    reports = [[int(rng.integers(0, 5))] if rng.random() < 0.1 else [] for _ in range(n)]
    eod = [[int(rng.integers(50, 55))] if rng.random() < 0.1 else [] for _ in range(n)]
    eng = hs.dfa_from_table(nxt, 1, 2, reports, eod, kind=2)
    assert eng[8] == 7 and len(eng) > 300 * 256 * 2                   # NFA_MCCLELLAN_16
    blocks = [rng.integers(0, 256, size=m, dtype=np.uint8).tobytes() for m in (9000, 3000, 40, 0)]
    data, off, ln = _pack(blocks)
    want = _triples(ref.nfa_exec_blocks(eng, data, off, ln))
    assert len(want) > 100
    corpus = hs.Corpus.upload(data, off, ln)
    for seg in [-1] + SEGS:
        with _opts(hs, engine_segment=seg):
            got, _ = hs.nfa_scan_corpus(eng, corpus)
        assert _triples(got) == want, seg
    corpus.free()


def test_seams_sheng(hs, ref):
    """a literal set under outfix_engine compiles to one Sheng outfix"""
    hs.set_build_option("outfix_engine", 4)   # Sheng
    db = hs.compile_lit_multi([b"abc", b"hedge", b"cab"], [0, 0, 0], [1, 2, 3])
    blocks = _planted(3, [8000, 4097, 15], [b"abc", b"hedge", b"cab"], b"abcdegh")
    blocks = _around_seams(blocks, b"hedge", 64)
    _check(hs, ref, db, blocks, min_matches=20)


@pytest.mark.parametrize("seed", [0, 2, 3])
@pytest.mark.parametrize("wide", [False, True])
def test_seams_limex_random(hs, ref, seed, wide):
    """the random LimEx-32 / -64 tables of test_limex through hs_b200_nfa_scan_corpus"""
    spec = _random_nfa(seed, wide)
    _check_nfa(hs, ref, _emit(hs, spec), spec[0], 40 + seed)


@pytest.mark.parametrize("n", [100, 200, 450])
def test_seams_limex_wide_random(hs, ref, n):
    """LimEx-128, -256 and -512"""
    reach, init, succ, reports, eod, sqm, sk = _random_wide_nfa(1000 * n, n)
    eng = hs.limex_from_spec_wide(reach, init, init, succ, reports, eod, sqm, sk)
    _check_nfa(hs, ref, eng, reach, n, segs=[64, 1000])


def _check_nfa(hs, ref, eng, reach, seed, segs=SEGS):
    """blocks mostly of the bytes that keep state 0 on (the automaton's start is at offset 0 only: on other bytes
    it soon dies), with others among them"""
    rng = np.random.default_rng(seed)
    keep = np.array([b for b in range(256) if int(reach[b]) & 1], dtype=np.uint8)
    blocks = []
    for n in [6000, 2500, 17, 0, 1100]:
        d = rng.choice(keep, size=n)
        other = rng.random(n) < 0.3
        d[other] = rng.integers(0, 256, size=int(other.sum()), dtype=np.uint8)
        blocks.append(d.tobytes())
    data, off, ln = _pack(blocks)
    want = _triples(ref.nfa_exec_blocks(eng, data, off, ln))
    assert want
    corpus = hs.Corpus.upload(data, off, ln)
    for seg in [-1] + segs:
        with _opts(hs, engine_segment=seg):
            got, _ = hs.nfa_scan_corpus(eng, corpus, cap=64)
        assert _triples(got) == want, seg
    corpus.free()


# ---- the rules that cross seams --------------------------------------------------------------------------------------

RULES = [(rb"^abc", 0, 21, None), (rb"\Ahed", 0, 22, None), (rb"\bfeed\b", 0, 23, None), (rb"\Bace\B", 0, 24, None),
         (rb"dead$", 0, 25, None), (rb"bad\z", 0, 26, None), (rb"cab\Z", 0, 27, None),
         (rb"be+f", 0, 28, {"min_length": 6}), (rb"ca+b", 0, 29, {"min_offset": 3000, "max_offset": 9000}),
         (rb"d[a-f]{2}e", SINGLE, 30, None), (rb"fa+c", 0, 31, None), (rb"ga+c", 0, 31, None)]


@pytest.mark.parametrize("dfa", [1, 0])
def test_rules_at_seams(hs, ref, dfa):
    """anchors, word boundaries at a seam, end anchors, min_length across seams, hs_expr_ext bounds,
    HS_FLAG_SINGLEMATCH first matching in a later segment, an id shared by two expressions"""
    db = _db(hs, RULES, dfa)
    plants = [b" feed ", b"xacex", b"beeeef", b"caaab", b"faac", b"gaac"]
    at = [(0, 0, b"abc"), (1, 0, b"hed"), (2, 2000, b"dabe")]
    blocks = _planted(5, [9000, 5000, 4100, 3, 2000], plants, b"abcdefgh ", at)
    blocks[0] = blocks[0][:-4] + b"dead"
    blocks[1] = blocks[1][:-3] + b"bad"
    blocks[2] = blocks[2][:-4] + b"cab\n"
    blocks[4] = blocks[4][:-3] + b"cab"
    blocks = _around_seams(blocks, b" feed ", 1000, b=4)
    _check(hs, ref, db, _words_at_seams(blocks), min_matches=30)


def _words_at_seams(blocks):
    """for every forced segment length: in block 0 a word that ends a segment (its \\b look-ahead byte starts the
    next) and one that starts a segment; in block 1 a \\B match whose last byte ends a segment"""
    d0, d1 = bytearray(blocks[0]), bytearray(blocks[1])
    for seg, k0, k1 in ((16, 7, 9), (64, 5, 7), (1000, 3, 2), (4096, 2, 1)):
        for end in (k0 * seg + 1, (k0 + 1) * seg + 5):      # " feed" ends at the seam / "feed" starts at it
            if end + 1 <= len(d0):
                d0[end - 6:end] = b" feed "
        d1[k1 * seg - 4:k1 * seg + 1] = b"xacex"
    return [bytes(d0), bytes(d1)] + blocks[2:]


def test_guesses_always_wrong(hs, ref):
    """foo[^X]*bar over data without X and foo only in segment 0: every guess is wrong, the join carries the
    state across every seam"""
    db = _db(hs, [(rb"foo[^X]*bar", 0, 41, None)])
    n = 40000
    rng = np.random.default_rng(6)
    d = bytearray(rng.choice(np.frombuffer(b"abcdefg", np.uint8), size=n).tobytes())
    d[3:6] = b"foo"
    for p in range(500, n, 3001):
        d[p:p + 3] = b"bar"
    blocks = [bytes(d)]
    want = _check(hs, ref, db, blocks, segs=[64, 1000, 4096], min_matches=10)
    got, st = _device(hs, db, blocks, 1000, stats=True)
    assert got == want and st["rewalks"] >= 1


# ---- the default rule --------------------------------------------------------------------------------------------------

def _big(seed, n, plants):
    rng = np.random.default_rng(seed)
    d = bytearray(rng.choice(np.frombuffer(b"abcdhexy0123. ", np.uint8), size=n).tobytes())
    for p in rng.integers(0, n - 16, size=max(8, n // 20000)).tolist():
        lit = plants[p % len(plants)]
        d[p:p + len(lit)] = lit
    return bytes(d)


BIG = 16 << 20


def test_default_rule_cuts_one_large_buffer(hs, ref):
    """one large buffer through hs_scan, and through a resident corpus with hs_b200_fetch_matches and the
    device ordering: the rule cuts it"""
    db = _db(hs, REGEX_MCC8)
    buf = _big(7, BIG, [b"abbc", b"1.23", b"xay", b"hedabc"])
    want = _ref_per_block(ref, db, [buf])[0]
    assert len(want) > 100
    scratch = hs.Scratch(db)
    rc, got = hs.scan(db, buf, scratch)
    assert rc == 0 and sorted((to, i) for i, to in got) == want
    st = scratch.segment_stats()
    assert st["runs"] == 1 and st["segments"] > 1
    data, off, ln = _pack([buf])
    corpus = hs.Corpus.upload(data, off, ln)
    assert _per_block(hs.scan_corpus(db, corpus, scratch), 1)[0] == want
    hs.scan_corpus_async(db, corpus, scratch)
    out, cnt = _alloc(len(want) + 64)
    hs.order_matches_async(db, scratch, out, cnt, cap=len(want) + 64)
    recs, c = _read(hs, out, cnt, len(want) + 64)
    assert c == len(want) and [(int(r["to"]), int(r["id"])) for r in recs] == want
    corpus.free()
    scratch.free()


def test_default_rule_mixed_corpus(hs, ref):
    """many 1 KiB blocks and a few long ones: the long ones are cut, the short ones stay one segment each"""
    db = _db(hs, REGEX_MCC8)
    big = 4 << 20
    blocks = _planted(8, [1024] * 600, [b"abbc", b"1.23", b"xay"], b"abcdxy0123.") + \
        [_big(9 + i, big, [b"abbc", b"xay"]) for i in range(3)]
    want = _ref_per_block(ref, db, blocks)
    got, st = _device(hs, db, blocks, 0, stats=True)
    assert got == want and st["runs"] == 1 and st["segments"] > len(blocks)


def test_corpus_that_fills_the_gpu_launches_as_before(hs, ref):
    """4 096 blocks of 1 KiB: no block is cut, and the engine run is the one launch it was"""
    db = _db(hs, REGEX_MCC8)
    blocks = _planted(10, [1024] * 4096, [b"abbc", b"1.23"], b"abcd0123.")
    data, off, ln = _pack(blocks)
    scratch = hs.Scratch(db)
    corpus = hs.Corpus.upload(data, off, ln)
    counts = []
    for seg in (-1, 0):
        with _opts(hs, engine_segment=seg):
            n0 = hs.launch_count()
            got = _per_block(hs.scan_corpus(db, corpus, scratch), len(blocks))
            counts.append(hs.launch_count() - n0)
    assert counts[0] == counts[1] and scratch.segment_stats()["runs"] == 0
    assert got == _ref_per_block(ref, db, blocks)
    corpus.free()
    scratch.free()


# ---- other database shapes ----------------------------------------------------------------------------------------------

def test_literals_beside_an_engine(hs, ref):
    """a literal matcher beside one engine (FULL_ROSE with one outfix)"""
    lits, _ = _lits(1000, 6)
    ms = MixedSet(lits, [0] * 1000, list(range(1000)), REGEX_MCC8)
    hs.set_build_option("regex_dfa", 1)
    db = ms.compile(hs)
    blocks = _planted(11, [30000, 9000], list(lits[:20]) + [b"abbbc", b"9.99", b"xqy"],
                      b"abcdefghijklmnopqrstuvwxyz0123.")
    _check(hs, ref, db, blocks, segs=[1000, 4096], min_matches=20)


def test_five_engines(hs, ref):
    """a set split over five engines (FULL_ROSE with several outfixes): each engine's chain joins on its own"""
    from test_multi_outfix import _seeded
    rs, samples = _seeded(2, 60)
    db = rs.compile(hs)
    assert db.info().engine_count == 5
    blocks = _planted(12, [20000, 7000], samples, b"abcdqrstxyz0123 ")
    _check(hs, ref, db, blocks, segs=[64, 4096], min_matches=20)


# ---- the scan driver ---------------------------------------------------------------------------------------------------

def test_ring_overflow_upload_chunks_and_termination(hs, ref):
    """a 16-record ring (the scan grows it and runs again), 1 MiB upload chunks, and a callback that stops"""
    db = _db(hs, REGEX_MCC8)
    blocks = _planted(13, [3 << 20, 5000], [b"abbc", b"1.23", b"xay"], b"abcdxy0123.")
    want = _ref_per_block(ref, db, blocks)
    data, off, ln = _pack(blocks)
    with _opts(hs, engine_segment=1000, initial_ring=16, chunk_mb=1):
        scratch = hs.Scratch(db)
        assert _per_block(hs.scan_blocks(db, data, off, ln, scratch), len(blocks)) == want
        rc, full = hs.scan(db, blocks[0], scratch)
        assert rc == 0 and sorted((to, i) for i, to in full) == want[0]
        rc, got = hs.scan(db, blocks[0], scratch, stop_after=3)
        assert rc == hs.HS_SCAN_TERMINATED and got == full[:3]
        scratch.free()
