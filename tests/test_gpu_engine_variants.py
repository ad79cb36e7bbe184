"""Every launch variant of the DFA / NFA kernel, dfaStagedKernel<ENGINE, SMEM_TABLE, CH, ILP, FUSED, SEG, MASK>
(dfa_kernels.cu, chosen in launchStaged), against the unmodified reference engines: each engine kind in each walk
that applies to it.

  one block per lane      dfa_ilp=1, engine_segment=-1                    <E, T, 128, 1, false, false, false>
  two blocks per lane     dfa_ilp=2, engine_segment=-1 (below LimEx-128)  <E, T, 64, 2, false, false, false>
  segmented               engine_segment=16 / 64                          <E, T, 128, 1, false, true, false>
  mask                    a mask pass over a single-outfix database       <E, T, 128, 1, false, false, true>
  mask + segmented        the same with engine_segment=16 / 64            <E, T, 128, 1, false, true, true>
  fused, fused + mask     databases of several outfixes                   <E, T, 128, 1, true, false, false / true>

The engine kinds are McClellan-8, McClellan-16 with its table in shared memory (T=1) and read through L2 (T=0),
Sheng, and LimEx-32 / 64 / 128 / 256 / 512.  Raw engines run through hs_b200_nfa_scan_corpus and are compared with
the reference's nfaExec*_B / nfaExecLimEx*_Q + _testEOD; databases through the resident-corpus scan and its mask
pass, compared with the reference hs_scan per block.  dfa_ilp is read by hs_b200_nfa_scan_corpus on every call and
by a database scan when its scratch is made.

The two-blocks-per-lane walk gets corpora with a case on each side of its edges: block counts around multiples of
32 and 64 (so that the last group's second chain lies wholly, partly or not at all past the last block), block
lengths around the 16-byte piece and the 64-byte refill, ragged offsets and a uniform pitch, pairs of blocks 32
apart of which one is short and the other long (each way round), chains that die in their first piece beside one
that lives, matches ending on the last byte of a refill and on the first of the next, and end-of-data accepts in
blocks whose partner chain is past the last block.  The two walks agree record for record.

Instantiations no public call can reach (the 63 are listed, with call counts, by tests/emu/kernel_coverage.py):
  - <LimEx-128 / 256 / 512, 1, 64, 2, false, false, false>: launchStaged instantiates the two-chain walk for every
    engine kind, but selects it only below LimEx-128 (a wide state set in two chains does not fit the registers).
  - <Sheng, 1, 128, 1, true, false, false / true>: Sheng engines come only from literal sets compiled as one
    outfix (build option outfix_engine); the regular-expression route, which alone builds databases of several
    outfixes, emits McClellan-8 / 16 or LimEx, so a fused launch never holds a Sheng engine.
One pair is reachable but not reached here:
  - <McClellan-16, 0, 128, 1, true, false, false / true>: a fused launch of a McClellan-16 whose table does not fit
    shared memory beside the tiles.  The regular-expression route determinises a group only up to 1 024 states and
    compresses its rows (Sherman states), so it needs a group whose remaining table passes about 67 KiB; the
    groups built here stay in shared memory.
Runs on the H100 and, smaller, on the SIMT emulator."""
import contextlib
import os

import numpy as np
import pytest

from hyperscan_b200 import synth
from test_dfa import _random_table
from test_gpu_match_mask import _host_arr, _mask_of
from test_gpu_scan_rows import _dev
from test_limex import _emit, _random_nfa, _random_wide_nfa, _triples
from test_mixed_rose import _per_block
from test_multi_outfix import KIND_GROUPS, RegexSet

pytestmark = pytest.mark.gpu

EMU = os.environ.get("HSB200_EMU") == "1"
KILL = 0xFF          # the byte that sends every engine built here to its dead state
ILP2_KINDS = ("sheng", "mcclellan8", "mcclellan16", "mcclellan16_l2", "limex32", "limex64")
NFA_TYPE = {"sheng": 17, "mcclellan8": 6, "mcclellan16": 7, "mcclellan16_l2": 7, "limex32": 0, "limex64": 1,
            "limex128": 2, "limex256": 3, "limex512": 5}


@contextlib.contextmanager
def _opts(hs, **kw):
    defaults = {"dfa_ilp": 1, "engine_segment": 0, "initial_ring": 1 << 20}
    for k, v in kw.items():
        hs.set_runtime_option(k, v)
    try:
        yield
    finally:
        for k in kw:
            hs.set_runtime_option(k, defaults[k])


# ---- corpora ---------------------------------------------------------------------------------------------------------

COUNTS = [1, 31, 33, 64, 65, 129, 300] if EMU else [1, 31, 32, 33, 63, 64, 65, 96, 127, 129, 3000]
LENS = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 300]       # 300: several 64- and 128-byte refills
SEGS = [16, 64]


def _layout(blocks, seed):
    """ragged: blocks in random order with gaps, at offsets of every residue mod 16"""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(blocks))
    off = np.zeros(len(blocks), np.uint64)
    buf = bytearray()
    for b in order.tolist():
        buf += bytes(int(rng.integers(0, 20)))
        off[b] = len(buf)
        buf += blocks[b]
    data = np.frombuffer(bytes(buf) + bytes(16), np.uint8).copy()
    return data, off, np.array([len(d) for d in blocks], np.uint32)


def _uniform(blocks, pitch):
    data = np.zeros(len(blocks) * pitch + 16, np.uint8)
    for i, d in enumerate(blocks):
        data[i * pitch:i * pitch + len(d)] = np.frombuffer(d, np.uint8)
    return data, np.arange(len(blocks), dtype=np.uint64) * pitch, np.array([len(d) for d in blocks], np.uint32)


def _corpora(gen, kill=True):
    """(name, blocks, layout) for the two-chain walk's edges; gen(rng, n) makes n bytes an engine lives on"""
    rng = np.random.default_rng(7)
    out = []
    for n in COUNTS:
        lens = [300] + [LENS[int(i)] for i in rng.integers(0, len(LENS), size=n - 1)]
        out.append(("count%d" % n, [gen(rng, m) for m in lens], "ragged"))
    # chain pairs: block t short and t + 32 long, then the reverse; the last group partial
    short = [0, 1, 5, 15, 16, 17, 31, 33]
    lens = [short[t % 8] for t in range(32)] + [250 + t for t in range(32)]
    lens += [250 + t for t in range(32)] + [short[t % 8] for t in range(32)] + [200] * 9 + [3] * 9
    out.append(("pairs", [gen(rng, m) for m in lens], "ragged"))
    if kill:
        # a chain that dies in its first piece (at byte t % 16) while its partner lives, each way round; and deaths
        # in later pieces and refills
        blocks = []
        for t in range(128):
            d = bytearray(gen(rng, 200 + t))
            if (t // 32) % 2 == 0:
                d[t % 16] = KILL
            elif t >= 96:
                d[16 + 37 * (t % 5)] = KILL
            blocks.append(bytes(d))
        out.append(("dead", blocks, "ragged"))
    # refill edges: blocks of 60-200 bytes, matches at and around 64 and 128
    out.append(("edges", [gen(rng, 60 + 2 * t) for t in range(70)], "ragged"))
    # uniform pitch: every block equally long (no offset tables), a whole and a partial last group
    out.append(("uniform100", [gen(rng, 100) for _ in range(97)], 112))
    out.append(("uniform128", [gen(rng, 128) for _ in range(64 if EMU else 640)], 128))
    return out


def _pack(blocks, layout, seed):
    return _layout(blocks, seed) if layout == "ragged" else _uniform(blocks, layout)


# ---- raw engines -----------------------------------------------------------------------------------------------------

def _random_bytes(avoid):
    keep = np.array([b for b in range(256) if b not in avoid], np.uint8)
    return lambda rng, n: rng.choice(keep, size=n).tobytes()


def _table_engine(hs, kind, nstates, seed):
    """a random table of test_dfa (a dead state 0, report lists of one or two ids, EOD reports 50-54), never dead
    but on KILL"""
    nxt, reports, eod = _random_table(seed, nstates, dead_frac=0.0)
    nxt[1:, KILL] = 0
    eng = hs.dfa_from_table(nxt, 1, 1, reports, eod, kind={"sheng": 3, "mcclellan8": 1, "mcclellan16": 2}[kind])
    return eng, _random_bytes({KILL})


def _limex_engine(hs, spec):
    """a random LimEx of test_limex, alive on the bytes that keep its state 0 on, dead after KILL"""
    reach = spec[0]
    if isinstance(reach, np.ndarray):
        reach = reach.copy()
        reach[KILL] = 0
        eng = _emit(hs, (reach,) + tuple(spec[1:]))
    else:
        reach = list(reach)
        reach[KILL] = 0
        eng = hs.limex_from_spec_wide(reach, spec[1], spec[1], *spec[2:])
    keep = np.array([b for b in range(256) if int(reach[b]) & 1], np.uint8)
    return eng, lambda rng, n: rng.choice(keep, size=n).tobytes()


LIT_ENDS = (64, 65, 128, 129, 192, 193)


def _literal_engine(hs):
    """the 2 000-literal McClellan-16 of test_dfa: its table (about 700 KB) is read through L2; literals planted to
    end at the refill edges"""
    lits, flags, ids = synth.literal_set(2000, min_len=4, max_len=8, seed=9, caseless_frac=0.0)
    eng = hs.dfa_from_literals(lits, [f & 1 for f in flags], ids, kind=2)
    assert len(eng) > 227 << 10
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8)

    def gen(rng, n):
        d = bytearray(rng.choice(alpha, size=n).tobytes())
        for _ in range(n // 24):
            lit = lits[int(rng.integers(0, len(lits)))]
            p = int(rng.integers(0, n - len(lit) + 1))
            d[p:p + len(lit)] = lit
        for end in LIT_ENDS:
            lit = lits[end % 7]
            if end <= n:
                d[end - len(lit):end] = lit
        return bytes(d)
    return eng, gen


def _raw_engine(hs, name):
    if name == "sheng":
        return _table_engine(hs, "sheng", 16, 31)
    if name == "mcclellan8":
        return _table_engine(hs, "mcclellan8", 256, 32)      # 64 KiB table beside 160 KiB of two-chain tiles
    if name == "mcclellan16":
        return _table_engine(hs, "mcclellan16", 700, 33)     # a table of a few KiB: in shared memory
    if name == "mcclellan16_l2":
        return _literal_engine(hs)
    if name in ("limex32", "limex64"):   # (seeds whose automata match often, at end of data too)
        return _limex_engine(hs, _random_nfa(20, False) if name == "limex32" else _random_nfa(11, True))
    n = {"limex128": 100, "limex256": 200, "limex512": 450}[name]
    return _limex_engine(hs, _random_wide_nfa(1000 * n, n))


def _modes(name, corpus):
    """(dfa_ilp, engine_segment) walks of a corpus"""
    modes = [(1, -1)]
    if name in ILP2_KINDS or corpus == "pairs":
        modes.append((2, -1))
    if corpus in ("pairs", "dead", "count%d" % COUNTS[-1]):
        modes += [(1, s) for s in SEGS]
    return modes


@pytest.mark.parametrize("name", list(NFA_TYPE))
def test_raw_engine_every_walk(hs, ref, name):
    eng, gen = _raw_engine(hs, name)
    assert eng[8] == NFA_TYPE[name]
    cases = [(c, _pack(blocks, layout, i)) for i, (c, blocks, layout) in
             enumerate(_corpora(gen, kill=name != "mcclellan16_l2"))]
    wants = [ref.nfa_exec_blocks(eng, *packed) for _, packed in cases]     # (all recorded before the device runs)
    eod_beside_past = edge_hits = 0
    for (corpus, (data, off, ln)), want in zip(cases, wants):
        want = _triples(want)
        nonempty = int(np.count_nonzero(ln))
        assert len(want) >= min(nonempty, 8), corpus                        # an empty result cannot pass
        n = ln.size
        eod_beside_past += sum(1 for r, b, _ in want if r >= 50 and b % 64 < 32 and b + 32 >= n)
        edge_hits += sum(1 for _, _, to in want if to in (64, 65, 128, 129))
        c = hs.Corpus.upload(data, off, ln)
        try:
            got = {}
            for ilp, seg in _modes(name, corpus):
                with _opts(hs, dfa_ilp=ilp, engine_segment=seg):
                    got[ilp, seg], _ = hs.nfa_scan_corpus(eng, c)
                assert _triples(got[ilp, seg]) == want, (corpus, ilp, seg)
            if (2, -1) in got:
                assert np.array_equal(got[2, -1], got[1, -1]), corpus
        finally:
            c.free()
    assert edge_hits >= 4
    if name != "mcclellan16_l2":   # (literals have no end-of-data reports)
        assert eod_beside_past >= 1


# ---- databases: one outfix, masks, segments --------------------------------------------------------------------------

def _single_outfix_db(hs, name):
    """(database, strings to plant, alphabet): literal sets compiled as one outfix of the given kind, and
    regular expressions compiled to LimEx"""
    if name == "mcclellan16_l2":
        lits, flags, ids = synth.literal_set(2000, min_len=4, max_len=8, seed=9, caseless_frac=0.0)
        hs.set_build_option("outfix_engine", 3)
        db = hs.compile_lit_multi(lits, [f & 1 for f in flags], [i % 40 for i in ids])
        return db, lits[:60], b"abcdefghijklmnopqrstuvwxyz"
    outfix = {"sheng": 4, "mcclellan8": 2, "mcclellan16": 3, "limex32": 5}
    if name in outfix:
        lits = [b"abc", b"bcd", b"dab"] if name == "sheng" else [b"abcd", b"bcad", b"dab", b"hgfe", b"ccc"]
        hs.set_build_option("outfix_engine", outfix[name])
        db = hs.compile_lit_multi(lits, [0] * len(lits), [1 + i % 4 for i in range(len(lits))])
        return db, lits, b"abcdefgh "
    n = {"limex64": 40, "limex128": 100, "limex256": 200, "limex512": 300}[name]
    hs.set_build_option("regex_dfa", 0)
    db = hs.compile_multi([b"q[a-d0-3]{%d}z" % n, rb"ab+c", rb"d[0-3]+d"], [0, 0, 0], [1, 2, 3])
    return db, [b"q" + b"a0b1" * (n // 4) + b"c3"[: n % 4] + b"z", b"abbbc", b"d0123d"], b"abcd0123qz "


def _planted_blocks(seed, lens, plant, alpha):
    rng = np.random.default_rng(seed)
    a = np.frombuffer(alpha, np.uint8)
    blocks = []
    for n in lens:
        d = bytearray(rng.choice(a, size=n).tobytes())
        for _ in range(1 + n // 64):
            lit = plant[int(rng.integers(0, len(plant)))]
            if len(lit) <= n:
                p = int(rng.integers(0, n - len(lit) + 1))
                d[p:p + len(lit)] = lit
        blocks.append(bytes(d))
    return blocks


def _db_lens(long_, n):
    rng = np.random.default_rng(n)
    lens = [LENS[int(i)] for i in rng.integers(0, len(LENS), size=n)]
    lens[:3] = [long_, 129, long_ // 2 + 5]
    return lens


def _mask_pass(hs, db, corpus, scratch, nblocks, wpb):
    mask, status = _dev(np.full((nblocks, wpb), -1, np.int32)), _dev(np.full(1, 7, np.int32))
    hs.scan_corpus_mask_async(db, corpus, scratch, mask, wpb, status)
    m, st = _host_arr(mask).reshape(nblocks, wpb), int(_host_arr(status)[0])
    rc, n, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS and st == 0 and n == 0
    return m


def _scratch(hs, db, ilp, seg):
    """a scratch made under dfa_ilp=ilp (the database's engine parameters are taken then)"""
    with _opts(hs, dfa_ilp=ilp, engine_segment=seg, initial_ring=(1 << 14) if EMU else 1 << 20):
        return hs.Scratch(db)


def _check_db(hs, ref, db, blocks, layout, seg_modes, min_matches):
    """ordinary passes under both dfa_ilp settings, and mask passes, equal the reference per block"""
    data, off, ln = _pack(blocks, layout, 3)
    recs = ref.scan_sorted(db.ptr, data, off, ln)
    want = _per_block(recs, len(blocks))
    assert sum(map(len, want)) >= min_matches
    ids = hs.report_ids(db)
    wpb = (ids.size + 31) // 32
    want_mask = _mask_of(ids, recs, len(blocks), wpb)
    corpus = hs.Corpus.upload(data, off, ln)
    try:
        got = {}
        for ilp in (1, 2):
            scratch = _scratch(hs, db, ilp, -1)
            with _opts(hs, engine_segment=-1):
                got[ilp] = hs.scan_corpus(db, corpus, scratch)
                assert _per_block(got[ilp], len(blocks)) == want, ilp
                assert np.array_equal(_mask_pass(hs, db, corpus, scratch, len(blocks), wpb), want_mask), ilp
            scratch.free()
        assert np.array_equal(got[1], got[2])
        for seg in seg_modes:
            scratch = _scratch(hs, db, 1, seg)
            with _opts(hs, engine_segment=seg):
                runs = scratch.segment_stats()["runs"]
                assert _per_block(hs.scan_corpus(db, corpus, scratch), len(blocks)) == want, seg
                assert np.array_equal(_mask_pass(hs, db, corpus, scratch, len(blocks), wpb), want_mask), seg
                assert scratch.segment_stats()["runs"] >= runs + 2, seg
            scratch.free()
    finally:
        corpus.free()
    return want


@pytest.mark.parametrize("name", list(NFA_TYPE))
def test_single_outfix_database_every_walk(hs, ref, name):
    db, plant, alpha = _single_outfix_db(hs, name)
    info = db.info()
    assert info.runtime_impl == 2 and info.engine_id == NFA_TYPE[name]
    long_ = 1200 if EMU else 5000
    blocks = _planted_blocks(11, _db_lens(long_, 70 if EMU else 400), plant, alpha)
    _check_db(hs, ref, db, blocks, "ragged", SEGS, 40)


# ---- databases of several outfixes: fused launches ------------------------------------------------------------------

# Each row is one engine: its first expression does not fit beside the row before (test_multi_outfix).  With
# regex_dfa=0 every row is a LimEx, sized by its positions; a big row between two small ones keeps them apart.
BIG = [(rb"q[a-d]{495}z", 0, 1, None), (rb"r[a-d]{495}s", 0, 2, None), (rb"t[a-d]{495}u", 0, 3, None)]
LIMEX_GROUPS = [[BIG[0]], [(rb"x[ab]{18}y+", 0, 4, None), (rb"ab+c", 0, 5, None)],
                [BIG[1]], [(rb"x[0-3]{45}y+", 0, 6, None)],
                [BIG[2]], [(rb"v[a-d0-3]{95}w+", 0, 7, None), (rb"d[0-3]+d", 0, 8, None)],
                [(rb"q[0-3]{495}z", 0, 9, None)], [(rb"v[ab]{190}w+", 0, 10, None)]]
LIMEX_KINDS = [5, 0, 5, 1, 5, 2, 5, 3]
FUSED = {"dfa": (KIND_GROUPS, 1, [7, 5, 6]), "limex": (LIMEX_GROUPS, 0, LIMEX_KINDS)}


def _fused_plant(groups):
    """a match of every expression's body"""
    return [b"q" + b"abcd" * 75 + b"z", b"r" + b"0123" * 75 + b"s", b"t" + b"30" * 100 + b"u",
            b"xba" + b"ab" * 5 + b"y", b"xYYz",
            b"q" + b"abcd" * 123 + b"abcz", b"r" + b"dcba" * 123 + b"dcbs", b"t" + b"badc" * 123 + b"bacu",
            b"x" + b"ab" * 9 + b"yy", b"abbc", b"x" + b"0123" * 11 + b"3y", b"v" + b"a0b1c2" * 15 + b"d3c2bw",
            b"d012d", b"q" + b"0123" * 123 + b"012z", b"v" + b"ab" * 95 + b"ww"]


@pytest.mark.parametrize("which", list(FUSED))
def test_fused_database_every_walk(hs, ref, which):
    groups, dfa, kinds = FUSED[which]
    hs.set_build_option("regex_dfa", dfa)
    for g, kind in zip(groups, kinds):
        info = RegexSet(g).compile(hs).info()
        assert info.runtime_impl == 2 and info.engine_count == 1 and info.engine_id == kind
    db = RegexSet([r for g in groups for r in g]).compile(hs)
    assert db.info().engine_count == len(groups)
    plant = _fused_plant(groups)
    lens = [600, 520, 300] + [LENS[i % len(LENS)] for i in range(30 if EMU else 130)]
    blocks = _planted_blocks(12, lens, plant, b"abcd0123qrstuvwxyz") + [b" " + p + b" " for p in plant]
    want = _check_db(hs, ref, db, blocks, "ragged", [], 10)
    assert {i for b in want for _, i in b} == {r[2] for g in groups for r in g}   # every engine fires
