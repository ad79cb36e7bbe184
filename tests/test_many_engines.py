"""Regular-expression sets split over any number of engines (rose_build.cpp buildMultiOutfixRose; DESIGN.md
section 10e): K outfix queues in one FULL_ROSE database without a literal matcher, for K past one multibit word
(65), at the end of the flat multibit (256) and in its tree form (257, 1 000).

CPU half: the unmodified reference hs_scan on these databases equals the definition (every end offset of a match,
restated below with Python's re) for sampled expressions, including ones that accept at end of data in engines at
queue indices past 64 and 256 and a single-match id shared by many engines; the same set always compiles to the
same bytes; databases of up to 64 engines keep the bytes they had before the limit was lifted; a database whose
queue count or EOD iterator was corrupted is refused.  GPU half: every scan entry point and the device ordering
equal the reference, with every engine_segment mode and dfa_ilp, and long blocks cut into segments keep a
segment area that does not grow with K."""
import hashlib
import json
import os
import re
import struct

import numpy as np
import pytest

from test_gpu_engine_segments import _opts
from test_mixed_rose import _blocks, _device_all_entries, _pack, _per_block, _ref_per_block

CASELESS, SINGLE = 1, 8
HERE = os.path.dirname(os.path.abspath(__file__))
TAGS = b"klmnop"
ALPHA = b"#%&~!klmnop0123456789abxy "
SHARED = 7   # the single-match id of the `~digits~` expressions, in every fifth engine
MCC8, MCC16, LIMEX512 = 6, 7, 5   # enum NFAEngineType


def _tag(i):
    """four bytes of TAGS that name engine i"""
    return bytes(TAGS[(i // 6 ** j) % 6] for j in range(4))


def _set(k):
    """expressions that split into exactly k engines: each engine has one leader of 200-300 positions (two do not
    fit one engine), in turn McClellan-16 (a counter over a-d), LimEx-512 (a counter beside a set whose DFA passes
    1 024 states) and McClellan-8; beside it `#tag digits!`, in every fourth engine an expression that accepts at
    end of data ($, \\z or a trailing \\b: queues 0, 4, ..., 64, ..., 256, ...), and in every fifth `~digits~`
    under the shared single-match id.  (pattern, flags, id, engine)"""
    out = []
    for i in range(k):
        t = _tag(i)
        if i % 3 == 0:
            out.append((b"q[a-d]{300}z", 0, 1000000 + i, i))
        elif i % 3 == 1:
            out += [(b"r[0-3]{300}s", 0, 1000000 + i, i), (b"x[ab]*a[ab]{10}y", 0, 2000000 + i, i)]
        else:
            out += [(b"t[0-3]{200}u", 0, 1000000 + i, i), (b"x" + t + b"y+", CASELESS, 2000000 + i, i)]
        out.append((b"#" + t + b"[0-9]+!", 0, 3000000 + i, i))
        if i % 4 == 0:
            eod = [b"%" + t + b"[5-9]$", b"%" + t + b"[0-4]+\\z", b"&" + t + b"[0-9]+\\b"][(i // 4) % 3]
            out.append((eod, 0, 4000000 + i, i))
        if i % 5 == 2:
            out.append((b"~[0-9]+~", SINGLE, SHARED, i))
    return out


_DBS = {}


def _db(hs, k):
    """the database of _set(k), compiled once per session"""
    if k not in _DBS:
        ex = _set(k)
        _DBS[k] = hs.compile_multi([e[0] for e in ex], [e[1] for e in ex], [e[2] for e in ex])
    return _DBS[k]


def _queues(db):
    """(NFAEngineType, accepts at end of data) of every queue, read from the serialized bytecode (RoseEngine
    queueCount at 156, nfaInfoOffset at 236; NfaInfo of 20 bytes, nfaOffset first; NFA flags at 0, type at 8)"""
    b = db.serialize()[32:]
    u32 = lambda o: struct.unpack_from("<I", b, o)[0]
    k, info = u32(156), u32(236)
    return [(b[u32(info + 20 * q) + 8], u32(u32(info + 20 * q)) & 1) for q in range(k)]


# ---- the definition ---------------------------------------------------------------------------------------------

def _ends(pat, flags, data):
    """every end offset e such that the expression matches some data[s:e] in context ($, \\z and \\b see the whole
    block): a fixed-width look-behind pins the match end to e"""
    fl = re.I if flags & CASELESS else 0
    pat = pat.replace(b"\\z", b"\\Z")   # PCRE's \z in Python's spelling
    out = []
    for e in range(1, len(data) + 1):
        rx = re.compile(b"(?:" + pat + b")(?<=(?s:\\A.{%d}))" % e, fl)
        if any(rx.match(data, s) for s in range(e)):
            out.append(e)
    return out


def _definition(exprs, block):
    """sorted (to, id) of `exprs` on one block: one report per (id, offset), the first only of a single-match id"""
    got, single = set(), set()
    for pat, fl, rid, _ in exprs:
        got.update((e, rid) for e in _ends(pat, fl, block))
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


def _sample(k):
    """engines whose expressions are checked: the first, some past 64 and 256, the last"""
    return sorted({e for e in (0, 1, 5, 63, 64, 65, 68, 72, 129, 255, 256, 257, 260, 264, 513, 996, k - 3, k - 2, k - 1)
                   if 0 <= e < k})


def _plants(engines):
    out = [b"~12~", b"~7~"]
    for i in engines:
        t = _tag(i)
        out += [b"#" + t + b"42!", b"#" + t + b"7!", b"x" + t.upper() + b"yY", b"%" + t + b"13", b"&" + t + b"9 "]
    return out


def _corpus(k, seed, n=60, max_len=72):
    """blocks over ALPHA with the sampled engines' matches planted, and blocks that end in each end-of-data
    expression of the sampled engines"""
    eng = _sample(k)
    blocks = _blocks(seed, n, max_len=max_len, plant=_plants(eng), alphabet=ALPHA, empty_every=7)
    for i in eng:
        t = _tag(i)
        blocks += [b"ab #" + t + b"3! %" + t + b"7", b"%" + t + b"0123", b"~3~ &" + t + b"55", b"&" + t + b"5%" + t + b"4"]
    return blocks + [b"", b"~", b"~1~~2~"]


def _restrict(per_block, ids):
    return [[(to, i) for to, i in blk if i in ids] for blk in per_block]


# ---- CPU half ---------------------------------------------------------------------------------------------------

KS = [65, 256, 257, 1000]


@pytest.mark.parametrize("k", KS)
def test_sets_split_into_k_engines(hs, k):
    db = _db(hs, k)
    info = db.info()
    assert (info.runtime_impl, info.hwlm_type, info.engine_count) == (0, 0, k)
    q = _queues(db)
    assert len(q) == k and {t for t, _ in q} == {MCC8, MCC16, LIMEX512}
    eod = [i for i, (_, e) in enumerate(q) if e]
    assert eod == [i for i in range(k) if i % 4 == 0]
    assert any(i >= 64 for i in eod) and (k <= 256 or any(i >= 256 for i in eod))


@pytest.mark.parametrize("k", KS)
def test_reference_scans_equal_the_definition(hs, ref, k):
    db = _db(hs, k)
    eng = set(_sample(k))
    ex = [e for e in _set(k) if e[3] in eng or e[2] == SHARED]
    ids = {e[2] for e in ex}
    blocks = _corpus(k, 11 + k)
    got = _restrict(_ref_per_block(ref, db, blocks), ids)
    assert got == [_definition(ex, b) for b in blocks]
    flat = {(i, to) for blk in got for to, i in blk}
    assert sum(map(len, got)) >= 4 * len(eng)
    # end-of-data accepts of engines past 64 (and past 256) were reported
    assert {i for i, _ in flat if i >= 4000064} and (k <= 256 or {i for i, _ in flat if i >= 4000256})
    assert all(sum(i == SHARED for _, i in blk) <= 1 for blk in got) and any(i == SHARED for i, _ in flat)


def test_same_set_same_bytes_and_round_trip(hs, ref):
    k = 257
    first = _db(hs, k).serialize()
    ex = _set(k)
    again = hs.compile_multi([e[0] for e in ex], [e[1] for e in ex], [e[2] for e in ex])
    assert again.serialize() == first
    back = hs.Database.deserialize(first)
    assert back.serialize() == first and back.info().engine_count == k
    blocks = _corpus(k, 5, n=20)
    assert _ref_per_block(ref, back, blocks) == _ref_per_block(ref, again, blocks)


def _small_sets():
    """sets of at most 64 engines whose bytes were recorded before the limit was lifted"""
    from test_multi_outfix import _seeded
    out = {"many_engines_%d" % k: [(e[0], e[1], e[2]) for e in _set(k)] for k in (2, 40, 64)}
    for seed, n in [(1, 30), (4, 170), (7, 950)]:
        rs, _ = _seeded(seed, n)
        out["multi_outfix_%d_%d" % (seed, n)] = [(r[0], r[1], r[2]) for r in rs.regexes]
    return out


def test_sets_of_up_to_64_engines_keep_their_bytes(hs):
    with open(os.path.join(HERE, "golden", "many_engines_sha256.json")) as f:
        want = json.load(f)
    got = {}
    for name, ex in _small_sets().items():
        db = hs.compile_multi([e[0] for e in ex], [e[1] for e in ex], [e[2] for e in ex])
        got[name] = (db.info().engine_count, hashlib.sha256(db.serialize()).hexdigest())
    assert got == {name: tuple(v) for name, v in want.items()}


def _crc32c(b):
    """the database checksum: CRC-32C from 0, without the final inversion (src/crypto/crc32.c as the reference
    calls it)"""
    table = []
    for n in range(256):
        c = n
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        table.append(c)
    c = 0
    for x in b:
        c = table[(c ^ x) & 0xFF] ^ (c >> 8)
    return c


def _patched(ser, at, value):
    """the serialized database with the bytecode's u32 at each offset of `at` set to `value` and its checksum made
    right again"""
    b = bytearray(ser)
    for a in (at if isinstance(at, tuple) else (at,)):
        struct.pack_into("<I", b, 32 + a, value)
    length = struct.unpack_from("<I", b, 8)[0]   # the bytecode is [32, 32 + length)
    struct.pack_into("<I", b, 20, _crc32c(bytes(b[32:32 + length])))
    return bytes(b)


def test_corrupted_tables_are_refused(hs):
    ser = _db(hs, 65).serialize()
    assert hs.Database.deserialize(ser).info().engine_count == 65
    u32 = lambda o: struct.unpack_from("<I", ser, 32 + o)[0]
    prog = u32(184)                      # RoseEngine.eodProgramOffset: ENGINES_EOD, its iter_offset at 4
    it = u32(prog + 4)
    queues = (148, 156, 400, 404)        # activeArrayCount, queueCount, outfixEndQueue, leftfixBeginQueue
    bad = [_patched(ser, queues, 66), _patched(ser, queues, 1 << 20),   # a queue count past the NfaInfo table
           _patched(ser, queues, 64),                                    # and one short of it
           _patched(ser, it, u32(it) ^ 1),                        # the iterator's root mask
           _patched(ser, it + 8, u32(it + 8) + 1),                # the root's first child
           _patched(ser, prog + 4, 1 << 30)]                      # an iterator past the bytecode
    for b in bad:
        db = hs.Database.deserialize(b)   # the checksum holds: the tables are checked where they are used
        with pytest.raises(hs.HsError) as e:
            db.info()
        assert e.value.code == hs.HS_INVALID


# ---- GPU half ---------------------------------------------------------------------------------------------------

def _device_order_equals_fetch(hs, db, blocks):
    from test_gpu_device_order import _order_last, _scan
    data, off, ln = _pack(blocks)
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
@pytest.mark.parametrize("k,seg,ilp", [(65, 0, 1), (65, -1, 1), (65, 0, 2), (65, 16, 1), (257, 0, 1), (257, 64, 1)])
def test_device_equals_reference(hs, ref, k, seg, ilp):
    db = _db(hs, k)
    blocks = _corpus(k, 23)
    with _opts(hs, engine_segment=seg):
        hs.set_runtime_option("dfa_ilp", ilp)
        try:
            want = _device_all_entries(hs, ref, db, blocks)
            assert _device_order_equals_fetch(hs, db, blocks) == want
        finally:
            hs.set_runtime_option("dfa_ilp", 1)
    assert sum(map(len, want)) > 40


@pytest.mark.gpu
def test_device_refuses_corrupted_tables(hs):
    ser = _db(hs, 65).serialize()
    db = hs.Database.deserialize(_patched(ser, (148, 156, 400, 404), 66))
    with pytest.raises(hs.HsError) as e:
        hs.Scratch(db)
    assert e.value.code == hs.HS_INVALID


def _long_blocks(k, seed, n, length):
    """n blocks of `length` bytes with the sampled engines' matches planted, each ending in a match of engine 0's
    end-of-data expression"""
    rng = np.random.default_rng(seed)
    a = np.frombuffer(ALPHA, dtype=np.uint8)
    plants = _plants(_sample(k))
    out = []
    for _ in range(n):
        d = bytearray(a[rng.integers(0, a.size, size=length)].tobytes())
        for p in rng.integers(0, length - 16, size=length // 256):
            lit = plants[int(rng.integers(0, len(plants)))]
            d[p:p + len(lit)] = lit
        tail = b"%" + _tag(0) + b"7"
        d[-len(tail):] = tail
        out.append(bytes(d))
    return out


def _resident_scan(hs, db, blocks, seg):
    """per-block matches of a resident corpus scan with engine_segment=seg; the segmented runs and their segments"""
    data, off, ln = _pack(blocks)
    with _opts(hs, engine_segment=seg):
        scratch = hs.Scratch(db)
        corpus = hs.Corpus.upload(data, off, ln)
        got = _per_block(hs.scan_corpus(db, corpus, scratch), len(blocks))
        st = scratch.segment_stats()
        runs, segments = st["runs"], st["segments"]
        corpus.free()
        scratch.free()
    return got, runs, segments


@pytest.mark.gpu
def test_long_blocks_equal_reference(hs, ref):
    """4 blocks of 12 KiB over 257 engines: the default rule, the one-lane walk and 4 KiB segments equal the
    reference"""
    k = 257
    db = _db(hs, k)
    blocks = _long_blocks(k, 3, 4, 12 << 10)
    want = _ref_per_block(ref, db, blocks)
    for seg in (0, -1, 4096):
        got, runs, _ = _resident_scan(hs, db, blocks, seg)
        assert got == want
        if seg != 0:
            assert (runs > 0) == (seg > 0)
    assert sum(map(len, want)) > 40 and all(blk[-1] == (12 << 10, 4000000) for blk in want)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [257, 1000])
def test_segment_area_bounded_by_the_gpu(hs, real_gpu, k):
    """4 blocks of 1 MiB: the default rule cuts them, and each run's engines x segments stay within 1.5 x the
    resident lanes (an H100 keeps at most 132 SMs x 1 024 lanes) however large K is; the matches are the one-lane
    walk's"""
    db = _db(hs, k)
    blocks = _long_blocks(k, 4, 4, 1 << 20)
    want, runs, _ = _resident_scan(hs, db, blocks, -1)
    got, runs, segments = _resident_scan(hs, db, blocks, 0)
    assert got == want and sum(map(len, want)) > 1000
    assert runs and runs % 3 == 0             # one fused run per engine kind, per pass of the grow-and-rescan driver
    assert segments / runs * ((k + 2) // 3) <= 1.5 * 132 * 1024
