"""Stream-set passes over rows tagged with their stream (hs_b200_streams_scan_rows_async): a batch of rows in device
memory, in arrival order, any number per stream.  Every pass, ordered on the device (hs_b200_order_matches_async) and
fetched (hs_b200_fetch_matches), equals the unmodified reference stream runtime fed each stream's rows in order, its
per-write records mapped back to rows.  Covers every literal first stage, interleaved and skewed stream ids, 1-byte and
empty rows, one stream with many rows, a batch of one write per stream against hs_b200_streams_scan_async on a twin
set, a first offset above 0, chars at the very end of their allocation, an empty batch, passes of both kinds and
resets interleaved on one set, the overflow and bad-batch protocols (an empty batch behind a failed pass included),
the set's state read back around passes, the refusals and 200 passes back to back.  Runs on the H100 and, with numpy
arrays as device memory, on the SIMT emulator."""
import ctypes as C
import os

import numpy as np
import pytest

from hyperscan_b200 import synth

EMU = os.environ.get("HSB200_EMU") == "1"

pytestmark = pytest.mark.gpu

# name: (literals, min length, runtime options, AVX2 platform)
ENGINES = {"noodle": (1, 3, {}, False), "teddy8": (40, 2, {}, False), "fat_teddy": (80, 2, {}, True),
           "fdr": (300, 2, {}, False), "gram4": (400, 4, {"gram": 2}, False)}
ALPHABET = b"abcdefAB"


# ---- device memory: torch CUDA tensors on the GPU, host arrays under the emulator ------------------------------------

def _dev(a):
    a = np.ascontiguousarray(a)
    if EMU:
        return a.copy()
    import torch
    if a.dtype == np.uint32:           # torch's CUDA kernels take int32; the bits are the same
        a = a.view(np.int32)
    elif a.dtype == np.uint64:
        a = a.view(np.int64)
    return torch.from_numpy(a.copy()).cuda()


def _out(cap):
    if EMU:
        return np.zeros(cap * 16, dtype=np.uint8), np.zeros(1, dtype=np.uint64)
    import torch
    return (torch.empty(cap * 16, dtype=torch.uint8, device="cuda"),
            torch.zeros(1, dtype=torch.int64, device="cuda"))


def _stream():
    """a CUDA stream of its own for the passes (None under the emulator, where every call completes at once)"""
    if EMU:
        return None
    import torch
    torch.cuda.synchronize()                       # the tensors were filled on torch's stream
    return torch.cuda.Stream()


def _sync():
    if not EMU:
        import torch
        torch.cuda.synchronize()


def _read(hs, out, cnt):
    o = out if EMU else out.cpu().numpy()
    c = int(cnt[0]) if EMU else int(cnt.cpu().numpy().view(np.uint64)[0])
    if c == hs.ORDER_RING_OVERFLOW:
        return None
    assert c * 16 <= o.size, "the test's output buffer is too small"
    return o.view(hs.MATCH_DTYPE)[:c].copy()


def _scratch(hs, db, ring=1 << 14):
    """under the emulator a small ring, as the emulated shapes are: the ordering kernels' grids follow the ring"""
    if not EMU and ring == 1 << 14:
        return hs.Scratch(db)
    hs.set_runtime_option("initial_ring", ring)
    try:
        return hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)


def _compile(hs, name, seed):
    n, min_len, opts, avx2 = ENGINES[name]
    for k, v in opts.items():
        hs.set_runtime_option(k, v)
    lits, flags, ids = synth.literal_set(n, min_len=min_len, max_len=8, seed=seed, caseless_frac=0.2,
                                         alphabet=b"abcdef")
    plat = None
    if avx2:
        plat = C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0))
    db = hs.compile_lit_multi(lits, flags, ids, mode=hs.HS_MODE_STREAM, platform=plat)
    if avx2:
        assert 3 <= db.info().engine_id <= 10
    return lits, db


@pytest.fixture(autouse=True)
def _gram_default(hs):
    yield
    hs.set_runtime_option("gram", 1)


# ---- batches and the reference -------------------------------------------------------------------------------------

class Batch:
    """rows (bytes) written to streams `sids`, in this order, laid out in one chars array behind `lead` bytes that
    belong to no row (d_offsets[0] = lead); `tail` bytes after the last row"""

    def __init__(self, rows, sids, lead=0, tail=0, seed=0):
        rng = np.random.default_rng(seed)
        self.rows = [bytes(r) for r in rows]
        self.sids = np.asarray(sids, dtype=np.uint32)
        assert len(self.rows) == self.sids.size
        lens = np.array([len(r) for r in self.rows], dtype=np.uint64)
        self.offsets = np.zeros(len(self.rows) + 1, dtype=np.uint64)
        self.offsets[1:] = np.cumsum(lens)
        self.offsets += np.uint64(lead)
        body = np.frombuffer(b"".join(self.rows), dtype=np.uint8)
        self.chars = np.concatenate([rng.integers(0, 256, size=lead, dtype=np.uint8), body,
                                     rng.integers(0, 256, size=tail, dtype=np.uint8)]).astype(np.uint8)

    def pieces(self):
        """(row, stream, bytes) in row order"""
        return [(r, int(s), b) for r, (s, b) in enumerate(zip(self.sids.tolist(), self.rows))]


def _random_batch(lits, nrows, nstreams, seed, max_len=40, active=None, empty_frac=0.1, lead=0, plant_per_kb=60):
    """rows of 0..max_len bytes over ALPHABET with literals planted, stream ids skewed (Zipf) over `active` streams
    scattered in the set"""
    rng = np.random.default_rng(seed)
    active = active or nstreams
    flows = rng.choice(nstreams, size=active, replace=False)
    z = np.minimum(rng.zipf(1.3, size=nrows) - 1, active - 1)
    sids = flows[z].astype(np.uint32)
    lens = rng.integers(1, max_len + 1, size=nrows)
    lens[rng.random(nrows) < empty_frac] = 0
    data, off, _ = synth.ragged_corpus([int(x) for x in lens], lits, seed=seed, plant_per_kb=plant_per_kb, align=1,
                                       alphabet=ALPHABET)
    rows = [data[int(o):int(o) + int(n)].tobytes() for o, n in zip(off, lens)]
    return Batch(rows, sids, lead=lead, tail=int(rng.integers(0, 9)), seed=seed)


def _want(ref, db, events):
    """the reference's matches of every pass, as sorted (block, to, id): events are ("rows", Batch),
    ("writes", [bytes per stream]) -- a pass of hs_b200_streams_scan_async, block = stream -- and ("reset", streams)"""
    per = {}   # stream -> segments (between resets) of [(pass, block, bytes)]
    want = {k: [] for k, e in enumerate(events) if e[0] != "reset"}
    for k, (kind, x) in enumerate(events):
        if kind == "reset":
            for s in x:
                if s in per:
                    per[s].append([])
            continue
        items = x.pieces() if kind == "rows" else [(s, s, b) for s, b in enumerate(x)]
        for blk, s, b in items:
            per.setdefault(s, [[]])[-1].append((k, blk, b))
    for s in sorted(per):
        for seg in per[s]:
            if not seg:
                continue
            cat = np.frombuffer(b"".join(b for (_, _, b) in seg), dtype=np.uint8)
            wl = np.array([len(b) for (_, _, b) in seg], dtype=np.uint32)
            recs, err = ref.stream_collect(db.ptr, cat, wl)
            assert err == 0
            for r in recs:
                k, blk, _ = seg[int(r["block"])]
                want[k].append((blk, int(r["to"]), int(r["id"])))
    return {k: sorted(v) for k, v in want.items()}


def _tuples(a):
    return None if a is None else [(int(r["block"]), int(r["to"]), int(r["id"])) for r in a]


def _enqueue(hs, sset, db, scratch, events, stream, cap=1 << 16):
    """every event back to back on `stream`, each pass followed by its ordering; returns what to read"""
    sp = stream.cuda_stream if stream is not None else None
    keep, outs = [], {}
    for k, (kind, x) in enumerate(events):
        if kind == "reset":
            d = _dev(np.asarray(x, dtype=np.uint32))
            keep.append(d)
            sset.reset_async(d, stream=sp)
            continue
        if kind == "rows":
            dev = (_dev(x.chars), _dev(x.offsets), _dev(x.sids))
            keep.append(dev)
            sset.scan_rows_async(*dev, scratch, stream=sp)
        else:
            pitch = 16 + max(16, (max(len(b) for b in x) + 15) // 16 * 16)
            buf = np.zeros(len(x) * pitch, dtype=np.uint8)
            for i, b in enumerate(x):
                buf[i * pitch + 16:i * pitch + 16 + len(b)] = np.frombuffer(b, dtype=np.uint8)
            dev = (_dev(buf), _dev(np.array([len(b) for b in x], dtype=np.uint32)))
            keep.append(dev)
            sset.scan_async(dev[0], pitch, dev[1], scratch, stream=sp)
        outs[k] = _out(cap)
        hs.order_matches_async(db, scratch, outs[k][0], outs[k][1], stream=sp)
    return keep, outs


def _run(hs, sset, db, scratch, events, cap=1 << 16):
    """enqueue everything, one synchronisation, one finish; the ordered matches of every pass"""
    keep, outs = _enqueue(hs, sset, db, scratch, events, _stream(), cap)
    _sync()
    rc, _, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS
    del keep
    return {k: _read(hs, o, c) for k, (o, c) in outs.items()}


def _check(got, want):
    assert set(got) == set(want)
    for k in want:
        assert got[k] is not None, k
        assert _tuples(got[k]) == want[k], k


# ---- tests ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(ENGINES))
def test_interleaved_rows_equal_reference(hs, ref, name):
    """Three batches of interleaved, Zipf-skewed stream ids (a few streams take most rows, most none), empty rows
    among them, a first offset above 0; fetch_matches serves the last pass."""
    if EMU and name != "teddy8":
        pytest.skip("the emulator rehearses one first stage of this shape; the H100 runs all five")
    lits, db = _compile(hs, name, seed=ENGINES[name][0] + 7)
    scratch = _scratch(hs, db)
    nstreams, nrows = (64, 300) if EMU else (4096, 6000)
    events = [("rows", _random_batch(lits, nrows, nstreams, seed=100 * k + len(name), active=nstreams // 2,
                                     lead=5 + k)) for k in range(3)]
    sset = hs.StreamSet(db, nstreams)
    got = _run(hs, sset, db, scratch, events, cap=1 << 16 if EMU else 1 << 20)
    want = _want(ref, db, events)
    _check(got, want)
    assert sum(len(v) for v in want.values()) > nrows // 4
    assert np.array_equal(hs.fetch_matches(db, scratch), got[2])
    sset.close()


def test_one_byte_rows_across_passes(hs, ref):
    """Every row one byte, streams interleaved: an 8-byte literal spans 8 rows, and passes cut through it, so its
    first bytes arrive as look-behind."""
    lit = b"abcdefgh"
    db = hs.compile_lit_multi([lit, b"hab", b"ga"], ids=[1, 2, 3], mode=hs.HS_MODE_STREAM)
    scratch = _scratch(hs, db)
    nstreams = 5
    text = {s: (b"x" * s + lit * 3 + b"ab")[:20 + s] for s in range(nstreams)}
    order = [(s, i) for i in range(max(len(t) for t in text.values())) for s in range(nstreams) if i < len(text[s])]
    cuts = [0, 13, 14, 50, len(order)]                   # passes of 13, 1, 36, ... rows
    events = []
    for a, b in zip(cuts, cuts[1:]):
        part = order[a:b]
        events.append(("rows", Batch([text[s][i:i + 1] for s, i in part], [s for s, _ in part], seed=a)))
    sset = hs.StreamSet(db, nstreams)
    got = _run(hs, sset, db, scratch, events)
    want = _want(ref, db, events)
    _check(got, want)
    assert sum(1 for v in want.values() for (_, _, i) in v if i == 1) == 2 * nstreams
    sset.close()


@pytest.mark.parametrize("spread", ["one_stream_of_many", "every_row_one_stream"])
def test_many_rows_on_one_stream(hs, ref, spread):
    """10^5 rows on one stream among a few others' (2 000 under the emulator), and a batch whose rows all go to one
    stream."""
    if EMU and spread == "every_row_one_stream":
        pytest.skip("the emulator rehearses one spread of this shape")
    lits, db = _compile(hs, "teddy8", seed=31)
    scratch = _scratch(hs, db, ring=1 << 16 if EMU else 1 << 22)
    nstreams, nrows = 8, (2000 if EMU else 100000)
    rng = np.random.default_rng(31)
    events = []
    for k in range(2):
        b = _random_batch(lits, nrows, nstreams, seed=40 + k, max_len=12, plant_per_kb=60 if EMU else 4)
        if spread == "every_row_one_stream":
            b.sids[:] = 6
        else:
            b.sids[rng.random(nrows) < 0.95] = 3
        events.append(("rows", b))
    sset = hs.StreamSet(db, nstreams)
    got = _run(hs, sset, db, scratch, events, cap=1 << 18 if EMU else 1 << 22)
    _check(got, _want(ref, db, events))
    sset.close()


@pytest.mark.parametrize("name", ["teddy8", "fdr"])
def test_one_write_per_stream_equals_pitched_pass(hs, ref, name):
    """A batch in which each stream appears at most once is a hs_b200_streams_scan_async pass: with row r written
    to stream r the ordered matches equal those of a twin set fed the same writes through the pitched path, bit for
    bit; with the rows in another order they are the same matches with the row in place of the stream.  The raw
    records exported from the ring, ordered, equal them too."""
    if EMU and name != "teddy8":
        pytest.skip("the emulator rehearses one first stage of this shape")
    lits, db = _compile(hs, name, seed=55)
    scratch = _scratch(hs, db)
    nstreams = 65 if EMU else 257
    rng = np.random.default_rng(55)
    rounds = []
    for k in range(3):
        b = _random_batch(lits, nstreams, nstreams, seed=60 + k, max_len=48)
        rounds.append([r for r in b.rows])
    rows_set, twin = hs.StreamSet(db, nstreams), hs.StreamSet(db, nstreams)
    perm = rng.permutation(nstreams).astype(np.uint32)
    for k, writes in enumerate(rounds):
        ident = Batch(writes, np.arange(nstreams), lead=k, seed=k)
        got = _run(hs, rows_set, db, scratch, [("rows", ident)])[0]
        want = _run(hs, twin, db, scratch, [("writes", writes)])[0]
        assert got.size > 0 and np.array_equal(got, want), k
    # the same writes once more, rows in another order, some streams without a row
    keep = perm[: nstreams - nstreams // 8]
    extra = [rounds[0][s] for s in keep]
    b = Batch(extra, keep, seed=9)
    events = [("rows", b)]
    got = _run(hs, rows_set, db, scratch, events)[0]
    want = _run(hs, twin, db, scratch, [("writes", [rounds[0][s] if s in set(keep.tolist()) else b""
                                                    for s in range(nstreams)])])[0]
    mapped = sorted((int(keep[r["block"]]), int(r["to"]), int(r["id"])) for r in got)
    assert mapped == _tuples(want)
    # the raw records of a pass, exported and ordered, equal its delivered matches
    L = hs.lib()
    dev = (_dev(b.chars), _dev(b.offsets), _dev(b.sids))
    cap = 1 << 14
    recs, cnt = _out(cap)
    s = _stream()
    sp = s.cuda_stream if s is not None else None
    rows_set.scan_rows_async(*dev, scratch, stream=sp)
    assert L.hs_b200_export_records_async(scratch.ptr, C.c_void_p(hs._dev_ptr(recs)), cap,
                                          C.c_void_p(hs._dev_ptr(cnt)), C.c_void_p(sp or 0)) == hs.HS_SUCCESS
    _sync()
    rc, n, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS and 0 < n <= cap
    fetched = hs.fetch_matches(db, scratch)
    raw = recs if EMU else recs.cpu().numpy()
    c = int(cnt[0]) if EMU else int(cnt.cpu().numpy().view(np.uint64)[0])
    assert c == n
    raw = np.sort(raw.view(hs.MATCH_DTYPE)[:c], order=["block", "to", "id"])
    keepm = np.ones(raw.size, dtype=bool)
    keepm[1:] = raw[1:] != raw[:-1]
    assert np.array_equal(raw[keepm], fetched)
    rows_set.close()
    twin.close()


def test_chars_at_the_end_of_their_allocation(hs, ref):
    """The last row ends on the last byte of the chars' allocation, with a literal on it, behind rows at every
    residue mod 16 and a first offset above 0: nothing past the allocation is read (the emulator's sanitizer build
    checks it)."""
    lits, db = _compile(hs, "fdr", seed=77)
    scratch = _scratch(hs, db)
    tail = max(lits, key=len)
    nstreams = 11
    rng = np.random.default_rng(77)
    events = []
    for k in range(3):
        b = _random_batch(lits, 60, nstreams, seed=80 + k, max_len=33, lead=3 + k)
        b.rows[-1] = b"zz" + tail
        b = Batch(b.rows, b.sids, lead=3 + k, tail=0, seed=k)
        assert int(b.offsets[-1]) == b.chars.size
        events.append(("rows", b))
    sset = hs.StreamSet(db, nstreams)
    got = _run(hs, sset, db, scratch, events)
    want = _want(ref, db, events)
    _check(got, want)
    for k in range(3):
        last = len(events[k][1].rows) - 1
        assert any(blk == last for (blk, _, _) in want[k])
    sset.close()
    del rng


def test_empty_batch_and_mixed_passes_and_resets(hs, ref):
    """Passes over rows, pitched passes, resets and an empty batch interleaved on one set and one CUDA stream: every
    pass equals the reference, so the streams a pass did not name kept their state, and the ones reset started
    afresh."""
    lits, db = _compile(hs, "teddy8", seed=88)
    scratch = _scratch(hs, db)
    nstreams = 40
    rng = np.random.default_rng(88)

    def writes(seed):
        b = _random_batch(lits, nstreams, nstreams, seed=seed, max_len=30)
        return [r if rng.random() < 0.8 else b"" for r in b.rows]

    events = [("rows", _random_batch(lits, 120, nstreams, seed=1, active=10)),
              ("writes", writes(2)),
              ("rows", Batch([], [], lead=4, seed=3)),
              ("reset", [1, 2, 3, 39, nstreams + 5]),
              ("rows", _random_batch(lits, 150, nstreams, seed=4, active=12)),
              ("reset", rng.choice(nstreams, size=7, replace=False).tolist()),
              ("writes", writes(5)),
              ("rows", _random_batch(lits, 90, nstreams, seed=6, lead=17)),
              ("writes", [b"" for _ in range(nstreams)])]
    sset = hs.StreamSet(db, nstreams)
    got = _run(hs, sset, db, scratch, events)
    want = _want(ref, db, events)
    _check(got, want)
    assert got[2].size == 0 and got[8].size == 0
    sset.close()


def test_overflow_marks_the_set_until_finish(hs, ref):
    """A 16-record ring.  Pass 1 overflows it; passes 2 and 3 and a reset enqueued behind it would fit, so only the
    mark holds them back: every ordering from pass 1 on reports the overflow.  One finish returns
    HS_INSUFFICIENT_SPACE and grows the ring, and the passes and the reset enqueued again from pass 1 deliver
    exactly the reference's matches, with no loss and no doubling."""
    db = hs.compile_lit_multi([b"abcd"] * 64 + [b"wxyz"], ids=list(range(64)) + [100], mode=hs.HS_MODE_STREAM)
    nstreams = 6
    dots = lambda n: b"." * n  # noqa: E731
    b0 = Batch([dots(5) + b"wx", b"w", dots(3)], [1, 2, 3], seed=0)
    b1 = Batch([b"yz" + dots(3), b"x", b"yz" + dots(20) + b"abcd", b"abcd", b"wxyz"], [1, 2, 2, 4, 5], lead=2, seed=1)
    b2 = Batch([b"wx", b"yz", b"wxyz"], [2, 2, 3], seed=2)
    b3 = Batch([b"yz" + dots(4), b"wxyz" + dots(2)], [2, 0], seed=3)
    events = [("rows", b0), ("rows", b1), ("rows", b2), ("reset", [2]), ("rows", b3)]
    scratch = _scratch(hs, db, ring=16)
    sset = hs.StreamSet(db, nstreams)
    got, first, tries = {}, 0, 0
    while first < len(events):
        tries += 1
        assert tries <= 2                                  # one finish is enough
        tail = events[first:]
        keep, outs = _enqueue(hs, sset, db, scratch, tail, _stream())
        _sync()
        res = {k + first: _read(hs, o, c) for k, (o, c) in outs.items()}
        rc, _, _ = hs.scan_corpus_finish(scratch)
        ks = sorted(res)
        if tries == 1:
            assert rc == hs.HS_INSUFFICIENT_SPACE
            assert res[0] is not None and all(res[k] is None for k in ks[1:])
        ok = 0
        while ok < len(ks) and res[ks[ok]] is not None:
            got[ks[ok]] = res[ks[ok]]
            ok += 1
        assert all(res[k] is None for k in ks[ok:])         # nothing after an overflow is delivered
        assert (rc == hs.HS_SUCCESS) == (ok == len(ks))
        first = ks[ok] if ok < len(ks) else len(events)
        del keep
    sset.close()
    want = _want(ref, db, events)
    _check(got, want)
    assert len(want[1]) == 2 * 64 + 3 and (0, 7 + 2, 100) in want[1] and (2, 4, 100) in want[1]


@pytest.mark.parametrize("fault", ["stream_id", "decreasing_offset", "offset_past_chars"])
def test_bad_batch_fails_the_pass(hs, ref, fault):
    """A stream id at or above nstreams, an offset below the one before, an offset past chars_bytes: the pass
    delivers nothing (the ordering reports the overflow), finish returns HS_INVALID, the streams stay where they
    were, and the next passes are fine."""
    lits, db = _compile(hs, "teddy8", seed=99)
    scratch = _scratch(hs, db)
    nstreams = 9
    good = [("rows", _random_batch(lits, 50, nstreams, seed=90 + k)) for k in range(2)]
    bad = _random_batch(lits, 50, nstreams, seed=95)
    chars, offsets, sids = bad.chars, bad.offsets.copy(), bad.sids.copy()
    if fault == "stream_id":
        sids[17] = nstreams
    elif fault == "decreasing_offset":
        offsets[20] = offsets[21] + 5                      # row 20 ends before it starts
    else:
        offsets[-1] = chars.size + 1
    sset = hs.StreamSet(db, nstreams)
    s = _stream()
    sp = s.cuda_stream if s is not None else None
    dev = (_dev(chars), _dev(offsets), _dev(sids))
    outs = [_out(1024) for _ in range(2)]
    sset.scan_rows_async(*dev, scratch, stream=sp)
    hs.order_matches_async(db, scratch, outs[0][0], outs[0][1], stream=sp)
    dev2 = (_dev(good[0][1].chars), _dev(good[0][1].offsets), _dev(good[0][1].sids))
    sset.scan_rows_async(*dev2, scratch, stream=sp)                # behind the bad pass: held back by the mark
    hs.order_matches_async(db, scratch, outs[1][0], outs[1][1], stream=sp)
    _sync()
    assert [_read(hs, o, c) for (o, c) in outs] == [None, None]
    assert hs.scan_corpus_finish(scratch)[0] == hs.HS_INVALID
    got = _run(hs, sset, db, scratch, good)
    _check(got, _want(ref, db, good))
    sset.close()


def test_refusals(hs, ref):
    lits, db = _compile(hs, "teddy8", seed=4)
    scratch = _scratch(hs, db)
    sset = hs.StreamSet(db, 8)
    chars = _dev(np.zeros(64, dtype=np.uint8))
    offs = _dev(np.arange(0, 40, 8, dtype=np.uint64))
    ids = _dev(np.zeros(5, dtype=np.uint32))
    P = (lambda x: x.ctypes.data) if EMU else (lambda x: x.data_ptr())
    c, o, i = P(chars), P(offs), P(ids)
    L = hs.lib()
    V = C.c_void_p
    other = hs.compile_lit_multi([b"qqqq"], ids=[1], mode=hs.HS_MODE_STREAM)
    other_scratch = _scratch(hs, other)
    bad = [
        (None, c, 64, o, i, 4, scratch.ptr),               # no set
        (sset.ptr, None, 64, o, i, 4, scratch.ptr),        # no chars
        (sset.ptr, c, 64, None, i, 4, scratch.ptr),        # no offsets
        (sset.ptr, c, 64, o + 4, i, 4, scratch.ptr),       # misaligned offsets
        (sset.ptr, c, 64, o, None, 4, scratch.ptr),        # no stream ids
        (sset.ptr, c, 64, o, i + 2, 4, scratch.ptr),       # misaligned stream ids
        (sset.ptr, c, 64, o, i, 0xfffffff1, scratch.ptr),  # too many rows
        (sset.ptr, c, 64, o, i, 4, None),                  # no scratch
        (sset.ptr, c, 64, o, i, 4, other_scratch.ptr),     # a scratch with no image of the set's database
    ]
    for set_, ch, nb, of, si, n, scr in bad:
        assert L.hs_b200_streams_scan_rows_async(set_, V(ch) if ch else None, nb, V(of) if of else None,
                                                 V(si) if si else None, n, scr, None) == hs.HS_INVALID
    # a batch of no rows needs no chars and no ids
    assert L.hs_b200_streams_scan_rows_async(sset.ptr, None, 0, V(o), None, 0, scratch.ptr, None) == hs.HS_SUCCESS
    assert hs.scan_corpus_finish(scratch)[:2] == (hs.HS_SUCCESS, 0)
    sset.close()


def test_200_passes(hs, ref):
    """200 batches back to back (6 under the emulator), one synchronisation: offsets grow far past any batch."""
    lits, db = _compile(hs, "teddy8", seed=21)
    scratch = _scratch(hs, db, ring=1 << 12)
    nstreams = 9
    npasses = 6 if EMU else 200
    events = [("rows", _random_batch(lits, 40, nstreams, seed=3000 + k, max_len=24)) for k in range(npasses)]
    sset = hs.StreamSet(db, nstreams)
    got = _run(hs, sset, db, scratch, events, cap=1 << 12)
    want = _want(ref, db, events)
    _check(got, want)
    assert max(to for v in want.values() for (_, to, _) in v) > npasses * 40 * 12 // nstreams // 2
    sset.close()


def _state(sset):
    _sync()
    return sset.state()


def test_streams_outside_the_batch_keep_their_state(hs, ref):
    """The set's look-behind and offsets, read back before and after each pass: a stream the batch does not name
    keeps them byte for byte, a stream it names advances its offset by its rows' bytes; a pass that overflows the
    ring or a bad batch leaves every stream as it was."""
    lits, db = _compile(hs, "teddy8", seed=123)
    nstreams = 48
    scratch = _scratch(hs, db)
    sset = hs.StreamSet(db, nstreams)
    rng = np.random.default_rng(123)
    _run(hs, sset, db, scratch, [("writes", [bytes(rng.choice(list(b"abcdef"), size=int(n)).astype(np.uint8))
                                             for n in rng.integers(1, 20, size=nstreams)])])
    for k in range(3):
        b = _random_batch(lits, 60, nstreams, seed=130 + k, active=9)
        lb0, off0 = _state(sset)
        _run(hs, sset, db, scratch, [("rows", b)])
        lb1, off1 = _state(sset)
        named = np.zeros(nstreams, dtype=bool)
        named[b.sids] = True
        assert np.array_equal(lb1[~named], lb0[~named]) and np.array_equal(off1[~named], off0[~named]), k
        added = np.zeros(nstreams, dtype=np.uint64)
        np.add.at(added, b.sids, np.diff(b.offsets))
        assert np.array_equal(off1, off0 + added), k
        assert (lb1[named & (added > 0)] != lb0[named & (added > 0)]).any() or k
    # a bad batch, and a pass that overflows a 16-record ring: nothing moves
    small = _scratch(hs, db, ring=16)
    bad = _random_batch(lits, 60, nstreams, seed=140)
    bad.sids[5] = nstreams + 1
    dense = Batch([b"".join(lits) * 4] * 3, [2, 7, 2], seed=141)
    for batch, scr, rc_want in ((bad, scratch, hs.HS_INVALID), (dense, small, hs.HS_INSUFFICIENT_SPACE)):
        lb0, off0 = _state(sset)
        keep, outs = _enqueue(hs, sset, db, scr, [("rows", batch)], _stream())
        _sync()
        assert _read(hs, *outs[0]) is None
        assert hs.scan_corpus_finish(scr)[0] == rc_want
        lb1, off1 = _state(sset)
        assert np.array_equal(lb1, lb0) and np.array_equal(off1, off0)
    sset.close()


@pytest.mark.parametrize("fault", ["overflow", "bad_batch"])
def test_empty_batch_behind_a_failed_pass(hs, ref, fault):
    """An empty batch enqueued behind a pass that overflowed the ring or was bad takes the set's verdict like any
    pass: its ordering reports the overflow, the pass after it is held back too, and finish returns
    HS_INSUFFICIENT_SPACE (HS_INVALID); enqueued again from the failed pass (with the bad batch mended), every pass
    equals the reference."""
    db = hs.compile_lit_multi([b"abcd"] * 64 + [b"wxyz"], ids=list(range(64)) + [100], mode=hs.HS_MODE_STREAM)
    nstreams = 4
    scratch = _scratch(hs, db, ring=16) if fault == "overflow" else _scratch(hs, db)
    sset = hs.StreamSet(db, nstreams)
    first = Batch([b"..ab", b"wx"], [1, 3], seed=1)
    failed = Batch([b"cd..", b"yz"], [1, 3], seed=2)
    if fault == "bad_batch":
        bad = Batch(failed.rows, [1, nstreams], seed=2)
    else:
        bad = failed
    empty = Batch([], [], lead=3, seed=3)
    after = Batch([b"ab", b"cd.", b"wxyz"], [0, 0, 2], seed=4)
    _run(hs, sset, db, _scratch(hs, db), [("rows", first)])
    keep, outs = _enqueue(hs, sset, db, scratch, [("rows", bad), ("rows", empty), ("rows", after)], _stream())
    _sync()
    assert [_read(hs, *outs[k]) for k in range(3)] == [None, None, None]
    rc, _, _ = hs.scan_corpus_finish(scratch)
    assert rc == (hs.HS_INVALID if fault == "bad_batch" else hs.HS_INSUFFICIENT_SPACE)
    events = [("rows", failed), ("rows", empty), ("rows", after)]
    got = _run(hs, sset, db, scratch, events)
    want = _want(ref, db, [("rows", first)] + events)
    assert _tuples(got[1]) == []
    assert [_tuples(got[k]) for k in range(3)] == [want[k + 1] for k in range(3)]
    assert (0, 6, 0) in want[1] and (1, 4, 100) in want[1] and (2, 4, 100) in want[3]
    sset.close()
