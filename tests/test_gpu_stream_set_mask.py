"""Stream-set passes into a match mask (hs_b200_streams_scan_mask_async / hs_b200_streams_scan_rows_mask_async): bit r
of mask row b is set iff the ordinary pass, ordered on the device, delivers a match with block b and id
report_ids(db)[r].  Every mask equals the reduction of a twin set's ordered matches, fed the same writes by ordinary
passes, and of the unmodified reference stream runtime fed each stream's writes in order; the set's state equals the
twin's after every pass.  Covers every literal first stage, matches that span rows and passes, 1-byte and empty rows,
a batch all on one stream, Zipf-skewed stream ids, several words per row and spare words, the overflow protocol (a
candidate-list overflow marks the set, and the passes enqueued again after finish reproduce the twin), bad lengths and
bad batches, mask, record and reset passes interleaved over 200 passes, the refusals, and what the record readers
serve after a mask pass.  Runs on the H100 and, with numpy arrays as device memory, on the SIMT emulator."""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_stream_rows import (ENGINES, Batch, _compile, _dev, _out, _random_batch, _read, _scratch, _stream,
                                  _sync, _tuples, _want)

EMU = os.environ.get("HSB200_EMU") == "1"

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gram_default(hs):
    yield
    hs.set_runtime_option("gram", 1)


# ---- passes --------------------------------------------------------------------------------------------------------

def _host(x):
    _sync()
    a = x if EMU else x.cpu().numpy()
    return np.ascontiguousarray(a).view(np.uint32)


def _mask_of(ids, tuples, nrows, wpb):
    """the mask a list of (block, to, id) matches makes"""
    rank = {int(v): i for i, v in enumerate(ids)}
    m = np.zeros((nrows, wpb), np.uint32)
    for blk, _, i in tuples:
        r = rank[i]
        m[blk, r // 32] |= np.uint32(1 << (r % 32))
    return m


def _wpb(hs, db, spare=1):
    ids = hs.report_ids(db)
    return ids, (ids.size + 31) // 32 + spare


def _pitched(writes, lengths=None):
    """one write per stream at a pitch, and its device lengths (the real ones unless given)"""
    pitch = 16 + max(16, (max(len(b) for b in writes) + 15) // 16 * 16)
    buf = np.zeros(len(writes) * pitch, dtype=np.uint8)
    for i, b in enumerate(writes):
        buf[i * pitch + 16:i * pitch + 16 + len(b)] = np.frombuffer(b, dtype=np.uint8)
    ln = np.array([len(b) for b in writes] if lengths is None else lengths, dtype=np.uint32)
    return (_dev(buf), _dev(ln)), pitch


def _enqueue(hs, sset, db, scratch, events, stream, wpb, masked=lambda k: True, cap=1 << 16, order=True):
    """every event back to back on `stream`: a mask pass (masked(k)) into a buffer pre-filled with ones and a status
    that is not 0, or a record pass followed, given `order`, by its ordering; returns what to keep alive and what to
    read"""
    sp = stream.cuda_stream if stream is not None else None
    keep, outs = [], {}
    for k, (kind, x) in enumerate(events):
        if kind == "reset":
            d = _dev(np.asarray(x, dtype=np.uint32))
            keep.append(d)
            sset.reset_async(d, stream=sp)
            continue
        if kind == "rows":
            dev, n = (_dev(x.chars), _dev(x.offsets), _dev(x.sids)), len(x.rows)
        else:
            lengths = x[1] if kind == "bad_writes" else None
            writes = x[0] if kind == "bad_writes" else x
            dev, pitch = _pitched(writes, lengths)
            n = sset.n
        keep.append(dev)
        if masked(k):
            mask, status = _dev(np.full((n, wpb), -1, np.int32)), _dev(np.full(1, 7, np.int32))
            if kind == "rows":
                sset.scan_rows_mask_async(*dev, scratch, mask, wpb, status, stream=sp)
            else:
                sset.scan_mask_async(dev[0], pitch, dev[1], scratch, mask, wpb, status, stream=sp)
            outs[k] = ("mask", n, mask, status)
        else:
            if kind == "rows":
                sset.scan_rows_async(*dev, scratch, stream=sp)
            else:
                sset.scan_async(dev[0], pitch, dev[1], scratch, stream=sp)
            if not order:
                outs[k] = ("unordered",)
                continue
            out, cnt = _out(cap)
            hs.order_matches_async(db, scratch, out, cnt, stream=sp)
            outs[k] = ("records", out, cnt)
    return keep, outs


def _collect(hs, outs, wpb):
    """per pass: (mask, status) of a mask pass, the ordered matches (None: overflow) of a record pass"""
    _sync()
    res = {}
    for k, o in outs.items():
        if o[0] == "mask":
            res[k] = (_host(o[2]).reshape(o[1], wpb), int(_host(o[3])[0]))
        elif o[0] == "records":
            res[k] = _read(hs, o[1], o[2])
    return res


def _run(hs, sset, db, scratch, events, wpb, masked=lambda k: True, cap=1 << 16, rc=None, order=True):
    """enqueue everything, one synchronisation, one finish (HS_SUCCESS unless rc says otherwise)"""
    keep, outs = _enqueue(hs, sset, db, scratch, events, _stream(), wpb, masked, cap, order)
    res = _collect(hs, outs, wpb)
    if not outs:                                        # resets only: nothing to finish
        return res
    got_rc, n, _ = hs.scan_corpus_finish(scratch)
    assert got_rc == (hs.HS_SUCCESS if rc is None else rc)
    if got_rc == hs.HS_SUCCESS and masked(max(outs)):
        assert n == 0                                   # a mask pass writes no records
    del keep
    return res


def _state(sset):
    _sync()
    return sset.state()


def _same_state(a, b):
    (la, oa), (lb, ob) = _state(a), _state(b)
    return np.array_equal(la, lb) and np.array_equal(oa, ob)


def _nrows(sset, kind, x):
    return len(x.rows) if kind == "rows" else sset.n


def _ordinary(hs, sset, db, scratch, event, cap=1 << 16):
    """one ordinary pass of `event` (nothing for a reset), then its delivered matches: fetched (the host ordering)
    and, on the H100, ordered on the device as well, which must agree.  (The emulator runs no device ordering here:
    it emulates the ordering's many radix passes over 64-bit stream offsets slowly, and test_gpu_stream_rows already
    holds its output equal to the fetched matches there.)"""
    if event[0] == "reset":
        _run(hs, sset, db, scratch, [event], 0)
        return None
    got = _run(hs, sset, db, scratch, [event], 0, masked=lambda _: False, cap=cap, order=not EMU)
    fetched = hs.fetch_matches(db, scratch)
    if not EMU:
        assert got[0] is not None and np.array_equal(got[0], fetched)
    return fetched


def _against_twin(hs, ref, db, events, nstreams, ring=1 << 14, cap=1 << 16):
    """each event on a mask set and on a twin fed by ordinary passes, one at a time: the masks equal the twin's
    ordered matches and the reference's, reduced, and the two sets' state is the same after every pass"""
    ids, wpb = _wpb(hs, db)
    want = _want(ref, db, events)
    sset, twin = hs.StreamSet(db, nstreams), hs.StreamSet(db, nstreams)
    scratch, tscratch = _scratch(hs, db, ring=ring), _scratch(hs, db, ring=ring)
    masks = {}
    for k, (kind, x) in enumerate(events):
        got = _run(hs, sset, db, scratch, [(kind, x)], wpb)
        tw = _ordinary(hs, twin, db, tscratch, (kind, x), cap)
        assert _same_state(sset, twin), k
        if kind == "reset":
            continue
        n = _nrows(sset, kind, x)
        mask, status = got[0]
        assert status == 0, k
        assert np.array_equal(mask, _mask_of(ids, _tuples(tw), n, wpb)), k
        assert np.array_equal(mask, _mask_of(ids, want[k], n, wpb)), k
        masks[k] = mask
    sset.close()
    twin.close()
    return masks, want


# ---- tests ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(ENGINES))
def test_both_passes_equal_twin_and_reference(hs, ref, name):
    """Batches of Zipf-skewed rows with empty rows among them and a first offset above 0, a pitched pass of one write
    per stream, a reset and a batch all on one stream: every mask equals the twin's and the reference's."""
    if EMU and name not in ("noodle", "teddy8"):
        pytest.skip("the emulator rehearses two first stages of this shape; the H100 runs all five")
    lits, db = _compile(hs, name, seed=ENGINES[name][0] + 11)
    nstreams, nrows = (40, 160) if EMU else (4096, 6000)
    rng = np.random.default_rng(len(name))
    one = _random_batch(lits, nrows // 4, nstreams, seed=7, max_len=30)
    one.sids[:] = nstreams // 3
    writes = [r if rng.random() < 0.8 else b"" for r in _random_batch(lits, nstreams, nstreams, seed=5).rows]
    events = [("rows", _random_batch(lits, nrows, nstreams, seed=1, active=nstreams // 2, lead=5)),
              ("writes", writes),
              ("rows", _random_batch(lits, nrows, nstreams, seed=2, active=nstreams // 4, lead=3)),
              ("reset", rng.choice(nstreams, size=nstreams // 8, replace=False).tolist()),
              ("rows", one),
              ("writes", [b""] * nstreams),
              ("rows", _random_batch(lits, nrows, nstreams, seed=3, lead=1))]
    masks, want = _against_twin(hs, ref, db, events, nstreams, cap=1 << 16 if EMU else 1 << 20)
    assert all(masks[k].any() for k in (0, 1, 2, 4, 6)) and not masks[5].any()
    assert sum(len(want[k]) for k in want) > nrows // 2
    assert len({r for (r, _, _) in want[4]}) > 1              # the one-stream batch fires on several rows


def test_matches_spanning_rows_and_passes(hs, ref):
    """Every row one byte, streams interleaved, passes cut through the literals; empty rows; 70 ids over three words
    and a spare word, with ids in the third word firing."""
    lit = b"abcdefgh"
    extra = [b"q%02d" % i for i in range(67)]
    db = hs.compile_lit_multi([lit, b"hab", b"ga"] + extra, ids=list(range(1, 71)), mode=hs.HS_MODE_STREAM)
    ids, wpb = _wpb(hs, db)
    assert ids.size == 70 and wpb == 4
    nstreams = 5
    text = {s: b"x" * s + lit * 3 + b"q66" + b"ab" for s in range(nstreams)}
    order = [(s, i) for i in range(max(len(t) for t in text.values())) for s in range(nstreams) if i < len(text[s])]
    cuts = [0, 13, 14, 50, 80, len(order)]
    events = []
    for a, b in zip(cuts, cuts[1:]):
        part = order[a:b]
        rows = [text[s][i:i + 1] for s, i in part]
        sids = [s for s, _ in part]
        if a == 14:                                           # empty rows between the bytes
            rows = [r for x in rows for r in (x, b"")]
            sids = [s for x in sids for s in (x, (x + 1) % nstreams)]
        events.append(("rows", Batch(rows, sids, seed=a)))
    events.insert(3, ("writes", [b"q05" + b"h" * s for s in range(nstreams)]))
    masks, want = _against_twin(hs, ref, db, events, nstreams)
    rank = {int(v): i for i, v in enumerate(ids)}
    fired = {i for v in want.values() for (_, _, i) in v}
    assert {1, 9, 70} <= fired and {rank[i] // 32 for i in fired} == {0, 2}
    assert not any(m[:, 3].any() for m in masks.values())  # the spare word stays zero


def _dense_db(hs):
    return hs.compile_lit_multi([b"abcd"] * 64 + [b"wxyz"], ids=list(range(64)) + [100], mode=hs.HS_MODE_STREAM)


def test_candidate_overflow_marks_the_set_until_finish(hs, ref):
    """A 16-record ring, so a 16-candidate list.  Pass 1 overflows the list: its status is 1 and the set is marked,
    and the passes and the reset behind it, which would fit, commit nothing (status 1, state unchanged).  One finish
    returns HS_INSUFFICIENT_SPACE; enqueued again from pass 1, every mask equals the twin's and the reference's, and
    so does the state."""
    db = _dense_db(hs)
    ids, wpb = _wpb(hs, db)
    nstreams = 6
    dots = lambda n: b"." * n  # noqa: E731
    b0 = Batch([dots(5) + b"wx", b"w", dots(3)], [1, 2, 3], seed=0)
    b1 = Batch([b"yz" + dots(3), b"x" + b"abcd" * 12, b"yz" + dots(20) + b"abcd" * 12, b"abcd", b"wxyz"], [1, 2, 2, 4, 5],
               lead=2, seed=1)
    w2 = [b"", b"abcd", b"yz", b"wxyz", b"", b"ab"]
    b3 = Batch([b"yz" + dots(4), b"wxyz" + dots(2), b"cd"], [2, 0, 5], seed=3)
    events = [("rows", b0), ("rows", b1), ("writes", w2), ("reset", [2]), ("rows", b3)]
    twin = hs.StreamSet(db, nstreams)
    tscratch = _scratch(hs, db)
    _ordinary(hs, twin, db, tscratch, events[0])
    sset = hs.StreamSet(db, nstreams)
    scratch = _scratch(hs, db, ring=16)
    first = _run(hs, sset, db, scratch, events[:1], wpb)
    assert first[0][1] == 0 and _same_state(sset, twin)
    res = _run(hs, sset, db, scratch, events[1:], wpb, rc=hs.HS_INSUFFICIENT_SPACE)
    assert [res[k][1] for k in (0, 1, 3)] == [1, 1, 1]
    assert _same_state(sset, twin)                            # nothing committed, the reset included
    res = _run(hs, sset, db, scratch, events[1:], wpb)
    tw = {k: _ordinary(hs, twin, db, tscratch, e) for k, e in enumerate(events[1:])}
    assert _same_state(sset, twin)
    want = _want(ref, db, events)
    for k in (0, 1, 3):
        n = _nrows(sset, *events[k + 1])
        mask, status = res[k]
        assert status == 0
        assert np.array_equal(mask, _mask_of(ids, _tuples(tw[k]), n, wpb)), k
        assert np.array_equal(mask, _mask_of(ids, want[k + 1], n, wpb)), k
    assert res[0][0][1].any() and res[0][0][2].any()
    sset.close()
    twin.close()


@pytest.mark.parametrize("fault", ["length", "stream_id", "decreasing_offset"])
def test_bad_lengths_and_batches(hs, ref, fault):
    """A device length above pitch - 16, a stream id at or above nstreams, offsets that decrease: status 1, and so
    for the pass behind it; finish returns HS_INVALID, the streams stay where they were, and the passes enqueued
    again (mended) equal the reference."""
    lits, db = _compile(hs, "teddy8", seed=99)
    ids, wpb = _wpb(hs, db)
    nstreams = 9
    good = _random_batch(lits, 50, nstreams, seed=91)
    after = _random_batch(lits, 40, nstreams, seed=92)
    if fault == "length":
        writes = _random_batch(lits, nstreams, nstreams, seed=93).rows
        bad = ("bad_writes", (writes, [len(b) for b in writes[:4]] + [4096] + [len(b) for b in writes[5:]]))
        mended = ("writes", writes)
    else:
        b = _random_batch(lits, 50, nstreams, seed=95)
        mended = ("rows", b)
        offsets, sids = b.offsets.copy(), b.sids.copy()
        if fault == "stream_id":
            sids[17] = nstreams
        else:
            offsets[20] = offsets[21] + 5
        bad = Batch(b.rows, sids, seed=95)
        bad.offsets, bad.chars = offsets, b.chars
        bad = ("rows", bad)
    sset = hs.StreamSet(db, nstreams)
    scratch = _scratch(hs, db)
    _run(hs, sset, db, scratch, [("rows", good)], wpb)
    before = _state(sset)
    res = _run(hs, sset, db, scratch, [bad, ("rows", after)], wpb, rc=hs.HS_INVALID)
    assert [res[0][1], res[1][1]] == [1, 1]
    after_state = _state(sset)
    assert np.array_equal(before[0], after_state[0]) and np.array_equal(before[1], after_state[1])
    events = [("rows", good), mended, ("rows", after)]
    res = _run(hs, sset, db, scratch, events[1:], wpb)
    want = _want(ref, db, events)
    for k in (0, 1):
        mask, status = res[k]
        assert status == 0
        assert np.array_equal(mask, _mask_of(ids, want[k + 1], _nrows(sset, *events[k + 1]), wpb)), k
    sset.close()


def test_mask_record_and_reset_passes_interleaved(hs, ref):
    """200 passes on one set and one CUDA stream (9 under the emulator), one synchronisation: mask passes over rows
    and pitched writes, record passes of both kinds and resets, in a random order.  Every mask and every ordered pass
    equals the reference; empty batches and empty writes among them."""
    lits, db = _compile(hs, "teddy8", seed=21)
    ids, wpb = _wpb(hs, db)
    nstreams = 9
    npasses = 9 if EMU else 200
    rng = np.random.default_rng(21)
    events = []
    for k in range(npasses):
        u = rng.random()
        if u < 0.1:
            events.append(("reset", rng.choice(nstreams, size=int(rng.integers(1, 4)), replace=False).tolist()))
        elif u < 0.35:
            b = _random_batch(lits, nstreams, nstreams, seed=4000 + k, max_len=24)
            events.append(("writes", [r if rng.random() < 0.8 else b"" for r in b.rows]))
        elif u < 0.4:
            events.append(("rows", Batch([], [], lead=2, seed=k)))
        else:
            events.append(("rows", _random_batch(lits, 40, nstreams, seed=3000 + k, max_len=24)))
    if EMU:
        events[1:4] = [("reset", [0, 4]), ("writes", [b"abcdef"] * nstreams), ("rows", Batch([], [], seed=0))]
        events[7] = ("writes", [b"fedcba"[:s] for s in range(nstreams)])
    masked = lambda k: k % 2 == 0 or k % 5 == 0  # noqa: E731
    sset = hs.StreamSet(db, nstreams)
    scratch = _scratch(hs, db, ring=1 << 12)
    got = _run(hs, sset, db, scratch, events, wpb, masked=masked, cap=1 << 12)
    want = _want(ref, db, events)
    kinds = set()
    for k, (kind, x) in enumerate(events):
        if kind == "reset":
            continue
        if masked(k):
            mask, status = got[k]
            assert status == 0, k
            assert np.array_equal(mask, _mask_of(ids, want[k], _nrows(sset, kind, x), wpb)), k
        else:
            assert got[k] is not None and _tuples(got[k]) == want[k], k
        kinds.add((kind, masked(k)))
    assert kinds == {("rows", True), ("rows", False), ("writes", True), ("writes", False)}
    assert sum(1 for k, e in enumerate(events) if e[0] != "reset" and masked(k) and got[k][0].any()) > npasses // 4
    sset.close()


def test_record_readers_after_a_mask_pass(hs, ref):
    """after a mask pass of either kind, finish, fetch, the device ordering and the export serve no records"""
    lits, db = _compile(hs, "teddy8", seed=4)
    ids, wpb = _wpb(hs, db)
    nstreams = 8
    scratch = _scratch(hs, db)
    sset = hs.StreamSet(db, nstreams)
    b = _random_batch(lits, 40, nstreams, seed=8)
    writes = _random_batch(lits, nstreams, nstreams, seed=9).rows
    for ev in (("rows", b), ("writes", writes)):
        assert _ordinary(hs, sset, db, scratch, ev).size > 0
        s = _stream()
        sp = s.cuda_stream if s is not None else None
        keep, outs = _enqueue(hs, sset, db, scratch, [ev], s, wpb)
        out, cnt = _out(64)
        hs.order_matches_async(db, scratch, out, cnt, stream=sp)
        exp_out, exp_cnt = _out(64)
        assert hs.lib().hs_b200_export_records_async(scratch.ptr, C.c_void_p(hs._dev_ptr(exp_out)), 64,
                                                     C.c_void_p(hs._dev_ptr(exp_cnt)), C.c_void_p(sp or 0)) == 0
        res = _collect(hs, outs, wpb)
        got = _read(hs, out, cnt)
        assert got is not None and got.size == 0
        assert int((exp_cnt if EMU else exp_cnt.cpu().numpy()).view(np.uint64)[0]) == 0
        rc, n, _ = hs.scan_corpus_finish(scratch)
        assert rc == hs.HS_SUCCESS and n == 0
        assert hs.fetch_matches(db, scratch).size == 0
        assert res[0][1] == 0 and res[0][0].any()
        del keep
    sset.close()


def test_refusals(hs, ref):
    lits, db = _compile(hs, "teddy8", seed=4)
    ids, wpb = _wpb(hs, db, spare=0)
    scratch = _scratch(hs, db)
    nstreams = 8
    sset = hs.StreamSet(db, nstreams)
    chars = _dev(np.zeros(64, dtype=np.uint8))
    offs = _dev(np.arange(0, 40, 8, dtype=np.uint64))
    sids = _dev(np.zeros(4, dtype=np.uint32))
    writes = _dev(np.zeros(nstreams * 32, dtype=np.uint8))
    lens = _dev(np.zeros(nstreams, dtype=np.uint32))
    mask, status = _dev(np.zeros((nstreams, wpb), np.int32)), _dev(np.full(1, 7, np.int32))
    P = (lambda x: x.ctypes.data) if EMU else (lambda x: x.data_ptr())
    c, o, i, w, ln, m, st = (P(x) for x in (chars, offs, sids, writes, lens, mask, status))
    L = hs.lib()
    V = lambda x: C.c_void_p(x) if x else None  # noqa: E731
    other = hs.compile_lit_multi([b"qqqq"], ids=[1], mode=hs.HS_MODE_STREAM)
    other_scratch = _scratch(hs, other)

    def pitched(set_=sset.ptr, w_=w, pitch=32, ln_=ln, uni=0, scr=scratch.ptr, m_=m, wpb_=wpb, st_=st):
        return L.hs_b200_streams_scan_mask_async(set_, V(w_), pitch, V(ln_), uni, scr, V(m_), wpb_, V(st_), None)

    def rows(set_=sset.ptr, c_=c, nb=64, o_=o, i_=i, n=4, scr=scratch.ptr, m_=m, wpb_=wpb, st_=st):
        return L.hs_b200_streams_scan_rows_mask_async(set_, V(c_), nb, V(o_), V(i_), n, scr, V(m_), wpb_, V(st_),
                                                      None)

    bad = [pitched(set_=None), pitched(w_=None), pitched(w_=w + 8), pitched(pitch=24), pitched(pitch=40),
           pitched(ln_=None, uni=17), pitched(scr=None),
           rows(set_=None), rows(c_=None), rows(o_=None), rows(o_=o + 4), rows(i_=None), rows(i_=i + 2),
           rows(n=0xfffffff1), rows(scr=None), rows(scr=other_scratch.ptr)]
    for call in (pitched, rows):                              # the mask's own
        bad += [call(m_=None), call(m_=m + 2), call(st_=st + 1), call(wpb_=wpb - 1)]
    assert bad == [hs.HS_INVALID] * len(bad)
    peer, _ = _out(64)
    bases = (C.c_void_p * 1)(hs._dev_ptr(peer))
    assert L.hs_b200_set_peer_exchange(scratch.ptr, 1, 0, bases, 3, 0) == hs.HS_SUCCESS
    assert pitched() == hs.HS_ARCH_ERROR and rows() == hs.HS_ARCH_ERROR
    assert L.hs_b200_set_peer_exchange(scratch.ptr, 0, 0, None, 0, 0) == hs.HS_SUCCESS
    # accepted: a batch of no rows needs no chars, ids or mask; a NULL status; a uniform length
    assert L.hs_b200_streams_scan_rows_mask_async(sset.ptr, None, 0, V(o), None, 0, scratch.ptr, None, wpb, V(st),
                                                  None) == hs.HS_SUCCESS
    _sync()
    assert hs.scan_corpus_finish(scratch)[:2] == (hs.HS_SUCCESS, 0) and int(_host(status)[0]) == 0
    assert rows(st_=None) == hs.HS_SUCCESS and hs.scan_corpus_finish(scratch)[0] == hs.HS_SUCCESS
    assert pitched(ln_=None, uni=16) == hs.HS_SUCCESS and hs.scan_corpus_finish(scratch)[0] == hs.HS_SUCCESS
    sset.close()
