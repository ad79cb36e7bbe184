"""Stream sets fed from device memory (hs_b200_streams_scan_async / hs_b200_streams_reset_async): passes enqueued
back to back with no host wait, each ordered on the device (hs_b200_order_matches_async), equal the unmodified
reference stream runtime, one stream per stream, and, bit for bit, a second set fed the same writes from host
memory (hs_b200_streams_scan_collect).  Covers every literal first stage, the overflow protocol (no pass commits
after an overflow until finish; the passes enqueued again lose and double nothing), reset, writes that fill the
pitch, a buffer of exactly nstreams * pitch bytes, long-lived streams and the refusals.  Runs on the H100 and,
with numpy arrays as device memory, on the SIMT emulator."""
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
        return None, None
    import torch
    torch.cuda.synchronize()                       # the tensors above were filled on torch's stream
    s = torch.cuda.Stream()
    return s, s.cuda_stream


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
    """under the emulator a small ring, as the emulated shapes are: the ordering kernels' grids follow the
    ring's capacity"""
    if not EMU:
        return hs.Scratch(db)
    hs.set_runtime_option("initial_ring", ring)
    try:
        return hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)


def _compile(hs, name, seed):
    n, min_len, opts, avx2 = ENGINES[name]
    lits, flags, ids = synth.literal_set(n, min_len=min_len, max_len=8, seed=seed, caseless_frac=0.2,
                                         alphabet=b"abcdef")
    plat = None
    if avx2:
        plat = C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0))
    db = hs.compile_lit_multi(lits, flags, ids, mode=hs.HS_MODE_STREAM, platform=plat)
    if avx2:
        assert 3 <= db.info().engine_id <= 10
    return lits, db


def _round(lits, lens, pitch, seed, tail_lit=None):
    """one write per stream at i * pitch + 16 of a buffer whose headroom and tails are random bytes; returns the
    buffer and the host form of the same writes (data, offsets)"""
    rng = np.random.default_rng(seed)
    n = lens.size
    data, off, _ = synth.ragged_corpus([int(x) for x in lens], lits, seed=seed, plant_per_kb=30, align=1,
                                       alphabet=ALPHABET)
    if tail_lit is not None:   # the literal again on the last bytes of every write long enough
        for i in range(n):
            if lens[i] >= len(tail_lit):
                e = int(off[i]) + int(lens[i])
                data[e - len(tail_lit):e] = np.frombuffer(tail_lit, dtype=np.uint8)
    buf = rng.integers(0, 256, size=n * pitch, dtype=np.uint8)
    for i in range(n):
        buf[i * pitch + 16:i * pitch + 16 + int(lens[i])] = data[int(off[i]):int(off[i]) + int(lens[i])]
    return buf, data, off


def _want(ref, db, rounds, s, first=0):
    """the reference stream of stream s over rounds[first:], as (id, round, to)"""
    pieces = [d[int(o[s]):int(o[s]) + int(ln[s])] for (_, d, o, ln) in rounds[first:]]
    cat = np.concatenate(pieces) if sum(p.size for p in pieces) else np.zeros(0, np.uint8)
    wl = np.array([p.size for p in pieces], dtype=np.uint32)
    recs, err = ref.stream_collect(db.ptr, cat, wl)
    assert err == 0
    return sorted((int(r["id"]), int(r["block"]) + first, int(r["to"])) for r in recs)


def _mine(got, s, rounds):
    return sorted((int(r["id"]), k, int(r["to"])) for k in rounds for r in got[k][got[k]["block"] == s])


def _run_device(hs, sset, db, scratch, rounds, stream, uniform_of=None, cap=1 << 19):
    """enqueue every round and its ordering back to back on `stream`, one synchronisation at the end"""
    keep, outs = [], []
    for k, (buf, _, _, ln) in enumerate(rounds):
        d_buf = _dev(buf)
        uni = uniform_of(k) if uniform_of else None
        lens = int(uni) if uni is not None else _dev(ln)
        keep += [d_buf, lens]
        outs.append(_out(cap))
    s, sp = _stream()
    for k in range(len(rounds)):
        sset.scan_async(keep[2 * k], rounds[k][0].size // sset.n, keep[2 * k + 1], scratch, stream=sp)
        hs.order_matches_async(db, scratch, outs[k][0], outs[k][1], stream=sp)
    _sync()
    rc, _, _ = hs.scan_corpus_finish(scratch)
    assert rc == hs.HS_SUCCESS
    return [_read(hs, o, c) for (o, c) in outs]


@pytest.mark.parametrize("name,nstreams,wlen", [(name, 257, 200) for name in ENGINES] +
                         [("teddy8", 4096, 64), ("gram4", 4096, 64)])
def test_device_passes_equal_reference_and_host_path(hs, ref, name, nstreams, wlen):
    if EMU:
        if nstreams > 257:
            pytest.skip("the emulator runs the 257-stream shapes")
        wlen = 32                                # the same shape, shorter writes
    n, _, opts, _ = ENGINES[name]
    for k, v in opts.items():
        hs.set_runtime_option(k, v)
    try:
        lits, db = _compile(hs, name, seed=n + nstreams)
        scratch = _scratch(hs, db)
        pitch = 16 + (wlen + 15) // 16 * 16
        rng = np.random.default_rng(nstreams + n)
        rounds = []
        for k in range(5):
            if k % 2:      # ragged, a tenth of the streams without a write, lengths in device memory
                ln = rng.integers(0, pitch - 16 + 1, size=nstreams).astype(np.uint32)
                ln[rng.random(nstreams) < 0.1] = 0
            else:
                ln = np.full(nstreams, wlen, dtype=np.uint32)
            buf, data, off = _round(lits, ln, pitch, seed=1000 * k + nstreams + n)
            rounds.append((buf, data, off, ln))
        dev = hs.StreamSet(db, nstreams)
        got = _run_device(hs, dev, db, scratch, rounds, None,
                          uniform_of=lambda k: wlen if k % 2 == 0 else None)
        dev.close()
        host = hs.StreamSet(db, nstreams)
        hscratch = _scratch(hs, db)
        for k, (_, data, off, ln) in enumerate(rounds):
            want = host.scan(data, off, ln, hscratch)
            assert got[k] is not None and np.array_equal(got[k], want), k
        host.close()
        assert sum(g.size for g in got) > nstreams
        for s in rng.choice(nstreams, size=40, replace=False).tolist() + [0, nstreams - 1]:
            assert _mine(got, s, range(len(rounds))) == _want(ref, db, rounds, s), s
    finally:
        hs.set_runtime_option("gram", 1)


def _text_round(texts, pitch, seed):
    """writes given as bytes per stream, in a buffer of random bytes"""
    ln = np.array([len(t) for t in texts], dtype=np.uint32)
    data = np.frombuffer(b"".join(texts), dtype=np.uint8).copy()
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    buf = np.random.default_rng(seed).integers(0, 256, size=len(texts) * pitch, dtype=np.uint8)
    for i, t in enumerate(texts):
        buf[i * pitch + 16:i * pitch + 16 + len(t)] = np.frombuffer(t, dtype=np.uint8)
    return buf, data, off, ln


def test_overflow_marks_the_set_until_finish(hs, ref):
    """A 16-record ring.  Pass 1 overflows it (16 candidates, 1 024 records); passes 2 and 3 and a reset
    enqueued behind it would fit, so only the mark holds them back: every ordering from pass 1 on reports the
    overflow and the reset commits nothing.  One finish grows the ring for the largest count, and the passes and
    the reset enqueued again from pass 1 deliver exactly the reference's matches -- the match across the pass
    0 / pass 1 boundary of the reset stream included -- and what the host path delivers."""
    db = hs.compile_lit_multi([b"abcd"] * 64 + [b"wxyz"], ids=list(range(64)) + [100], mode=hs.HS_MODE_STREAM)
    nstreams, wlen = 16, 64
    pitch = 16 + wlen
    fill = lambda n: b"." * n  # noqa: E731
    texts = [[fill(wlen) for _ in range(nstreams)] for _ in range(4)]
    for s in (1, 2):                    # "wx" | "yz" across the boundaries of passes 0, 1 and 2
        texts[0][s] = fill(wlen - 2) + b"wx"
        texts[1][s] = b"yz" + fill(wlen - 4) + b"wx"
        texts[2][s] = b"yz" + fill(wlen - 2)
    texts[0][3] = fill(10) + b"wxyz" + fill(wlen - 14)
    for s in range(nstreams):           # one "abcd" per stream: 64 records each
        t = texts[1][s]
        texts[1][s] = t[:20] + b"abcd" + t[24:]
    texts[3][4] = fill(30) + b"wxyz" + fill(wlen - 34)
    rounds = [_text_round(t, pitch, seed=k) for k, t in enumerate(texts)]
    reset = np.array([1, nstreams + 3], dtype=np.uint32)
    hs.set_runtime_option("initial_ring", 16)
    try:
        scratch = hs.Scratch(db)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)
    sset = hs.StreamSet(db, nstreams)
    bufs = [(_dev(b), _dev(ln)) for (b, _, _, ln) in rounds]
    d_reset = _dev(reset)
    got, first, tries = [None] * 4, 0, 0
    while first < 4:
        tries += 1
        assert tries <= 2                # one finish is enough
        outs = [_out(1 << 12) for _ in range(first, 4)]
        s, sp = _stream()
        for k in range(first, 4):
            if k == 2:
                sset.reset_async(d_reset, stream=sp)
            sset.scan_async(bufs[k][0], pitch, bufs[k][1], scratch, stream=sp)
            hs.order_matches_async(db, scratch, outs[k - first][0], outs[k - first][1], stream=sp)
        _sync()
        res = [_read(hs, o, c) for (o, c) in outs]
        rc, _, _ = hs.scan_corpus_finish(scratch)
        if tries == 1:
            assert rc == hs.HS_INSUFFICIENT_SPACE
            assert res[0] is not None and all(r is None for r in res[1:])
        ok = 0
        while ok < len(res) and res[ok] is not None:
            got[first + ok] = res[ok]
            ok += 1
        assert all(r is None for r in res[ok:])      # nothing after an overflow is delivered
        assert (rc == hs.HS_SUCCESS) == (ok == len(res))
        first += ok
    sset.close()
    assert got[1].size == nstreams * 64 + 2 and got[2].size <= 16 and got[3].size <= 16
    host = hs.StreamSet(db, nstreams)
    hscratch = _scratch(hs, db)
    for k, (_, data, off, ln) in enumerate(rounds):
        if k == 2:
            host.reset_async(d_reset, stream=None)
            _sync()
        assert np.array_equal(got[k], host.scan(data, off, ln, hscratch)), k
    host.close()
    for s in range(nstreams):
        want = _want(ref, db, rounds, s)
        if s == 1:
            want = _want(ref, db, rounds[:2], s) + _want(ref, db, rounds, s, first=2)
        assert _mine(got, s, range(4)) == sorted(want), s
    assert (100, 1, wlen + 2) in _mine(got, 1, range(4))   # "wx" | "yz" across passes 0 and 1 of stream 1


def test_fetch_and_export_serve_a_pass(hs, ref):
    """hs_b200_fetch_matches and hs_b200_export_records_async after a pass: the delivered matches equal the host
    path's, and the exported raw records, ordered and deduplicated, equal them too."""
    lits, db = _compile(hs, "teddy8", seed=12)
    scratch = _scratch(hs, db)
    nstreams, wlen = 257, 48
    pitch = 16 + wlen
    rng = np.random.default_rng(12)
    rounds = []
    for k in range(2):
        ln = rng.integers(0, wlen + 1, size=nstreams).astype(np.uint32)
        buf, data, off = _round(lits, ln, pitch, seed=70 + k)
        rounds.append((buf, data, off, ln))
    sset = hs.StreamSet(db, nstreams)
    host = hs.StreamSet(db, nstreams)
    hscratch = _scratch(hs, db)
    L = hs.lib()
    for buf, data, off, ln in rounds:
        d_buf, d_ln = _dev(buf), _dev(ln)
        cap = 1 << 14
        recs, cnt = _out(cap)
        s, sp = _stream()
        sset.scan_async(d_buf, pitch, d_ln, scratch, stream=sp)
        assert L.hs_b200_export_records_async(scratch.ptr, C.c_void_p(hs._dev_ptr(recs)), cap,
                                              C.c_void_p(hs._dev_ptr(cnt)), C.c_void_p(sp or 0)) == hs.HS_SUCCESS
        _sync()
        rc, n, _ = hs.scan_corpus_finish(scratch)
        assert rc == hs.HS_SUCCESS and 0 < n <= cap
        want = host.scan(data, off, ln, hscratch)
        assert np.array_equal(hs.fetch_matches(db, scratch), want)
        raw = recs if EMU else recs.cpu().numpy()
        c = int(cnt[0]) if EMU else int(cnt.cpu().numpy().view(np.uint64)[0])
        assert c == n
        raw = np.sort(raw.view(hs.MATCH_DTYPE)[:c], order=["block", "to", "id"])
        keep = np.ones(raw.size, dtype=bool)
        keep[1:] = raw[1:] != raw[:-1]
        assert np.array_equal(raw[keep], want)
    sset.close()
    host.close()


def test_reset_ends_the_listed_flows(hs, ref):
    """After round 1 a subset of the streams is reset (out-of-range indices among the list are ignored): they
    start afresh while the others carry on; after round 2 every stream is reset (NULL list)."""
    lits, db = _compile(hs, "teddy8", seed=3)
    scratch = _scratch(hs, db)
    nstreams, wlen = 257, 48
    pitch = 16 + wlen
    rng = np.random.default_rng(17)
    rounds = []
    for k in range(4):
        ln = rng.integers(0, wlen + 1, size=nstreams).astype(np.uint32)
        buf, data, off = _round(lits, ln, pitch, seed=50 + k)
        rounds.append((buf, data, off, ln))
    subset = np.array(sorted(rng.choice(nstreams, size=60, replace=False).tolist()) + [nstreams, 2**32 - 1],
                      dtype=np.uint32)
    sset = hs.StreamSet(db, nstreams)
    bufs = [(_dev(b), _dev(ln)) for (b, _, _, ln) in rounds]
    d_subset = _dev(subset)
    outs = [_out(1 << 15) for _ in range(4)]
    s, sp = _stream()
    for k in range(4):
        if k == 2:
            sset.reset_async(d_subset, stream=sp)
        if k == 3:
            sset.reset_async(None, stream=sp)
        sset.scan_async(bufs[k][0], pitch, bufs[k][1], scratch, stream=sp)
        hs.order_matches_async(db, scratch, outs[k][0], outs[k][1], stream=sp)
    _sync()
    assert hs.scan_corpus_finish(scratch)[0] == hs.HS_SUCCESS
    got = [_read(hs, o, c) for (o, c) in outs]
    sset.close()
    reset = set(subset.tolist())
    for s in range(nstreams):
        if s in reset:
            want = _want(ref, db, rounds[:2], s) + _want(ref, db, rounds[:3], s, first=2)
        else:
            want = _want(ref, db, rounds[:3], s)
        want += _want(ref, db, rounds, s, first=3)
        assert _mine(got, s, range(4)) == sorted(want), s


def test_writes_that_fill_the_buffer(hs, ref):
    """Writes that fill the pitch exactly, a literal on the last byte of each, in a buffer of exactly
    nstreams * pitch bytes: the pass reads and writes nothing outside it (on the GPU a torch tensor of that
    size; under the emulator an array of that size)."""
    lits, db = _compile(hs, "fdr", seed=9)
    scratch = _scratch(hs, db)
    tail = max(lits, key=len)
    for nstreams, pitch in ((1, 32), (5, 48), (16, 272) if EMU else (300, 1040)):
        rounds = []
        for k in range(3):
            ln = np.full(nstreams, pitch - 16, dtype=np.uint32)
            if k == 1:
                ln[::3] = 0
            buf, data, off = _round(lits, ln, pitch, seed=7 * k + pitch, tail_lit=tail)
            rounds.append((buf, data, off, ln))
        sset = hs.StreamSet(db, nstreams)
        got = _run_device(hs, sset, db, scratch, rounds, None)
        sset.close()
        for s in range(nstreams):
            mine = _mine(got, s, range(3))
            assert mine == _want(ref, db, rounds, s), (nstreams, s)
            if nstreams > 1:
                assert any(to == (k + 1) * (pitch - 16) for (_, k, to) in mine if k != 1)


def test_offsets_far_beyond_one_write(hs, ref):
    """200 passes (12 under the emulator): the stream offsets grow far past any write's length."""
    lits, db = _compile(hs, "teddy8", seed=21)
    scratch = _scratch(hs, db, ring=1 << 12)
    nstreams, wlen = 9, 64
    pitch = 16 + wlen
    rng = np.random.default_rng(5)
    rounds = []
    npasses = 12 if EMU else 200
    for k in range(npasses):
        ln = rng.integers(wlen // 2, wlen + 1, size=nstreams).astype(np.uint32)
        buf, data, off = _round(lits, ln, pitch, seed=3000 + k)
        rounds.append((buf, data, off, ln))
    sset = hs.StreamSet(db, nstreams)
    got = _run_device(hs, sset, db, scratch, rounds, None, cap=1 << 12)
    sset.close()
    for s in range(nstreams):
        mine = _mine(got, s, range(npasses))
        assert mine == _want(ref, db, rounds, s), s
        assert max(to for (_, _, to) in mine) > npasses // 2 * wlen


def test_refusals(hs, ref):
    lits, db = _compile(hs, "teddy8", seed=4)
    scratch = _scratch(hs, db)
    nstreams, pitch = 8, 48
    sset = hs.StreamSet(db, nstreams)
    buf = _dev(np.zeros(nstreams * pitch + 16, dtype=np.uint8))
    ln = _dev(np.full(nstreams, 8, dtype=np.uint32))
    p = int(buf.ctypes.data if EMU else buf.data_ptr())
    L = hs.lib()
    V = C.c_void_p
    bad = [
        (None, p, pitch, ln, 0, scratch.ptr),          # no set
        (sset.ptr, None, pitch, ln, 0, scratch.ptr),   # no buffer
        (sset.ptr, p + 8, pitch, ln, 0, scratch.ptr),  # misaligned buffer
        (sset.ptr, p, 16, ln, 0, scratch.ptr),         # pitch below 32
        (sset.ptr, p, 40, ln, 0, scratch.ptr),         # pitch not a multiple of 16
        (sset.ptr, p, pitch, None, pitch - 15, scratch.ptr),   # uniform length above pitch - 16
        (sset.ptr, p, pitch, ln, 0, None),             # no scratch
    ]
    for set_, b, pt, lens, uni, scr in bad:
        d_len = None if lens is None else (lens.ctypes.data if EMU else lens.data_ptr())
        assert L.hs_b200_streams_scan_async(set_, V(b) if b else None, pt, V(d_len) if d_len else None, uni,
                                            scr, None) == hs.HS_INVALID
    assert L.hs_b200_streams_reset_async(None, None, 0, None) == hs.HS_INVALID
    # a device length above pitch - 16: the pass delivers nothing, the streams stay, finish says HS_INVALID
    good = np.full(nstreams, pitch - 16, dtype=np.uint32)
    over = good.copy()
    over[3] = pitch - 15
    rounds = []
    for k in range(2):
        b, data, off = _round(lits, good, pitch, seed=90 + k)
        rounds.append((b, data, off, good))
    d_bad = [(_dev(rounds[0][0]), _dev(over)), (_dev(rounds[1][0]), _dev(good))]
    outs = [_out(1024) for _ in range(2)]
    s, sp = _stream()
    for k in range(2):
        sset.scan_async(d_bad[k][0], pitch, d_bad[k][1], scratch, stream=sp)
        hs.order_matches_async(db, scratch, outs[k][0], outs[k][1], stream=sp)
    _sync()
    assert [_read(hs, o, c) for (o, c) in outs] == [None, None]
    assert hs.scan_corpus_finish(scratch)[0] == hs.HS_INVALID
    # the mark is gone and the streams are where they were: the same rounds with good lengths
    got = _run_device(hs, sset, db, scratch, rounds, None)
    sset.close()
    for st in range(nstreams):
        assert _mine(got, st, range(2)) == _want(ref, db, rounds, st), st
