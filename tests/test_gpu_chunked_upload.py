"""Host-buffer scans whose corpus reaches the device in several chunk_mb pieces.

hs_scan, hs_b200_scan_blocks / _collect and hs_scan_stream copy their corpus to the device
in chunk_mb pieces and launch the tiles of piece i as soon as piece i has arrived: one
scan-and-confirm range per piece, each launching only the tiles that end 16 bytes before
the copied prefix.  A caller layout whose block starts are 16-byte aligned is copied as it
lies; any other is packed through two alternating pinned staging buffers, and a block that
straddles a piece edge travels whole with the piece it starts in.

Every test here sets chunk_mb=1 and checks the scan twice: against the definition
(oracle/brute.py, or a closed form for the floods), and against scan_corpus over
Corpus.upload of the same blocks, which is resident and never chunked.  For literal
databases each range is two launches; the launch count shows how many ranges ran."""
import functools

import numpy as np
import pytest

from hyperscan_b200 import synth
import oracle.brute as brute
import oracle.ref as reference

pytestmark = pytest.mark.gpu

MiB = 1 << 20
F_CASELESS, F_SINGLE = 1, 8
OPTION_DEFAULTS = {"chunk_mb": 128, "tile_bytes": 1024, "initial_ring": 1 << 20, "gram": 1}


@pytest.fixture
def opts(hs):
    """chunk_mb=1 (and whatever else the test sets through the returned function); every
    runtime option is back at its default afterwards."""
    def set_options(**kw):
        for k, v in kw.items():
            hs.set_runtime_option(k, v)
    set_options(chunk_mb=1)
    yield set_options
    set_options(**OPTION_DEFAULTS)


def _up16(x):
    return (x + 15) // 16 * 16


def _chunks(nbytes):
    return -(-nbytes // MiB)


def _device_layout(off, ln):
    """Where the library puts each block on the device and how long the corpus is there:
    the caller's layout as it lies when every start is 16-byte aligned relative to the
    first and the blocks ascend without overlap, else packed back to back at 16-byte
    aligned starts (a zero-length block takes 16 bytes)."""
    off = np.asarray(off, dtype=np.int64)
    ln = np.asarray(ln, dtype=np.int64)
    rel = off - off[0]
    if np.all(rel % 16 == 0) and np.all(rel[1:] >= rel[:-1] + ln[:-1]):
        dev = rel
    else:
        step = _up16(ln) + 16 * (ln == 0)
        dev = np.concatenate([[0], np.cumsum(step)[:-1]])
    return dev, int(dev[-1] + ln[-1])


def _sorted(recs):
    return np.sort(np.asarray(recs), order=["block", "to", "id"])


def _ranges_ran(hs, n0, total):
    """The last host scan ran one range per chunk: at least 2 launches per chunk.  Every
    corpus here has 4 chunks or more, so 8 launches or more, which three unchunked passes
    (6 launches) never reach."""
    assert _chunks(total) >= 4, total
    launches = hs.launch_count() - n0
    assert launches >= 2 * _chunks(total), (launches, _chunks(total))


def _check(hs, db, scratch, lits, flags, ids, data, off, ln, want=None):
    """Host scan == definition == resident-corpus scan, with one range per chunk."""
    if want is None:
        want = brute.scan_blocks(lits, flags, ids, data, off, ln)
    _, total = _device_layout(off, ln)
    n0 = hs.launch_count()
    got = hs.scan_blocks(db, data, off, ln, scratch)
    _ranges_ran(hs, n0, total)
    assert got.size == want.size, (got.size, want.size)
    assert np.array_equal(got, want)
    corpus = hs.Corpus.upload(data, off, ln)
    try:
        assert np.array_equal(_sorted(hs.scan_corpus(db, corpus, scratch)), want)
    finally:
        corpus.free()
    return want


# ---- corpora whose blocks cross the chunk edges ------------------------------------------

SIZES = [0, 1, 3, 15, 16, 17, 100, 511, 1000, 1025, 4096, 9000, 30000]
TOTAL = int(4.4 * MiB)          # 5 chunks


def _edge_layout(rng, packed):
    """Device starts and lengths of blocks over TOTAL bytes: at the first chunk edge a block
    ending 5 bytes short of it, then two zero-length blocks; from just before the second
    edge one block longer than a chunk (it also crosses the third); elsewhere blocks of
    SIZES, some straddling an edge.  packed: starts follow the packing rule of
    _device_layout; else starts are 16-byte aligned with 0-32 byte gaps."""
    starts, lens = [], []
    pos = 0

    def add(n, gap=0):
        nonlocal pos
        starts.append(pos)
        lens.append(n)
        pos = _up16(pos + n) + (16 if packed and n == 0 else 0) + gap

    done = set()
    while pos < TOTAL:
        edge = (pos // MiB + 1) * MiB
        n = int(rng.choice(SIZES))
        if pos + n + 16 >= edge and edge not in done:
            done.add(edge)
            if edge == MiB:
                if pos <= edge - 5:
                    add(edge - 5 - pos)
                add(0)
                add(0)
            elif edge == 2 * MiB:
                add(MiB + MiB // 4 + 3)
            else:
                add(max(n, 40))
            continue
        add(n, 0 if packed else 16 * int(rng.integers(0, 3)))
    return np.array(starts, dtype=np.int64), np.array(lens, dtype=np.int64)


def _plant_near(data, off, ln, dev, lits, positions, rng):
    """Write literals ending within 16 bytes of each device position, inside whichever block
    holds the spot, without overwriting each other."""
    taken = []
    for i, p in enumerate(positions):
        for d in ((-16, -1, 15), (-15, 0, 16), (-12, 2, 9))[i % 3]:
            lit = lits[int(rng.integers(len(lits)))]
            end = int(p) + d
            start = end - len(lit)
            b = int(np.searchsorted(dev, start, side="right")) - 1
            if b < 0 or start < dev[b] or end > dev[b] + ln[b] or any(s < end and start < e for s, e in taken):
                continue
            taken.append((start, end))
            h = int(off[b]) + start - int(dev[b])
            data[h:h + len(lit)] = np.frombuffer(lit, dtype=np.uint8)


def _edge_positions(dev, total):
    """Every chunk edge, and where the packed layout's pieces really end (the start of the
    first block at or past the edge)."""
    edges = [k * MiB for k in range(1, _chunks(total))]
    covered = [int(dev[np.searchsorted(dev, e)]) for e in edges if np.searchsorted(dev, e) < dev.size]
    return sorted(set(edges + covered))


LAYOUTS = ["pitch", "ragged", "align1", "align3"]


def _corpus(layout, lits, seed, alphabet):
    """(data, offsets, lengths) of TOTAL-ish bytes in one of LAYOUTS, with literals planted
    at random and near every chunk edge."""
    rng = np.random.default_rng(seed)
    al = np.frombuffer(alphabet, dtype=np.uint8)
    if layout == "pitch":                                   # the direct, hsbench-shaped path
        off = np.arange(TOTAL // 4000, dtype=np.int64) * 4000
        ln = np.full(off.size, 3995, dtype=np.int64)
        data = al[rng.integers(0, al.size, size=off.size * 4000)]
    else:
        packed = layout != "ragged"
        dev, ln = _edge_layout(rng, packed)
        if packed:                                          # unaligned starts: the staged, repacked path
            align = int(layout[5:])
            off, pos = [], 0
            for n in ln:
                pos = (pos + align - 1) // align * align
                off.append(pos)
                pos += int(n)
            off = np.array(off, dtype=np.int64)
        else:                                               # aligned starts, the first not at 0
            off = dev + 48
        data = al[rng.integers(0, al.size, size=int(off[-1] + ln[-1]) + 40)]
        assert np.array_equal(_device_layout(off, ln)[0], dev)
        assert (not packed) == bool(np.all((off - off[0]) % 16 == 0))
    dev, total = _device_layout(off, ln)
    for b in range(off.size):                               # random plants
        for _ in range(rng.poisson(ln[b] / 1024.0 * 2.0)):
            lit = lits[int(rng.integers(len(lits)))]
            if len(lit) <= ln[b]:
                s = int(off[b]) + int(rng.integers(0, ln[b] - len(lit) + 1))
                data[s:s + len(lit)] = np.frombuffer(lit, dtype=np.uint8)
    _plant_near(data, off, ln, dev, lits, _edge_positions(dev, total), rng)
    return data, off.astype(np.uint64), ln.astype(np.uint32)


def _avx2(hs):
    import ctypes as C
    return C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0))


# name: (literal_set arguments, runtime options, AVX2 platform)
ENGINES = {
    "noodle": (dict(n=1, min_len=2, max_len=12, seed=71), {}, False),
    "teddy-30": (dict(n=30, min_len=2, max_len=12, seed=72), {}, False),
    "fdr-300": (dict(n=300, min_len=4, max_len=12, seed=73), {}, False),
    "fdr-1000": (dict(n=1000, min_len=4, max_len=12, seed=74), {}, False),
    "class-4-gram": (dict(n=400, min_len=4, max_len=10, seed=75), {"gram": 2}, False),
    "fat-teddy": (dict(n=64, min_len=3, max_len=12, seed=76), {}, True),
}


def _literals(name):
    a = ENGINES[name][0]
    return synth.literal_set(a["n"], min_len=a["min_len"], max_len=a["max_len"], seed=a["seed"],
                             caseless_frac=0.2, alphabet=b"abcdefgh")


@functools.lru_cache(maxsize=None)
def _case(name, layout):
    """Literals, corpus and the definition's records of one engine and layout (shared by
    the tile sizes)."""
    lits, flags, ids = _literals(name)
    data, off, ln = _corpus(layout, lits, seed=len(name) * 10 + LAYOUTS.index(layout), alphabet=b"abcdefghABCDxy")
    want = brute.scan_blocks(lits, flags, ids, data, off, ln)
    return lits, flags, ids, data, off, ln, want


@pytest.mark.parametrize("tile", [1024, 512, 8192])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name", list(ENGINES))
def test_layouts_across_chunk_edges(hs, opts, name, layout, tile):
    """Noodle, Teddy, FDR, the class 4-gram stage and fat Teddy over 5 chunks of uniform,
    ragged-aligned and repacked layouts, with the tile edges falling differently against the
    chunk edges."""
    _, options, avx2 = ENGINES[name]
    if avx2 and reference.best_isa() == "corei7":
        pytest.skip("the reference build on this host has no fat Teddy")
    lits, flags, ids, data, off, ln, want = _case(name, layout)
    opts(tile_bytes=tile, **options)
    db = hs.compile_lit_multi(lits, flags, ids, platform=_avx2(hs) if avx2 else None)
    if avx2:
        assert 3 <= db.info().engine_id <= 10, db.info().engine_id
    scratch = hs.Scratch(db)
    _check(hs, db, scratch, lits, flags, ids, data, off, ln, want)
    assert want.size > 1000
    scratch.free()


# ---- record ring and candidate list overflowing during a chunked upload ------------------

FLOOD = [b"a" * k for k in range(1, 13)]           # ~12 records per byte of a flood of `a`


def _flood(layout):
    """48 blocks of `a`, 3 MiB in all: 64 KiB at a 64 KiB pitch, or 65531 bytes back to back
    (repacked)."""
    L = 65536 if layout == "pitch" else 65531
    off = np.arange(48, dtype=np.uint64) * np.uint64(L)
    data = np.full(48 * L, ord("a"), dtype=np.uint8)
    return data, off, np.full(48, L, dtype=np.uint32), L


def _flood_records(L):
    """One block's records of FLOOD over L bytes of `a`, ordered by (to, id): every `to`
    reports ids 1..min(to, 12)."""
    per = np.minimum(np.arange(1, L + 1), len(FLOOD))
    to = np.repeat(np.arange(1, L + 1), per)
    first = np.repeat(np.cumsum(per) - per, per)
    return to, np.arange(to.size) - first + 1


@pytest.mark.parametrize("layout", ["pitch", "packed"])
def test_flood_overflows_ring_during_chunked_upload(hs, opts, real_gpu, layout):
    """3 MiB of `a` against `a` .. `a` x 12 from a 16-record ring: the candidate list
    overflows in every range of the chunked first pass, and the rescans overflow the ring
    again until it holds all 37 M records.  The scan still returns every record, collected
    and as a count.  One pass over 3 chunks is 6 launches, as many as three unchunked
    passes: a rescan after it makes 8 or more."""
    opts(initial_ring=16)
    data, off, ln, L = _flood(layout)
    expect = sum(L - len(x) + 1 for x in FLOOD) * off.size
    db = hs.compile_lit_multi(FLOOD, [0] * len(FLOOD), list(range(1, len(FLOOD) + 1)))
    scratch = hs.Scratch(db)
    _, total = _device_layout(off, ln)
    out = np.zeros(expect, dtype=hs.MATCH_DTYPE)
    n0 = hs.launch_count()
    n = hs.scan_blocks_collect(db, data, off, ln, scratch, out)
    launches = hs.launch_count() - n0
    assert _chunks(total) == 3
    assert launches >= 2 * _chunks(total) + 2, launches    # every chunk's range, then a rescan
    assert n == expect
    to, ids = _flood_records(L)
    assert np.array_equal(out["block"], np.repeat(np.arange(off.size, dtype=np.uint32), to.size))
    assert np.array_equal(out["to"].reshape(off.size, -1), np.broadcast_to(to, (off.size, to.size)))
    assert np.array_equal(out["id"].reshape(off.size, -1), np.broadcast_to(ids, (off.size, to.size)))
    del out
    scratch.free()
    scratch = hs.Scratch(db)                        # a fresh 16-record ring for the count
    n0 = hs.launch_count()
    assert hs.scan_blocks(db, data, off, ln, scratch, collect=False) == expect
    assert hs.launch_count() - n0 >= 2 * _chunks(total) + 2
    corpus = hs.Corpus.upload(data, off, ln)
    try:
        assert hs.scan_corpus(db, corpus, scratch, fetch=False) == expect
    finally:
        corpus.free()
    scratch.free()


@pytest.mark.parametrize("layout", ["pitch", "align3"])
def test_mixed_literals_small_ring_across_chunks(hs, opts, layout):
    """A Teddy set with caseless and single-match literals from a 16-record ring: every
    range of the first pass overflows, and the rescan's records equal the definition's."""
    opts(initial_ring=16)
    lits, flags, ids = synth.literal_set(24, min_len=2, max_len=9, seed=81, caseless_frac=0.3,
                                         singlematch_frac=0.2, alphabet=b"abcdefgh")
    data, off, ln = _corpus(layout, lits, seed=82, alphabet=b"abcdefghABxy")
    db = hs.compile_lit_multi(lits, flags, ids)
    scratch = hs.Scratch(db)
    want = _check(hs, db, scratch, lits, flags, ids, data, off, ln)
    assert want.size > 10000
    scratch.free()


# ---- bytes a chunked upload never writes -------------------------------------------------

# the literal API takes a literal that begins with NUL for an empty one, as the reference
# does: every NUL here follows another byte
NUL_LITS = [b"ab\x00", b"b\x00\x00", b"ab", b"x\x00\x00a"]
NUL_IDS = [1, 2, 3, 4]
TAILS = [b"ab", b"b\x00", b"x\x00\x00", b"a"]


def _nul_blocks(seed, total, packed):
    """Blocks over about `total` device bytes over the alphabet `ab\\0xy`, each ending in one of
    TAILS, so that a match of a NUL literal past the tail would cross the block's end.
    Not packed: 1000-byte blocks at a 1008-byte pitch with NUL bytes between them.  Packed:
    ragged blocks back to back from host offset 1; the last block of every chunk ends in `ab`
    at a device position 2 past a multiple of 4, before up to 14 bytes of padding."""
    rng = np.random.default_rng(seed)
    al = np.frombuffer(b"ab\x00xy", dtype=np.uint8)
    if not packed:
        off = np.arange(total // 1008, dtype=np.int64) * 1008
        ln = np.full(off.size, 1000, dtype=np.int64)
        data = np.zeros(off.size * 1008, dtype=np.uint8)
        for o in off:
            data[o:o + 1000] = al[rng.integers(0, al.size, size=1000)]
        tails = [TAILS[b % len(TAILS)] for b in range(off.size)]
    else:
        starts, lens, tails, pos = [], [], [], 0
        while pos < total:
            n = int(rng.choice([1, 2, 5, 17, 100, 1000, 3001, 20001]))
            edge = (pos // MiB + 1) * MiB
            tail = TAILS[len(lens) % len(TAILS)]
            if pos + n >= edge:                         # the last block of this chunk
                n = max(n, edge - pos + 8)
                n += (2 - (pos + n)) % 4
                tail = b"ab"
            starts.append(pos)
            lens.append(n)
            tails.append(tail)
            pos = _up16(pos + n)
        ln = np.array(lens, dtype=np.int64)
        off = np.concatenate([[0], np.cumsum(ln)[:-1]]) + 1
        data = al[rng.integers(0, al.size, size=int(off[-1] + ln[-1]) + 32)]
        assert np.array_equal(_device_layout(off, ln)[0], starts)
    for o, n, t in zip(off, ln, tails):
        t = np.frombuffer(t, dtype=np.uint8)[-int(n):]
        data[o + n - t.size:o + n] = t
    return data, off.astype(np.uint64), ln.astype(np.uint32)


@pytest.mark.parametrize("packed", [False, True], ids=["pitch-nul-gaps", "repacked-zero-padding"])
def test_nul_literals_stop_at_block_ends(hs, opts, packed):
    """NUL literals over blocks that end in `ab`, `b\\0` or `x\\0\\0`, followed by NUL bytes
    between the blocks (aligned layout) or by the zero padding of the repacked one."""
    data, off, ln = _nul_blocks(91, int(4.2 * MiB), packed)
    db = hs.compile_lit_multi(NUL_LITS, [0] * 4, NUL_IDS)
    scratch = hs.Scratch(db)
    want = _check(hs, db, scratch, NUL_LITS, [0] * 4, NUL_IDS, data, off, ln)
    assert want.size > 10000
    scratch.free()


def test_stale_device_bytes_between_chunks(hs, opts):
    """A scan leaves the scratch's device corpus full of `ab\\0\\0`; the next, repacked corpus
    leaves unwritten the padding after the last block of every chunk.  Those bytes hold the
    old corpus, and no match may reach into them."""
    db = hs.compile_lit_multi(NUL_LITS, [0] * 4, NUL_IDS)
    scratch = hs.Scratch(db)
    dense = np.frombuffer(b"ab\x00\x00" * (5 * MiB // 4), dtype=np.uint8)
    off = np.arange(5 * MiB // 16384, dtype=np.uint64) * np.uint64(16384)
    ln = np.full(off.size, 16384, dtype=np.uint32)
    per_block = len(brute.scan_block(NUL_LITS, [0] * 4, NUL_IDS, dense[:16384]))
    assert hs.scan_blocks(db, dense, off, ln, scratch, collect=False) == per_block * off.size
    data, off, ln = _nul_blocks(92, int(4.3 * MiB), True)
    dev, total = _device_layout(off, ln)
    assert total < dense.size
    ends = dev + ln.astype(np.int64)
    last = [int(ends[np.searchsorted(dev, k * MiB) - 1]) for k in range(1, _chunks(total))]
    assert all(e % 4 == 2 and e % 16 for e in last), last   # followed by unwritten `\0\0ab` bytes
    want = _check(hs, db, scratch, NUL_LITS, [0] * 4, NUL_IDS, data, off, ln)
    assert want.size > 10000
    scratch.free()


# ---- single-outfix databases -------------------------------------------------------------

OUTFIX_KINDS = {"mcclellan8": 2, "mcclellan16": 3, "limex32": 5}
OUTFIX_SET = ([b"abc", b"bcd", b"xyz", b"ab", b"abcdefghij"], [0, 0, F_CASELESS, F_SINGLE, 0], [10, 11, 12, 13, 10])


@pytest.mark.parametrize("kind,ring", [("mcclellan8", 0), ("mcclellan16", 0), ("limex32", 0), ("mcclellan16", 16)])
def test_outfix_databases_across_chunks(hs, opts, request, kind, ring):
    """A single-outfix database runs one engine launch once the last chunk has arrived; its
    blocks, one longer than a chunk, still give the definition's records."""
    if ring:
        request.getfixturevalue("real_gpu")                 # over 20 s on the SIMT emulator
        opts(initial_ring=ring)
    lits, flags, ids = OUTFIX_SET
    hs.set_build_option("outfix_engine", OUTFIX_KINDS[kind])
    try:
        db = hs.compile_lit_multi(lits, flags, ids)
    finally:
        hs.set_build_option("outfix_engine", 0)
    assert db.info().runtime_impl == 2                      # ROSE_RUNTIME_SINGLE_OUTFIX
    data, off, ln = _corpus("align3", lits, seed=93, alphabet=b"abcdxyzXYZefghij")
    want = brute.scan_blocks(lits, flags, ids, data, off, ln)
    _, total = _device_layout(off, ln)
    assert _chunks(total) > 2
    scratch = hs.Scratch(db)
    got = hs.scan_blocks(db, data, off, ln, scratch)
    assert np.array_equal(got, want) and want.size > 1000
    corpus = hs.Corpus.upload(data, off, ln)
    try:
        assert np.array_equal(_sorted(hs.scan_corpus(db, corpus, scratch)), want)
    finally:
        corpus.free()
    scratch.free()


# ---- hs_scan and hs_scan_stream ----------------------------------------------------------

def _one_buffer(lits, nbytes, seed):
    rng = np.random.default_rng(seed)
    al = np.frombuffer(b"abcdefghABxy", dtype=np.uint8)
    data = al[rng.integers(0, al.size, size=nbytes)]
    dev = np.zeros(1, dtype=np.int64)
    _plant_near(data, np.zeros(1, dtype=np.int64), np.array([nbytes]), dev, lits,
                [k * MiB for k in range(1, _chunks(nbytes))] + [nbytes], rng)
    return data


def test_hs_scan_past_one_chunk(hs, opts):
    """hs_scan over one 3.5 MiB buffer: the callbacks come in `to` order, and they are the
    definition's matches."""
    lits, flags, ids = synth.literal_set(20, min_len=3, max_len=10, seed=94, caseless_frac=0.3,
                                         alphabet=b"abcdefgh")
    data = _one_buffer(lits, int(3.5 * MiB), 95)
    db = hs.compile_lit_multi(lits, flags, ids)
    scratch = hs.Scratch(db)
    n0 = hs.launch_count()
    rc, out = hs.scan(db, data, scratch)
    assert rc == hs.HS_SUCCESS
    _ranges_ran(hs, n0, data.size)
    want = sorted(brute.scan_block(lits, flags, ids, data), key=lambda r: (r[1], r[0]))
    tos = [t for _, t in out]
    assert tos == sorted(tos)
    assert out == want and len(want) > 1000
    scratch.free()


def test_stream_write_past_one_chunk(hs, opts):
    """One stream: a short write, a 3.5 MiB write, a short write.  The matches, at stream
    offsets, are the definition's over the three writes joined, including those that
    cross from one write into the next."""
    lits, flags, ids = synth.literal_set(20, min_len=2, max_len=8, seed=96, caseless_frac=0.3,
                                         alphabet=b"abcdefgh")
    data = _one_buffer(lits, int(3.5 * MiB) + 100, 97)
    lens = [37, int(3.5 * MiB), 63]
    cuts = np.cumsum([0] + lens)
    longest = max(lits, key=len)
    for c in cuts[1:3]:                                      # a literal across each write boundary
        data[c + 2 - len(longest):c + 2] = np.frombuffer(longest, dtype=np.uint8)
    db = hs.compile_lit_multi(lits, flags, ids, mode=hs.HS_MODE_STREAM)
    scratch = hs.Scratch(db)
    stream = hs.Stream(db)
    got = []
    for i in range(3):
        n0 = hs.launch_count()
        rc, out = stream.scan(data[cuts[i]:cuts[i + 1]], scratch)
        assert rc == hs.HS_SUCCESS
        if i == 1:
            _ranges_ran(hs, n0, lens[1])
        got += out
    assert stream.close(scratch) == hs.HS_SUCCESS
    want = sorted(brute.scan_block(lits, flags, ids, data[:cuts[3]]), key=lambda r: (r[1], r[0]))
    assert got == want and len(want) > 1000
    scratch.free()
