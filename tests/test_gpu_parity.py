"""Parity of the H100 scan path (through the C ABI) against the unmodified
reference runtime scanning the SAME database, and against the definition-level
brute-force oracle.  Bit-exact on the sorted (block, to, id) multiset."""
import numpy as np
import pytest

from hyperscan_b200 import synth
import oracle.brute as brute

pytestmark = pytest.mark.gpu

F_CASELESS, F_SINGLE = 1, 8


def _sorted(recs):
    return np.sort(np.asarray(recs), order=["block", "to", "id"])


def _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=True, platform=None):
    db = hs.compile_lit_multi(lits, flags, ids, platform=platform)
    scratch = hs.Scratch(db)
    want = ref.scan_sorted(db.ptr, data, off, ln)
    if use_brute:
        b = brute.scan_blocks(lits, flags, ids, data, off, ln)
        assert np.array_equal(want, b), "reference runtime disagrees with the definition"
    got = _sorted(hs.scan_blocks(db, data, off, ln, scratch))
    assert got.size == want.size, (got.size, want.size)
    assert np.array_equal(got, want)
    corpus = hs.Corpus.upload(data, off, ln)
    got2 = _sorted(hs.scan_corpus(db, corpus, scratch))
    assert np.array_equal(got2, want)
    corpus.free()
    scratch.free()
    return db, want


# engine id 0 = FDR; 11..18 = Teddy (8 buckets); forced through the build
# option the way unit/internal/fdr.cpp:114-137 forces engines with hints
@pytest.mark.parametrize("nlits,engine", [(1, -1), (5, -1), (30, -1), (48, 15), (5, 0), (200, -1),
                                          (1000, -1), (3000, -1)])
def test_engines_random_blocks(hs, ref, nlits, engine):
    lits, flags, ids = synth.literal_set(nlits, min_len=2 if nlits < 40 else 4, max_len=12, seed=nlits,
                                         caseless_frac=0.2, alphabet=b"abcdefgh")
    if engine >= 0:
        hs.set_build_option("force_engine", engine)
    data, off, ln = synth.ragged_corpus([0, 1, 3, 7, 15, 16, 17, 31, 64, 100, 511, 512, 513, 1024, 2047, 2048,
                                         2049, 4096, 10000, 65536 + 5], lits, seed=3,
                                        alphabet=b"abcdefghABCDxy")
    _check_all(hs, ref, lits, flags, ids, data, off, ln)


def _avx2(hs):
    import ctypes as C
    return C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0))


@pytest.mark.parametrize("nlits,lo,hi", [(49, 2, 8), (64, 3, 12), (90, 3, 8), (96, 4, 12)])
def test_fat_teddy_16_buckets_folded(hs, ref, nlits, lo, hi):
    """Databases compiled for an AVX2 platform carry 16-bucket ("fat") Teddy
    (engine ids 3..10, src/fdr/teddy_avx2.c:395-447): the device runs them
    through the class-pair kernel with buckets i and i + 8 folded onto one
    first-stage bit, which confirmKernel unfolds."""
    if ref.best_isa() == "corei7":
        pytest.skip("the reference build on this host has no fat Teddy")
    lits, flags, ids = synth.literal_set(nlits, min_len=lo, max_len=hi, seed=90 + nlits, caseless_frac=0.2,
                                         alphabet=b"abcdefgh")
    data, off, ln = synth.ragged_corpus([0, 1, 3, 15, 16, 17, 33, 100, 511, 512, 513, 1024, 2049, 4096, 20000,
                                         65536 + 5], lits, seed=2, alphabet=b"abcdefghABCDxy", plant_per_kb=4)
    db, want = _check_all(hs, ref, lits, flags, ids, data, off, ln, platform=_avx2(hs))
    assert 3 <= db.info().engine_id <= 10, db.info().engine_id
    assert want.size > 100


def test_large_literal_set_two_level_prefilter(hs, ref):
    # config 5 shape (50 k literals -> FDR domain 15): the shared-memory bitmap
    # saturates and the second-level bitmap in HBM takes over
    lits, flags, ids = synth.literal_set(50000, min_len=4, max_len=16, seed=50, caseless_frac=0.1)
    data, off, ln, _ = synth.block_corpus(512, 1024, lits, plant_per_kb=1.0, seed=51)
    db, want = _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    assert (db.info().engine_id, db.info().fdr_domain, db.info().fdr_stride) == (0, 15, 1)
    assert want.size > 300


@pytest.mark.parametrize("opts,one_byte", [({}, False), ({"heavy": 0}, False), ({"heavy": 2}, False),
                                           ({"heavy": 0}, True), ({"heavy": 2}, True), ({"gram": 2}, False),
                                           ({"gram": 0}, False)],
                         ids=["default", "lane-entries", "word-entries", "lane-entries-no-prefilter",
                              "word-entries-no-prefilter", "class-4-gram", "no-4-gram"])
def test_large_literal_set_candidate_paths(hs, ref, opts, one_byte):
    """Both candidate paths of the class-pair kernel and the class 4-gram first
    stage give the same matches.  One 1-byte literal leaves the set without
    prefilter keys, so the candidates reach the list without the bitmap probe."""
    lits, flags, ids = synth.literal_set(20000, min_len=4, max_len=16, seed=52, caseless_frac=0.1)
    data, off, ln, _ = synth.block_corpus(256, 1024, lits, plant_per_kb=1.0, seed=53)
    if one_byte:
        lits, flags, ids = lits + [b"~"], flags + [0], ids + [max(ids) + 1]
    try:
        for k, v in opts.items():
            hs.set_runtime_option(k, v)
        _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    finally:
        for k, v in (("heavy", 1), ("gram", 1)):
            hs.set_runtime_option(k, v)


@pytest.mark.parametrize("alphabet", [b"abcdefghijklmnopqrstuvwxyz", bytes(range(0x21, 0x7f)), bytes(range(256))])
def test_class_4gram_first_stage_alphabets(hs, ref, alphabet):
    """FK_GRAM4 forced on sets over few and over many byte values (more than 31 in use:
    case folding, then the rarest values share classes)."""
    lits, flags, ids = synth.literal_set(400, min_len=4, max_len=10, seed=61, caseless_frac=0.3, alphabet=alphabet)
    data, off, ln = synth.ragged_corpus([0, 3, 4, 5, 100, 1024, 5000, 70000], lits, seed=62, plant_per_kb=5,
                                        alphabet=alphabet + b"AB")
    try:
        hs.set_runtime_option("gram", 2)
        _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    finally:
        hs.set_runtime_option("gram", 1)


def test_config5_shape_at_scale(hs, ref, real_gpu):
    """BASELINE config 5 shape (50 000 literals, FDR domain 15) over 64 Ki blocks:
    bit-exact against the reference runtime on the whole 64 MiB."""
    lits, flags, ids = synth.literal_set(50000, min_len=4, max_len=16, seed=50, caseless_frac=0.1)
    data, off, ln, _ = synth.block_corpus(65536, 1024, lits, plant_per_kb=0.05, seed=54)
    db, want = _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    assert (db.info().engine_id, db.info().fdr_domain, db.info().fdr_stride) == (0, 15, 1)
    assert want.size > 3000


def test_hs_scan_single_block_and_termination(hs, ref):
    lits = [b"mnopqr"]
    db = hs.compile_lit_multi(lits, [0], [7])
    scratch = hs.Scratch(db)
    data = b"mnopqrabcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ12345678901234567890mnopqr"
    rc, out = hs.scan(db, data, scratch)
    assert rc == hs.HS_SUCCESS
    # unit/internal/fdr.cpp:167-190 (ends 5, 23, 83) -> to = end + 1
    assert out == [(7, 6), (7, 24), (7, 84)]
    rc, out = hs.scan(db, data, scratch, stop_after=2)
    assert rc == hs.HS_SCAN_TERMINATED and out == [(7, 6), (7, 24)]
    rc, out = hs.scan(db, b"", scratch)
    assert rc == hs.HS_SUCCESS and out == []


def test_singlematch_and_shared_ids(hs, ref):
    lits = [b"abc", b"bcd", b"abcd", b"xyzw", b"ABC"]
    flags = [F_SINGLE, 0, 0, F_SINGLE | F_CASELESS, 0]
    ids = [1, 2, 2, 3, 1]
    # id 1 mixes singlematch and not -> compile error like the reference
    with pytest.raises(hs.HsError):
        hs.compile_lit_multi(lits, flags, ids)
    flags[4] = F_SINGLE
    data, off, ln = synth.ragged_corpus([300, 5000, 64], lits, plant_per_kb=30, seed=5,
                                        alphabet=b"abcdxyzwXYZW")
    _check_all(hs, ref, lits, flags, ids, data, off, ln)


def test_long_literals_med_lit_check(hs, ref):
    lits = [b"abcdefghijkl", b"zzabcdefghijkl", b"hijkl", b"ABCDEFGHIJKLMNOPQRSTUVWX"]
    flags = [0, F_CASELESS, 0, F_CASELESS]
    ids = [10, 11, 12, 13]
    data, off, ln = synth.ragged_corpus([2000, 3000, 30], lits, plant_per_kb=20, seed=9,
                                        alphabet=b"abcdefghijklz")
    _check_all(hs, ref, lits, flags, ids, data, off, ln)


def test_flood_and_ring_growth(hs, ref):
    # every byte matches (unit/internal/fdr_flood.cpp); the initial record ring
    # is made tiny so the overflow -> grow -> rescan path runs
    hs.set_runtime_option("initial_ring", 64)
    try:
        lits = [b"a", b"aa", b"aaaa", b"aaaaaaaa", b"aaaaaaaaaaaa"]
        data = np.full(20000, ord("a"), dtype=np.uint8)
        off = np.array([0, 10000], dtype=np.uint64)
        ln = np.array([9999, 10000], dtype=np.uint32)
        _check_all(hs, ref, lits, [0, 0, F_CASELESS, 0, 0], [1, 2, 3, 4, 5], data, off, ln)
    finally:
        hs.set_runtime_option("initial_ring", 1 << 20)


def test_block_boundaries_do_not_leak(hs, ref):
    # literals straddling two adjacent blocks must not match; blocks are packed
    # back to back (16-byte aligned) so the halo holds the neighbour's bytes
    lits = [b"abcdefgh", b"efgh", b"h"]
    data = np.frombuffer(b"xxxxxxxxxxxxabcdefghxxxxxxxxxxxxxxxx" * 4, dtype=np.uint8).copy()
    off = np.array([0, 16, 32, 48], dtype=np.uint64)
    ln = np.array([16, 16, 16, 5], dtype=np.uint32)
    _check_all(hs, ref, lits, [0, 0, 0], [1, 2, 3], data, off, ln)


def test_short_literals_pair_kernel_paths(hs, ref):
    """A 500-literal FDR set on the class-pair kernel, then the same set with 1- and
    2-byte literals added: slot base 0 and no prefilter bitmap."""
    lits, flags, ids = synth.literal_set(500, min_len=4, max_len=14, seed=21, caseless_frac=0.3,
                                         alphabet=b"abcdefgh")
    lits += [b"ab", b"b", b"cdc"]
    flags += [0, 1, 0]
    ids += [1000, 1001, 1002]
    data, off, ln = synth.ragged_corpus([70000, 33, 5000, 0, 12345], lits, seed=13, plant_per_kb=3,
                                        alphabet=b"abcdefghABCDEFGH")
    _check_all(hs, ref, lits[:500], flags[:500], ids[:500], data, off, ln, use_brute=False)
    _check_all(hs, ref, lits, flags, ids, data[:20000], off[:1], ln[:1] // 4, use_brute=False)


@pytest.mark.parametrize("tile,warps", [(512, 1), (1024, 4), (4096, 8), (2048, 16), (512, 3), (8192, 24)])
def test_tile_split_invariance(hs, ref, tile, warps):
    """The split of the tiles over the warps and CTAs never changes the matches."""
    lits, flags, ids = synth.literal_set(300, seed=4, alphabet=b"abcdefgh")
    data, off, ln, _ = synth.block_corpus(257, 1000, lits, plant_per_kb=2.0, seed=8)
    try:
        hs.set_runtime_option("tile_bytes", tile)
        hs.set_runtime_option("warps", warps)
        _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    finally:
        hs.set_runtime_option("tile_bytes", 1024)
        hs.set_runtime_option("warps", 0)


GEOMETRIES = [{"warps": 24},                        # the 768-thread kernel builds
              {"warps": 32},                        # the 1024-thread build of the wide kernel
              {"tile_bytes": 4096, "warps": 5},
              {"initial_ring": 16}]                 # candidate list and ring overflow -> grow and rescan
GEOMETRY_DEFAULTS = {"warps": 0, "tile_bytes": 1024, "initial_ring": 1 << 20}


@pytest.mark.parametrize("opts", GEOMETRIES, ids=[",".join("%s=%d" % kv for kv in g.items()) for g in GEOMETRIES])
@pytest.mark.parametrize("nlits", [1, 30, 48, 300, 1000])
def test_geometry_parity(hs, ref, opts, nlits):
    """Noodle (1), 8-bucket Teddy (30, 48) and FDR sets (300, 1000) under the kernel
    builds and ring sizes a geometry option selects."""
    lits, flags, ids = synth.literal_set(nlits, min_len=2 if nlits < 40 else 4, max_len=12, seed=nlits + 7,
                                         caseless_frac=0.2, alphabet=b"abcdefgh")
    data, off, ln = synth.ragged_corpus([0, 1, 3, 15, 16, 17, 31, 32, 33, 100, 511, 512, 513, 1023, 1024, 1025,
                                         2047, 2048, 2049, 4096, 10000, 65536 + 5, 200000], lits, seed=3,
                                        alphabet=b"abcdefghABCDxy")
    try:
        for k, v in opts.items():
            hs.set_runtime_option(k, v)
        _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    finally:
        for k, v in GEOMETRY_DEFAULTS.items():
            hs.set_runtime_option(k, v)


def test_config2_shape_sample(hs, ref):
    # BASELINE config 2 shape at a size the CPU oracles finish in seconds
    lits, flags, ids = synth.literal_set(1000)
    data, off, ln, planted = synth.block_corpus(16384, 1024, lits, plant_per_kb=0.05)
    db, want = _check_all(hs, ref, lits, flags, ids, data, off, ln, use_brute=False)
    assert db.info().engine_id == 0 and db.info().fdr_stride == 2
    assert want.size >= len(planted) * 0.9
