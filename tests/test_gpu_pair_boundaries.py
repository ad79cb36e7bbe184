"""Class-pair first stage (FK_PAIR32) at the seams of its work split: literals
planted to END on lane boundaries (byte 15/16 of a lane's 16), step boundaries
(511/512), tile and run boundaries under warp / tile geometries that start runs
in odd places, at corpus positions 0..3 and in the last bytes before the
readable end -- uploaded and, on the device, a wrapped buffer with nothing
readable before position 0.  Sets with slot base 1 (config-2 shape, 2-byte
literals), slot base 0 (1-byte literals) and fat Teddy with its buckets folded;
L2 prefetch distances 0, 4 and 16.  Bit-exact against the reference runtime."""
import os

import numpy as np
import pytest

from hyperscan_b200 import synth

pytestmark = pytest.mark.gpu

TOTAL = (256 << 10) + 59        # ends inside a lane, a step and a tile
FILLER = b"abcdefghijklmnopqrstuvwxyz"


def _sets(hs):
    import ctypes as C
    avx2 = C.byref(hs.PlatformInfo(0, hs.HS_CPU_FEATURES_AVX2, 0, 0))
    return {
        "config2": (synth.literal_set(1000, min_len=4, max_len=8, caseless_frac=0.1, seed=2), None),
        "two-byte": (synth.literal_set(200, min_len=2, max_len=5, caseless_frac=0.1, seed=21), None),
        "one-byte": (synth.literal_set(60, min_len=1, max_len=3, caseless_frac=0.0, seed=22,
                                       alphabet=b"0123456789"), None),
        "fat-teddy": (synth.literal_set(64, min_len=3, max_len=12, caseless_frac=0.2, seed=23), avx2),
    }


def _ends(total):
    """End positions: every step boundary and a rotating offset around every lane
    boundary of every fifth step, corpus start, and the last bytes."""
    ends = set(range(0, 4))
    for b in range(512, total, 512):
        ends.add(b - 1 + (b // 512) % 5 - 1)          # b - 2 .. b + 2
    for s in range(0, total // 512, 5):
        for lane in range(1, 32):
            ends.add(s * 512 + 16 * lane - 1 + lane % 3)  # byte 15 / 16 / 17 of the lane
    ends.update(range(total - 4, total))
    return sorted(e for e in ends if e < total)


def _corpus(lits, filler, seed):
    rng = np.random.default_rng(seed)
    al = np.frombuffer(filler, dtype=np.uint8)
    data = al[rng.integers(0, al.size, size=TOTAL)]
    short = sorted(lits, key=len)
    for i, e in enumerate(_ends(TOTAL)):
        fit = [l for l in short if len(l) <= e + 1]
        if not fit:
            continue
        lit = fit[i % min(len(fit), 40)] if e < 16 else lits[(7 * i) % len(lits)]
        data[e + 1 - len(lit):e + 1] = np.frombuffer(lit, dtype=np.uint8)
    return data


@pytest.mark.parametrize("geometry", [(0, 1024), (1, 512), (3, 1536)], ids=["default", "w1-t512", "w3-t1536"])
@pytest.mark.parametrize("name", ["config2", "two-byte", "one-byte", "fat-teddy"])
def test_pair_kernel_boundaries(hs, ref, name, geometry):
    (lits, flags, ids), platform = _sets(hs)[name]
    if platform is not None and ref.best_isa() == "corei7":
        pytest.skip("the reference build on this host has no fat Teddy")
    data = _corpus(lits, FILLER if name != "one-byte" else b"abcdefghij", seed=len(lits))
    off = np.array([0], dtype=np.uint64)
    ln = np.array([TOTAL], dtype=np.uint32)
    db = hs.compile_lit_multi(lits, flags, ids, platform=platform)
    engine = db.info().engine_id
    assert 3 <= engine <= 10 if name == "fat-teddy" else engine == 0, engine
    want = ref.scan_sorted(db.ptr, data, off, ln)
    assert want.size > 500
    torch = None
    if os.environ.get("HSB200_EMU") != "1":       # the emulator has no device buffers to wrap
        torch = pytest.importorskip("torch")
    warps, tile = geometry
    try:
        hs.set_runtime_option("warps", warps)
        hs.set_runtime_option("tile_bytes", tile)
        for pf in (0, 4, 16):
            hs.set_runtime_option("pf_dist", pf)
            scratch = hs.Scratch(db)
            corpus = hs.Corpus.upload(data, off, ln)
            got = np.sort(hs.scan_corpus(db, corpus, scratch), order=["block", "to", "id"])
            corpus.free()
            assert np.array_equal(got, want), (pf, got.size, want.size)
            if torch is not None:
                t = torch.from_numpy(data.copy()).cuda()
                corpus = hs.Corpus.wrap(t.data_ptr(), t.numel(), off, ln, keep=t)
                got = np.sort(hs.scan_corpus(db, corpus, scratch), order=["block", "to", "id"])
                corpus.free()
                assert np.array_equal(got, want), ("wrap", pf, got.size, want.size)
            scratch.free()
    finally:
        for k, v in (("warps", 0), ("tile_bytes", 1024), ("pf_dist", 4)):
            hs.set_runtime_option(k, v)
