"""The fused scan + exchange of multi-GPU runs (DESIGN.md section 8: emitMatch
stores every record into every rank's exchange buffer, publishCountKernel the
count) with both "ranks" in one process -- possible only on the SIMT emulator,
where a peer mapping is a plain pointer.  On real GPUs this path is exercised
by bench.py --gpus N under torchrun."""
import ctypes as C

import numpy as np
import pytest

from hyperscan_b200 import synth
from hyperscan_b200.capi import MATCH_DTYPE

pytestmark = pytest.mark.gpu


def test_two_ranks_deposit_records_in_both_buffers(hs, ref, emu_only):
    L = hs.lib()
    lits, flags, ids = synth.literal_set(300, seed=12, alphabet=b"abcdefgh")
    db = hs.compile_lit_multi(lits, flags, ids)
    data, off, ln, _ = synth.block_corpus(64, 1000, lits, plant_per_kb=2.0, seed=3)
    want = ref.scan_sorted(db.ptr, data, off, ln)
    world, cap, half = 2, 4096, 32
    nbytes = world * (cap + 1) * 16
    bufs, handles = [], []
    for r in range(world):
        p, h = C.c_void_p(), C.create_string_buffer(64)
        assert L.hs_b200_peer_buffer_alloc(nbytes, C.byref(p), h) == 0
        bufs.append(p)
        handles.append(h.raw)
    pitch = int(off[1] - off[0])
    for r in range(world):
        bases = (C.c_void_p * world)()
        for q in range(world):
            if q == r:
                bases[q] = bufs[q].value
            else:
                o = C.c_void_p()
                assert L.hs_b200_peer_buffer_open(handles[q], C.byref(o)) == 0
                assert o.value == bufs[q].value
                bases[q] = o.value
        scratch = hs.Scratch(db)
        assert L.hs_b200_set_peer_exchange(scratch.ptr, world, r, bases, cap, r * half) == 0
        lo = r * half
        corpus = hs.Corpus.upload(data[lo * pitch:(lo + half) * pitch], off[lo:lo + half] - off[lo], ln[lo:lo + half])
        hs.scan_corpus(db, corpus, scratch, fetch=False)
        assert L.hs_b200_set_peer_exchange(scratch.ptr, 0, 0, None, 0, 0) == 0
        corpus.free()
        scratch.free()
    for r in range(world):
        raw = np.zeros(world * (cap + 1), dtype=MATCH_DTYPE)
        assert L.hs_b200_peer_buffer_read(bufs[r], raw.ctypes.data, nbytes) == 0
        raw = raw.reshape(world, cap + 1)
        counts = [int(raw[q, 0]["id"]) for q in range(world)]
        merged = np.concatenate([raw[q, 1:1 + counts[q]] for q in range(world)])
        merged = hs.postprocess_matches(db, merged)
        got = np.sort(merged, order=["block", "to", "id"])
        assert sum(counts) >= want.size and np.array_equal(got, want)     # global block numbers, all ranks' records
    for p in bufs:
        assert L.hs_b200_peer_buffer_close(p, 0) == 0
