"""hs_b200_corpus_wrap: scanning a corpus that is ALREADY in device memory (a
torch tensor), with no padding before or after it -- the kernel must not touch
a byte outside [ptr, ptr + roundup16(nbytes))."""
import numpy as np
import pytest

from hyperscan_b200 import synth

pytestmark = pytest.mark.gpu


def test_wrap_reads_only_the_device_buffer(hs, ref, real_gpu):
    torch = pytest.importorskip("torch")
    lits, flags, ids = synth.literal_set(300, min_len=2, max_len=10, seed=12, alphabet=b"abcdef")
    db = hs.compile_lit_multi(lits, flags, ids)
    scratch = hs.Scratch(db)
    for total in (16, 48, 4096, 70000 - 70000 % 16):
        data, off, ln, _ = synth.block_corpus(total // 16, 16, lits, plant_per_kb=60, seed=total)
        # literals at the very first and very last bytes of the buffer
        data[: len(lits[0])] = np.frombuffer(lits[0], dtype=np.uint8)
        data[total - len(lits[1]):] = np.frombuffer(lits[1], dtype=np.uint8)
        off = np.array([0], dtype=np.uint64)
        ln = np.array([total], dtype=np.uint32)
        t = torch.from_numpy(data.copy()).cuda()
        corpus = hs.Corpus.wrap(t.data_ptr(), t.numel(), off, ln, keep=t)
        got = np.sort(hs.scan_corpus(db, corpus, scratch), order=["block", "to", "id"])
        assert np.array_equal(got, ref.scan_sorted(db.ptr, data, off, ln))
        corpus.free()
