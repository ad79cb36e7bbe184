"""Pins the oracles on the reference's OWN known-answer tests for the literal
path (SURVEY.md A.5): unit/internal/fdr.cpp and unit/internal/noodle.cpp run
at the hwlmExec() boundary, for every engine the table builder can emit.
Both the unmodified reference engines (oracle/_ref) and the C restatement
(oracle/hs_oracle.c) must reproduce them on tables built by OUR builder."""
import ctypes as C

import numpy as np
import pytest

import oracle.port as port

DATA1 = b"mnopqrabcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ12345678901234567890mnopqr\0"
DATA2 = b"mnopqrabcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ12345678901234567890m0m"

# engines valid for small sets: FDR (0) and the 8-bucket Teddies (11..18)
ENGINES = [0, 11, 12, 13, 14, 15, 16, 17, 18]


def build_hwlm(hs, lits, engine):
    """Raw HWLM table bytes for [(bytes, nocase, noruns, id)] via the product's
    table builder (exposed for tests through a pure-literal database whose
    literal ids are remapped to the requested HWLM ids)."""
    L = hs.lib()
    L.hs_b200_test_build_hwlm.restype = C.c_long
    L.hs_b200_test_build_hwlm.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.POINTER(C.c_uint),
                                          C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.c_uint, C.c_int,
                                          C.c_void_p, C.c_size_t]
    n = len(lits)
    s = (C.c_char_p * n)(*[x[0] for x in lits])
    ln = (C.c_size_t * n)(*[len(x[0]) for x in lits])
    nc = (C.c_uint * n)(*[x[1] for x in lits])
    nr = (C.c_uint * n)(*[x[2] for x in lits])
    ids = (C.c_uint * n)(*[x[3] for x in lits])
    cap = 1 << 22
    buf = C.create_string_buffer(cap)
    sz = L.hs_b200_test_build_hwlm(s, ln, nc, nr, ids, n, engine, buf, cap)
    if sz < 0:
        pytest.skip("engine %d cannot hold this set" % engine)
    return buf.raw[:sz]


def both(ref_mod, table, data, **kw):
    a = port.hwlm_exec(table, data, **kw)
    if ref_mod is not None:
        b = ref_mod.hwlm_exec(table, data, **kw)
        assert a == b, (a, b)
    return a


@pytest.fixture(scope="module")
def refm():
    import oracle.ref as r
    return r if r.usable() else None


@pytest.mark.parametrize("engine", ENGINES)
def test_fdr_simple(hs, refm, engine):            # unit/internal/fdr.cpp:167-190
    t = build_hwlm(hs, [(b"mnopqr", 0, 0, 0)], engine)
    assert both(refm, t, DATA1) == [(5, 0), (23, 0), (83, 0)]


@pytest.mark.parametrize("engine", ENGINES)
def test_fdr_simple_single(hs, refm, engine):     # fdr.cpp:192-216
    t = build_hwlm(hs, [(b"m", 0, 0, 0)], engine)
    assert both(refm, t, DATA2) == [(0, 0), (18, 0), (78, 0), (80, 0)]


@pytest.mark.parametrize("engine", ENGINES)
def test_fdr_multi_location(hs, refm, engine):    # fdr.cpp:218-244
    t = build_hwlm(hs, [(b"abc", 0, 0, 1)], engine)
    for i in range(0, 125):
        data = bytearray(128)
        data[i:i + 3] = b"abc"
        assert both(refm, t, bytes(data)) == [(i + 2, 1)]


@pytest.mark.parametrize("engine", ENGINES)
def test_fdr_norepeat(hs, refm, engine):          # fdr.cpp:246-320
    t = build_hwlm(hs, [(b"m", 0, 1, 0)], engine)
    assert both(refm, t, DATA2) == [(0, 0)]
    t = build_hwlm(hs, [(b"m", 0, 1, 0), (b"A", 0, 0, 42)], engine)
    r = both(refm, t, DATA2)
    assert r == [(0, 0), (32, 42), (78, 0)]
    t = build_hwlm(hs, [(b"90m", 0, 1, 0), (b"zA", 0, 1, 0)], engine)
    assert both(refm, t, DATA2) == [(32, 0)]


@pytest.mark.parametrize("engine", ENGINES)
def test_fdr_termination(hs, refm, engine):       # fdr.cpp:697-745 FDRTermS/B
    t = build_hwlm(hs, [(b"mnopqr", 0, 0, 0)], engine)
    assert both(refm, t, DATA1, stop_after=1) == [(5, 0)]


def test_noodle_kats(hs, refm):                   # unit/internal/noodle.cpp:81-262
    data = b"a" * 1024
    t = build_hwlm(hs, [(b"a", 0, 0, 1000)], -1)
    assert both(refm, t, data) == [(i, 1000) for i in range(1024)]
    t = build_hwlm(hs, [(b"A", 0, 0, 1000)], -1)
    assert both(refm, t, data) == []
    t = build_hwlm(hs, [(b"A", 1, 0, 1000)], -1)
    assert both(refm, t, data) == [(i, 1000) for i in range(1024)]
    for a in range(16):                            # 16 start alignments / truncations
        assert both(refm, t, data[a:]) == [(i, 1000) for i in range(1024 - a)]
        assert both(refm, t, data[:1024 - a]) == [(i, 1000) for i in range(1024 - a)]
    # nood2: two-byte literal; nood_n: long literal with case
    t = build_hwlm(hs, [(b"aa", 0, 0, 7)], -1)
    assert both(refm, t, data) == [(i, 7) for i in range(1, 1024)]
    t = build_hwlm(hs, [(b"FOOBARZZ", 1, 0, 9)], -1)
    d = b"xxfoobarzzFooBarZZ__FOOBARZ"
    assert both(refm, t, d) == [(9, 9), (17, 9)]


def test_flood_inputs_match_non_flood_path(hs, refm):   # unit/internal/fdr_flood.cpp
    if refm is None:
        pytest.skip("needs oracle/_ref or recorded reference answers")
    for engine in (0, 15):
        lits = [(b"aaaa", 0, 0, 1), (b"aaaaaaaa", 0, 0, 2), (b"bbbbb", 1, 0, 3), (b"ab", 0, 0, 4)]
        t = build_hwlm(hs, lits, engine)
        data = b"a" * 3000 + b"B" * 2000 + b"ab" * 50 + b"a" * 500
        # the reference's flood path emits the ids of one end offset in table
        # order rather than bucket order: equal as a set per offset
        a = port.hwlm_exec(t, data)
        b = refm.hwlm_exec(t, data)
        assert sorted(a) == sorted(b) and len(a) > 5000
