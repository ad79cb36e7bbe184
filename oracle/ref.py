"""ctypes binding of the unmodified reference runtime built into oracle/_ref/
(see oracle/ref/Makefile, oracle/ref/ref_driver.c).  TEST INFRASTRUCTURE ONLY.

Where the reference runtime is not built, the calls below that tests use answer
from tests/golden/ref_answers/: what the reference returned to the same call of
the same test on the same inputs, recorded by running the suite with the
reference built and HS_REF_RECORD=1.  (A compiled database is not part of the
key: its bytes are not reproducible from run to run, while what it must match
is.)  A question that was never recorded is an error, not a skip.
HS_REF_REPLAY=1 uses the recordings even where the reference is built."""
import atexit
import ctypes as C
import hashlib
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")
ANSWERS_DIR = os.path.join(os.path.dirname(_HERE), "tests", "golden", "ref_answers")
REC_DTYPE = np.dtype([("id", "<u4"), ("block", "<u4"), ("to", "<u8")])

_libs = {}
_answers = None      # digest -> (records, value), loaded from ANSWERS_DIR on first use
_recorded = {}       # test module -> {digest: (records, value)}, written at exit under HS_REF_RECORD=1
_calls = {}          # test node id -> reference calls made so far


def cpu_flags():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return set(line.split(":", 1)[1].split())
    except OSError:
        pass
    return set()


def best_isa():
    """Highest ISA level of the reference's fat runtime this host can run
    (reference: src/dispatcher.c:50-90)."""
    fl = cpu_flags()
    if {"avx512vbmi", "avx512bw", "avx512f"} <= fl:
        return "avx512vbmi"
    if {"avx512bw", "avx512f"} <= fl:
        return "avx512"
    if "avx2" in fl:
        return "avx2"
    return "corei7"


def available():
    """The reference runtime itself is built (oracle/_ref)."""
    return os.path.exists(os.path.join(REF_DIR, "libhsref_%s.so" % best_isa()))


def live():
    return available() and os.environ.get("HS_REF_REPLAY") != "1"


def usable():
    """Reference answers can be had: from the runtime itself, or recorded."""
    return live() or bool(_load_answers())


def _load_answers():
    global _answers
    if _answers is None:
        _answers = {}
        if os.path.isdir(ANSWERS_DIR):
            for name in sorted(os.listdir(ANSWERS_DIR)):
                if name.endswith(".npz"):
                    _answers.update(_read_answers(os.path.join(ANSWERS_DIR, name)))
    return _answers


def _read_answers(path):
    """Stored as columns, block and `to` as differences from the previous record."""
    z = np.load(path)
    recs = np.zeros(int(z["counts"].sum()), REC_DTYPE)
    recs["id"] = z["id"]
    recs["block"] = np.cumsum(z["dblock"])
    recs["to"] = np.cumsum(z["dto"])
    starts = np.zeros(z["counts"].size + 1, np.int64)
    starts[1:] = np.cumsum(z["counts"])
    return {k.tobytes(): (recs[starts[i]:starts[i + 1]], int(v)) for i, (k, v) in enumerate(zip(z["keys"], z["vals"]))}


def _write_answers():
    """One file per test module, split into parts of at most ~800 KB; processes that record
    at the same time (a test's worker processes) take turns."""
    import fcntl
    os.makedirs(ANSWERS_DIR, exist_ok=True)
    fd = os.open(ANSWERS_DIR, os.O_RDONLY)
    fcntl.flock(fd, fcntl.LOCK_EX)
    try:
        _merge_answers()
    finally:
        os.close(fd)


def _merge_answers():
    for module, new in _recorded.items():
        olds = [os.path.join(ANSWERS_DIR, f) for f in os.listdir(ANSWERS_DIR)
                if f == module + ".npz" or (f.startswith(module + ".") and f.endswith(".npz"))]
        table = {}
        for path in olds:
            table.update(_read_answers(path))
            os.remove(path)
        table.update(new)
        keys = sorted(table)
        parts = 1
        while True:
            paths = [os.path.join(ANSWERS_DIR, module + ("" if parts == 1 else ".%d" % i) + ".npz") for i in range(parts)]
            for i, path in enumerate(paths):
                _save_answers(path, {k: table[k] for k in keys[i::parts]})
            size = max(os.path.getsize(path) for path in paths)
            if size <= 800 << 10:
                break
            for path in paths:
                os.remove(path)
            parts = parts * size // (700 << 10) + 1


def _save_answers(path, table):
    keys = sorted(table)
    recs = np.concatenate([table[k][0] for k in keys] + [np.zeros(0, REC_DTYPE)])
    np.savez_compressed(path, keys=np.frombuffer(b"".join(keys), dtype=np.uint8).reshape(-1, 8),
                        vals=np.array([table[k][1] for k in keys], dtype=np.int64),
                        counts=np.array([table[k][0].size for k in keys], dtype=np.uint32), id=recs["id"],
                        dblock=np.diff(recs["block"].astype(np.int64), prepend=0),
                        dto=np.diff(recs["to"].astype(np.int64), prepend=0))


def _part(x):
    if isinstance(x, (bytes, bytearray, memoryview, np.ndarray)):
        b = _u8(x).tobytes()
    else:
        b = repr(x).encode()
    return len(b).to_bytes(8, "little") + b


def recorded(kind, parts, compute):
    """The reference's answer to question `kind` on inputs `parts`, asked by the
    running test: compute() with the reference runtime where it is built, else the
    recorded answer.  An answer is (records as REC_DTYPE, an int)."""
    test = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0].split("::", 1)
    node = "::".join([os.path.basename(test[0])] + test[1:])     # module.py::test[params]
    n = _calls.get(node, 0)
    _calls[node] = n + 1
    h = hashlib.sha1(kind.encode())
    for p in [node, n] + list(parts):
        h.update(_part(p))
    key = h.digest()[:8]
    if live():
        recs, val = compute()
        recs = np.ascontiguousarray(recs, dtype=REC_DTYPE)
        if os.environ.get("HS_REF_RECORD") == "1":
            module = os.path.splitext(node.split("::")[0])[0] or "other"
            if not _recorded:
                atexit.register(_write_answers)
            _recorded.setdefault(module, {})[key] = (recs.copy(), int(val))
        return recs, int(val)
    ans = _load_answers().get(key)
    if ans is None:
        raise RuntimeError("no recorded reference answer for this %s call (%s): build the reference runtime "
                           "(oracle/ref/Makefile) and rerun the test with HS_REF_RECORD=1" % (kind, key.hex()))
    return ans[0].copy(), ans[1]


def lib(isa=None):
    isa = isa or best_isa()
    if isa not in _libs:
        path = os.path.join(REF_DIR, "libhsref_%s.so" % isa)
        if not os.path.exists(path):
            raise RuntimeError("reference runtime not built: %s (run `make -C oracle/ref REF=<intel/hyperscan "
                               "5.4.2 checkout>`)" % path)
        L = C.CDLL(path)
        vp = C.c_void_p
        L.ref_scan_collect.restype = C.c_long
        L.ref_scan_collect.argtypes = [vp, vp, vp, vp, C.c_size_t, vp, C.c_size_t, C.c_size_t,
                                       C.POINTER(C.c_int)]
        L.ref_stream_collect.restype = C.c_long
        L.ref_vector_collect.restype = C.c_long
        L.ref_vector_collect.argtypes = [vp, vp, vp, C.c_size_t, vp, C.c_size_t, C.c_size_t, C.POINTER(C.c_int)]
        L.ref_stream_collect.argtypes = [vp, vp, vp, C.c_size_t, vp, C.c_size_t, C.c_size_t, C.POINTER(C.c_int)]
        L.ref_scan_blocks_mt.restype = C.c_double
        L.ref_scan_blocks_mt.argtypes = [vp, vp, vp, vp, C.c_size_t, C.c_uint, C.c_uint,
                                         C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
        L.ref_hwlm_exec.restype = C.c_long
        L.ref_hwlm_exec.argtypes = [vp, vp, C.c_size_t, C.c_size_t, C.c_ulonglong, vp, C.c_size_t,
                                    C.c_size_t]
        for f in (L.ref_shufti, L.ref_truffle):
            f.restype = C.c_long
            f.argtypes = [vp, vp, vp, C.c_size_t]
        L.ref_vermicelli.restype = C.c_long
        L.ref_vermicelli.argtypes = [C.c_ubyte, C.c_int, vp, C.c_size_t]
        L.ref_dvermicelli.restype = C.c_long
        L.ref_dvermicelli.argtypes = [C.c_ubyte, C.c_ubyte, C.c_int, vp, C.c_size_t]
        _libs[isa] = L
    return _libs[isa]


def _u8(data):
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data).view(np.uint8).reshape(-1)
    return np.frombuffer(bytes(data), dtype=np.uint8)


def scan_collect(db_ptr, data, offsets, lengths, stop_after=0, isa=None, cap=None):
    """Reference hs_scan() over blocks; records in delivery order.
    Returns (records, last_error)."""
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    ln = np.ascontiguousarray(lengths, dtype=np.uint32)
    return recorded("scan_collect", [data, off, ln, stop_after, isa],
                    lambda: _scan_collect(db_ptr, data, off, ln, stop_after, isa, cap))


def _scan_collect(db_ptr, data, offsets, lengths, stop_after, isa, cap):
    a = _u8(data)
    keep = a if a.size else np.zeros(1, dtype=np.uint8)
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    ln = np.ascontiguousarray(lengths, dtype=np.uint32)
    cap = cap or (1 << 20)
    while True:
        out = np.zeros(cap, dtype=REC_DTYPE)
        err = C.c_int()
        n = lib(isa).ref_scan_collect(db_ptr, keep.ctypes.data, off.ctypes.data, ln.ctypes.data, off.size,
                                      out.ctypes.data, cap, stop_after, C.byref(err))
        if n < 0:
            raise RuntimeError("reference hs_alloc_scratch failed: %d" % n)
        if n <= cap:
            return out[:n], err.value
        cap = int(n) + 16


def stream_collect(db_ptr, data, write_lengths, stop_after=0, isa=None):
    """Reference streaming scan of `data` cut into consecutive writes; records
    (id, write index, to = stream offset) in delivery order + last error."""
    wl = np.ascontiguousarray(write_lengths, dtype=np.uint32)
    return recorded("stream_collect", [data, wl, stop_after, isa],
                    lambda: _stream_collect(db_ptr, data, wl, stop_after, isa))


def _stream_collect(db_ptr, data, write_lengths, stop_after, isa):
    a = _u8(data)
    keep = a if a.size else np.zeros(1, dtype=np.uint8)
    wl = np.ascontiguousarray(write_lengths, dtype=np.uint32)
    assert int(wl.sum()) == a.size
    cap = 1 << 18
    while True:
        out = np.zeros(cap, dtype=REC_DTYPE)
        err = C.c_int()
        n = lib(isa).ref_stream_collect(db_ptr, keep.ctypes.data, wl.ctypes.data, wl.size, out.ctypes.data,
                                        cap, stop_after, C.byref(err))
        if n < 0:
            raise RuntimeError("reference stream open failed: %d" % n)
        if n <= cap:
            return out[:n], err.value
        cap = int(n) + 16


def vector_collect(db_ptr, data, buf_lengths, stop_after=0, isa=None):
    """Reference hs_scan_vector over `data` cut into consecutive buffers; records
    (id, 0, to counted from the first buffer) in delivery order + the call's
    return code."""
    bl = np.ascontiguousarray(buf_lengths, dtype=np.uint32)
    return recorded("vector_collect", [data, bl, stop_after, isa],
                    lambda: _vector_collect(db_ptr, data, bl, stop_after, isa))


def _vector_collect(db_ptr, data, buf_lengths, stop_after, isa):
    a = _u8(data)
    keep = a if a.size else np.zeros(1, dtype=np.uint8)
    bl = np.ascontiguousarray(buf_lengths, dtype=np.uint32)
    assert int(bl.sum()) == a.size
    cap = 1 << 18
    while True:
        out = np.zeros(cap, dtype=REC_DTYPE)
        err = C.c_int()
        n = lib(isa).ref_vector_collect(db_ptr, keep.ctypes.data, bl.ctypes.data, bl.size, out.ctypes.data,
                                        cap, stop_after, C.byref(err))
        if n < 0:
            raise RuntimeError("reference scratch allocation failed: %d" % n)
        if n <= cap:
            return out[:n], err.value
        cap = int(n) + 16


def scan_sorted(db_ptr, data, offsets, lengths, isa=None):
    """Match multiset sorted by (block, to, id): what 'bit-exact' is defined on
    (SURVEY.md F8)."""
    r, err = scan_collect(db_ptr, data, offsets, lengths, isa=isa)
    if err:
        raise RuntimeError("reference hs_scan error %d" % err)
    return np.sort(r, order=["block", "to", "id"])


def physical_core_cpus():
    """CPUs of the affinity mask, one hardware thread per physical core first (then
    the SMT siblings), for pinning the bench threads 1:1 the way hsbench does."""
    cpus = sorted(os.sched_getaffinity(0))
    first, rest, seen = [], [], set()
    for c in cpus:
        try:
            with open("/sys/devices/system/cpu/cpu%d/topology/thread_siblings_list" % c) as f:
                sib = f.read().strip()
        except OSError:
            sib = str(c)
        if sib in seen:
            rest.append(c)
        else:
            seen.add(sib)
            first.append(c)
    return first + rest


def pin_bench_threads(cpus):
    """Pin bench thread i to cpus[i % len(cpus)]; an empty list unpins."""
    arr = (C.c_int * max(1, len(cpus)))(*cpus)
    lib().ref_set_bench_cpus(arr, len(cpus))


def bench_blocks(db_ptr, data, offsets, lengths, threads, repeats, isa=None):
    """hsbench-style timing loop (tools/hsbench/main.cpp:503-527).  Returns
    (seconds, matches, bytes)."""
    a = _u8(data)
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    ln = np.ascontiguousarray(lengths, dtype=np.uint32)
    m = C.c_ulonglong()
    b = C.c_ulonglong()
    t = lib(isa).ref_scan_blocks_mt(db_ptr, a.ctypes.data, off.ctypes.data, ln.ctypes.data, off.size,
                                    threads, repeats, C.byref(m), C.byref(b))
    if t < 0:
        raise RuntimeError("reference bench failed")
    return t, int(m.value), int(b.value)


def hwlm_exec(hwlm_bytes, data, start=0, groups=0xFFFFFFFFFFFFFFFF, stop_after=0, isa=None):
    """Reference hwlmExec() on a raw HWLM table (64-byte aligned copy): [(end, id)]."""
    recs, _ = recorded("hwlm_exec", [data, start, groups, stop_after, isa],
                       lambda: (_hwlm_exec(hwlm_bytes, data, start, groups, stop_after, isa), 0))
    return [(int(r["to"]), int(r["id"])) for r in recs]


def _hwlm_exec(hwlm_bytes, data, start, groups, stop_after, isa):
    raw = np.zeros(len(hwlm_bytes) + 64, dtype=np.uint8)
    o = (-raw.ctypes.data) % 64
    raw[o:o + len(hwlm_bytes)] = np.frombuffer(hwlm_bytes, dtype=np.uint8)
    a = _u8(data)
    # the reference engines may read a few bytes around the buffer: pad it
    buf = np.zeros(a.size + 128, dtype=np.uint8)
    buf[64:64 + a.size] = a
    cap = 1 << 16
    out = np.zeros(cap, dtype=REC_DTYPE)
    n = lib(isa).ref_hwlm_exec(raw.ctypes.data + o, buf.ctypes.data + 64, a.size, start, groups,
                               out.ctypes.data, cap, stop_after)
    return out[:min(n, cap)]


def nfa_exec_blocks(nfa_bytes, data, offsets, lengths, isa=None, cap=1 << 20):
    """Reference nfaExecMcClellan8_B / 16_B / nfaExecSheng_B over every block (offset 0):
    the callbacks as records sorted by (block, to, id)."""
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    ln = np.ascontiguousarray(lengths, dtype=np.uint32)
    recs, _ = recorded("nfa_exec_blocks", [data, off, ln, isa],
                       lambda: (_nfa_exec_blocks(nfa_bytes, data, off, ln, isa, cap), 0))
    return recs


def _nfa_exec_blocks(nfa_bytes, data, offsets, lengths, isa, cap):
    a = _u8(data)
    keep = a if a.size else np.zeros(1, dtype=np.uint8)
    off = np.ascontiguousarray(offsets, dtype=np.uint64)
    ln = np.ascontiguousarray(lengths, dtype=np.uint32)
    raw = np.zeros(len(nfa_bytes) + 64, dtype=np.uint8)     # struct NFA is cache-line aligned
    shift = (-raw.ctypes.data) % 64
    raw[shift:shift + len(nfa_bytes)] = np.frombuffer(nfa_bytes, dtype=np.uint8)
    L = lib(isa)
    L.ref_nfa_exec_blocks.restype = C.c_long
    L.ref_nfa_exec_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.c_size_t]
    while True:
        out = np.zeros(cap, dtype=REC_DTYPE)
        n = L.ref_nfa_exec_blocks(raw.ctypes.data + shift, keep.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                  off.size, out.ctypes.data, cap)
        if n < 0:
            raise RuntimeError("reference: engine type not handled")
        if n <= cap:
            return np.sort(out[:n], order=["block", "to", "id"])
        cap = int(n) + 16
