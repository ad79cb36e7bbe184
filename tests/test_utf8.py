"""Expressions in UTF-8 mode (HS_FLAG_UTF8, without Unicode properties): a character is a code point and matches its
encoding; ".", negated classes, non-ASCII classes and \\W \\D \\S \\H \\V \\N match whole encoded characters through a
small byte automaton (regex_nfa.cpp, DESIGN.md section 10b).

CPU half: the UNMODIFIED reference hs_scan on the databases compiled here reports exactly the match ends the definition
gives -- Python's re on the decoded text, end offsets mapped back to bytes -- over seeded valid UTF-8 corpora mixing
1- to 4-byte characters; invalid bytes in the data, pinned; the refusals; widths and bounds in bytes; and the reference's
own recorded UTF-8 vectors (tests/golden/hscollider_utf8.json).
GPU half: the device equals the reference record for record through every scan entry point, both engines, a split
set, a literal matcher beside an engine, and segment seams inside multi-byte characters."""
import base64
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from test_expr_info import Info
from test_mixed_rose import _pack, _per_block, _ref_per_block

CASELESS, DOTALL, MULTILINE, SINGLE, UTF8, UCP = 1, 2, 4, 8, 32, 64
W = "[0-9A-Za-z_]"
NW = "[^0-9A-Za-z_]"
HSP = "\t \xa0\u1680\u180e\u2000-\u200a\u202f\u205f\u3000"

# (expression, flags, the same language in Python's re on str, ASCII \\w \\d \\s \\b spelled out)
CASES = [
    ("foo\\d+bar", 0, "foo[0-9]+bar"), ("é+x", 0, "é+x"), ("a.c", 0, "a.c"), ("a.c", DOTALL, "(?s:a.c)"),
    ("[^a-z]{2}q", 0, "[^a-z]{2}q"), ("[à-ÿ€-₿]+z", 0, "[à-ÿ€-₿]+z"), ("\\W\\D", 0, NW + "[^0-9]"),
    ("\\S\\H\\V!", 0, "[^ \t\n\x0b\f\r][^" + HSP + "][^\n\x0b\f\r\x85\u2028\u2029]!"), ("a\\N+z", DOTALL, "a[^\n]+z"),
    ("\\h\\v", 0, "[" + HSP + "][\n\x0b\f\r\x85\u2028\u2029]"), ("\\x{1F600}|\\x{12000}\\w", 0, "\U0001F600|\U00012000" + W),
    ("\\o{20254}+", 0, "€+"), ("(?i)k[s-t]", 0, "(?i:k[s-t])"), ("\\bab+\\b", 0, "(?<!%s)ab+(?!%s)" % (W, W)),
    ("^.{3}", 0, "^.{3}"), ("€$", 0, "€$"), ("[^\\x{80}-\\x{10FFFF}]+z", 0, "[^\x80-\U0010ffff]+z"),
    ("😀{2,3}", 0, "😀{2,3}"), ("(?m)^空.", MULTILINE, "(?m:^空.)"), ("\\Qé+\\E", 0, "é\\+"),
    ("[[:alpha:]]é", 0, "[A-Za-z]é"), ("x[^é😀]y", 0, "x[^é😀]y"), ("[\\x{100}-\\x{2FFF}a]{2,}", 0, "[\u0100-\u2fffa]{2,}"),
    ("\\Bé", 0, "(?<!%s)é" % W), ("a\\b.", 0, "(?<=a)(?!%s)." % W), ("(ü|空|𒀀)+(?i)[a-c]", 0, "(ü|空|𒀀)+(?i:[a-c])"),
]
PLANT = "foo12bar ééx a€c a\nc €éq àÿ€z ¬1! é\xa0\u2028! \u3000\u2028 \U00012000a 😀😀😀 Ks k\u017f abb é\n空x Āé+ x€y éaĀĀa 𒀀ü3 "
ALPHA = list("abcqxyzkKsS019 _!\nfooébarÿĀàü€₿空\u3000\u2028\u212a\u017f😀𒀀\U0010fffd\xa0\x85")


def _text(seed, n=40):
    rng = np.random.default_rng(seed)
    return "".join(ALPHA[int(i)] for i in rng.integers(0, len(ALPHA), size=n))


def _ends(py, text, min_offset=0, max_offset=None, min_length=0):
    """every byte end offset of a match of `py` in `text` (decoded): a fixed-width look-behind pins the match end
    in characters, and the offsets are mapped back to bytes"""
    byte_at = np.cumsum([0] + [len(c.encode()) for c in text])
    out = []
    for e in range(1, len(text) + 1):
        end = int(byte_at[e])
        if end < max(min_offset, 1) or (max_offset is not None and end > max_offset):
            continue
        rx = re.compile("(?:" + py + ")(?<=(?s:\\A.{%d}))" % e)
        if any(rx.match(text, s) for s in range(e) if end - int(byte_at[s]) >= max(min_length, 1)):
            out.append(end)
    return out


def _ref_ends(ref, db, data):
    a = np.frombuffer(data, dtype=np.uint8) if data else np.zeros(0, np.uint8)
    r = ref.scan_sorted(db.ptr, a, np.array([0], np.uint64), np.array([len(data)], np.uint32))
    return [(int(x["id"]), int(x["to"])) for x in r]


def _compile(hs, pat, fl, ext=None, dfa=1):
    hs.set_build_option("regex_dfa", dfa)
    try:
        return hs.compile_ext_multi([pat.encode()], [fl | UTF8], [7], [ext])
    finally:
        hs.set_build_option("regex_dfa", 1)


@pytest.mark.parametrize("dfa", [1, 0])
@pytest.mark.parametrize("ci", range(len(CASES)))
def test_reference_hs_scan_equals_definition(hs, ref, ci, dfa):
    pat, fl, py = CASES[ci]
    db = _compile(hs, pat, fl, dfa=dfa)
    hits = 0
    for seed in range(8):
        text = _text(100 * ci + seed) + (PLANT if seed % 2 else "€\n")
        want = [(7, e) for e in _ends(py, text)]
        assert _ref_ends(ref, db, text.encode()) == want, (pat, text)
        hits += len(want)
    assert hits > 0, pat


def test_finite_sets_of_non_ascii_literals_take_the_literal_route(hs, ref):
    """a case-sensitive finite set of non-ASCII literals is matched as its bytes by the literal matcher; caseless
    "k" / "s" (which also match KELVIN SIGN and LONG S) and escapes above \\x7F go to the regex route"""
    for pat, fl, impl in [("空|ü€", 0, 1), ("(é|ø)x?😀", 0, 1), ("abc", CASELESS, 1), ("ask", CASELESS, 2),
                          ("\\xe9", 0, 2), ("[éa]b", 0, 2)]:
        db = _compile(hs, pat, fl)
        assert db.info().runtime_impl == impl, pat
        py = "(?i:%s)" % pat if fl & CASELESS else pat.replace("\\xe9", "é")
        for seed in range(4):
            text = _text(7 + seed, 60) + "空ü€ éx😀 øx😀 ASK a\u212a\u017f\u212a é éb ab"
            assert _ref_ends(ref, db, text.encode()) == [(7, e) for e in _ends(py, text)], pat
    with pytest.raises(hs.HsError, match="literal API"):
        hs.compile_lit_multi(["空".encode()], [UTF8], [1])


# what `.` and a negated class accept in data that is not valid UTF-8 (DESIGN.md section 10b): the encodings of every
# code point of the set, surrogates D800-DFFF included, each as one whole sequence; nothing else
INVALID = [
    (b"a\x80b", []), (b"a\xc3b", []), (b"a\xc0\x80b", []), (b"a\xc1\xbfb", []), (b"a\xe0\x80\x80b", []),
    (b"a\xe0\x9f\xbfb", []), (b"a\xed\xa0\x80b", [5]), (b"a\xed\xbf\xbfb", [5]), (b"a\xf0\x8f\xbf\xbfb", []),
    (b"a\xf0\x90\x80\x80b", [6]), (b"a\xf4\x8f\xbf\xbfb", [6]), (b"a\xf4\x90\x80\x80b", []), (b"a\xf5\x80\x80\x80b", []),
    (b"a\xff\xfeb", []), (b"a\xc3\xa9\x80b", []), (b"a\xe2\x82b", []), (b"\xc3a\xc3\xa9b", [5]),
]


@pytest.mark.parametrize("pat", ["a.b", "a[^x]b", "a\\Wb"])
def test_invalid_bytes_in_the_data(hs, ref, pat):
    for dfa in (1, 0):
        db = _compile(hs, pat, 0, dfa=dfa)
        for data, want in INVALID:
            assert _ref_ends(ref, db, data) == [(7, e) for e in want], (pat, data)


def test_literals_and_one_byte_in_invalid_data(hs, ref):
    """a literal character matches its bytes wherever they are -- the scan does not resynchronise on characters --
    and \\C is one byte, whatever it is"""
    db = _compile(hs, "é", 0)
    assert _ref_ends(ref, db, b"\xc3\xc3\xa9\xa9\xe9") == [(7, 3)]
    db = _compile(hs, "a\\Cb", 0)
    assert _ref_ends(ref, db, b"a\x80b a\xffb ab a\xc3\xa9b") == [(7, 3), (7, 7)]
    db = _compile(hs, "é\\C+z", 0)
    assert _ref_ends(ref, db, "éz é\xe9z é😀z".encode()) == [(7, 9), (7, 17)]


@pytest.mark.parametrize("pat,flags,msg", [
    (b"\\p{L}", 0, "Unicode properties"), (b"[\\P{Lu}]", 0, "Unicode properties"), (b"a\\X", 0, "\\X"),
    (b"ab+c", UCP, "HS_FLAG_UCP"), (b"a\\d+", UCP, "HS_FLAG_UCP"), ("é+".encode(), CASELESS, "case folding"),
    ("(?i)x[à-ÿ]+".encode(), 0, "case folding"), ("[\\x{100}]+".encode(), CASELESS, "case folding"),
    (b"\xc0\x80+", 0, "Expression is not valid UTF-8."), (b"a\xed\xa0\x80+", 0, "Expression is not valid UTF-8."),
    (b"\xf4\x90\x80\x80", 0, "Expression is not valid UTF-8."), (b"\\Q\xe9\\E+", 0, "Expression is not valid UTF-8."),
    (b"[\xe9]", 0, "Expression is not valid UTF-8."), (b"a\xe2\x82", 0, "Expression is not valid UTF-8."),
    (b"\\x{110000}", 0, "Value in \\x{...} sequence is too large"), (b"\\x{zz}", 0, "non-hex or missing }"),
    (b"\\o{4200000}", 0, "Value in \\o{...} sequence is too large"), (b"\\o{9}", 0, "non-octal or missing braces"),
    (b"\\c\xc3\xa9", 0, "\\c must be followed by an ASCII character"), (b"[\\x{2000}-a]", 0, "Invalid range"),
    ("(.{100}){9}😀".encode(), 0, "too large")])
def test_refusals(hs, pat, flags, msg):
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi([pat], [flags | UTF8], [1])
    assert msg in str(e.value), str(e.value)


def _info(hs, pat, flags, ext=None):
    L = hs.lib()
    out = C.POINTER(Info)()
    err = C.POINTER(hs.CompileError)()
    x = None
    if ext:
        x = hs.ExprExt()
        for k, v in ext.items():
            x.flags |= {"min_offset": 1, "max_offset": 2, "min_length": 4}[k]
            setattr(x, k, v)
    L.hs_expression_ext_info.argtypes = [C.c_char_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = L.hs_expression_ext_info(pat.encode(), flags | UTF8, C.byref(x) if x else None, C.byref(out), C.byref(err))
    assert rc == 0, pat
    got = (out.contents.min_width, out.contents.max_width)
    C.CDLL(None).free(C.cast(out, C.c_void_p))
    return got


def test_expression_info_counts_bytes(hs):
    INF = 0xffffffff
    for pat, ext, want in [("é", None, (2, 2)), ("空😀", None, (7, 7)), (".", None, (1, 4)), ("[^a]x", None, (2, 5)),
                           ("\\W{2}", None, (2, 8)), ("a\\Cb", None, (3, 3)), ("[ü€]+", None, (2, INF)),
                           ("\\x{10000}?z", None, (1, 5)), ("é.*", {"min_length": 9}, (9, INF)),
                           ("😀.", {"max_offset": 6}, (5, 6))]:
        assert _info(hs, pat, 0, ext) == want, pat


@pytest.mark.parametrize("pat,fl,py,ext", [
    ("é.+z", 0, "é.+z", {"min_length": 6}), ("[^a]{2}q", 0, "[^a]{2}q", {"min_offset": 20}),
    ("😀\\w", 0, "😀" + W, {"max_offset": 40}), ("€.*!", DOTALL, "(?s:€.*!)", {"min_offset": 10, "max_offset": 90}),
    ("\\W+x", 0, NW + "+x", {"min_length": 5})])
def test_extended_parameters_count_bytes(hs, ref, pat, fl, py, ext):
    hits = 0
    for dfa in (1, 0):
        db = _compile(hs, pat, fl, ext=ext, dfa=dfa)
        for seed in range(6):
            text = _text(500 + seed, 50) + "é😀a! €€ x"
            want = [(7, e) for e in _ends(py, text, **ext)]
            assert _ref_ends(ref, db, text.encode()) == want, (pat, ext, text)
            hits += len(want)
    assert hits > 0


def test_single_match_and_shared_ids(hs, ref):
    pats = ["é+", "[^a-z]😀", "空.", "x\\Wy"]
    flags = [SINGLE | UTF8, UTF8, SINGLE | UTF8, UTF8]   # id 1: single-match over two expressions
    ids = [1, 2, 1, 3]
    db = hs.compile_multi([p.encode() for p in pats], flags, ids)
    for seed in range(8):
        text = _text(900 + seed, 60) + "éé x😀 空空 x€y"
        want = set()
        for p, f, i in zip(pats, flags, ids):
            e = _ends(re.sub(r"\\W", NW, p), text)
            want |= {(i, x) for x in (e[:1] if f & SINGLE else e)}
        got = _ref_ends(ref, db, text.encode())
        assert sorted(got, key=lambda t: (t[1], t[0])) == _single(want, flags, ids)


def _single(want, flags, ids):
    """the report rules: an id that some expression raises with HS_FLAG_SINGLEMATCH is delivered once (its first
    end over all its expressions)"""
    single = {i for f, i in zip(flags, ids) if f & SINGLE}
    out, seen = [], set()
    for i, e in sorted(want, key=lambda t: (t[1], t[0])):
        if i in single:
            if i in seen:
                continue
            seen.add(i)
        out.append((i, e))
    return out


with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hscollider_utf8.json")) as _f:
    GOLDEN = json.load(_f)


def test_golden_summary():
    """the generator kept the UTF-8 lines it could compile and counted why it skipped the others"""
    assert GOLDEN["lines"] == 167 and GOLDEN["kept"] == len(GOLDEN["cases"])
    assert GOLDEN["kept"] + sum(GOLDEN["skipped"].values()) == 167


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[str(c["id"]) for c in GOLDEN["cases"]])
def test_golden_recorded_vectors(hs, ref, case):
    """the reference's recorded offsets for its own UTF-8 test expressions, on the database compiled here"""
    db = hs.compile_ext_multi([base64.b64decode(case["pattern"])], [case["hs_flags"]], [case["id"]], [case["ext"]])
    assert db.info().runtime_impl == case["runtime_impl"]
    for c in case["corpora"]:
        tos = [e for _, e in _ref_ends(ref, db, base64.b64decode(c["data"]))]
        if "H" in case["flag_letters"]:
            assert (len(tos) == 1 and tos[0] in c["ends"]) if c["ends"] else not tos
        else:
            assert tos == c["ends"]


# ---- device --------------------------------------------------------------------------------------------------------

DEVICE_SET = [("é+x", 0, 1), ("a.c", DOTALL, 2), ("[^a-z]{2}q", 0, 3), ("\\W\\D", SINGLE, 4), ("😀{2,}", 0, 5),
              ("\\bab+\\b", 0, 6), ("[à-ÿ€-₿]+z", 0, 7), ("(?i)k[s-t]", 0, 8), ("€$", 0, 9), ("空.", 0, 2)]


def _set_db(hs, dfa, exprs=DEVICE_SET):
    hs.set_build_option("regex_dfa", dfa)
    try:
        return hs.compile_multi([p.encode() for p, _, _ in exprs], [f | UTF8 for _, f, _ in exprs],
                                [i for _, _, i in exprs])
    finally:
        hs.set_build_option("regex_dfa", 1)


def _utf8_blocks(seed, lengths):
    rng = np.random.default_rng(seed)
    out = []
    for n in lengths:
        t = "".join(ALPHA[int(i)] for i in rng.integers(0, len(ALPHA), size=n))
        out.append((t + "ééx aéc €€q 😀😀 abb 空x kS €").encode()[:max(0, 3 * n)])
    return out


def _device_paths(hs, db, blocks):
    """per-block delivered matches through hs_scan, scan_blocks, scan_blocks_collect, a resident corpus with
    hs_b200_fetch_matches, and hs_b200_order_matches_async"""
    from test_gpu_device_order import _alloc, _read
    data, off, ln = _pack(blocks)
    scratch = hs.Scratch(db)
    paths = {"scan_blocks": _per_block(hs.scan_blocks(db, data, off, ln, scratch), len(blocks))}
    out = np.zeros(1 << 16, dtype=hs.MATCH_DTYPE)
    k = hs.scan_blocks_collect(db, data, off, ln, scratch, out)
    paths["collect"] = _per_block(out[:k], len(blocks))
    per = []
    for b in blocks:
        rc, got = hs.scan(db, b, scratch)
        assert rc == hs.HS_SUCCESS
        per.append(sorted((to, i) for i, to in got))
    paths["hs_scan"] = per
    corpus = hs.Corpus.upload(data, off, ln)
    paths["fetch"] = _per_block(hs.scan_corpus(db, corpus, scratch), len(blocks))
    hs.scan_corpus_async(db, corpus, scratch)
    cap = 1 << 16
    o, cnt = _alloc(cap)
    hs.order_matches_async(db, scratch, o, cnt, cap=cap)
    recs, _ = _read(hs, o, cnt, cap)
    paths["order"] = _per_block(recs, len(blocks))
    corpus.free()
    scratch.free()
    return paths


@pytest.mark.gpu
@pytest.mark.parametrize("dfa", [1, 0])
def test_device_equals_reference(hs, ref, dfa):
    db = _set_db(hs, dfa)
    assert db.info().runtime_impl == 2 and db.info().engine_id in ((6, 7) if dfa else (0, 1, 2, 3, 5))
    blocks = _utf8_blocks(1 + dfa, [0, 1, 3, 17, 64, 100, 300, 1000, 40])
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    for name, got in _device_paths(hs, db, blocks).items():
        assert got == want, name


@pytest.mark.gpu
def test_device_split_set_and_literals_beside_an_engine(hs, ref):
    """a set too large for one automaton (several engines), and literals with a UTF-8 engine (mixed_rose=1)"""
    big = [("%s[^a]{%d}%s" % (c, 20 + k, c), 0, 100 + k) for k, c in enumerate("éü€空😀𒀀ÿĀ₿")]
    db = _set_db(hs, 1, big + DEVICE_SET)
    assert db.info().runtime_impl == 0 and db.info().engine_count >= 2
    blocks = _utf8_blocks(5, [200, 900, 0, 50, 2000])
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    assert _device_paths(hs, db, blocks)["fetch"] == want
    hs.set_build_option("mixed_rose", 1)
    try:
        exprs = ["ü€", "空空", "abb", "😀😀"]
        db = hs.compile_multi([e.encode() for e in exprs] + [p.encode() for p, _, _ in DEVICE_SET],
                              [UTF8] * 4 + [f | UTF8 for _, f, _ in DEVICE_SET],
                              [50, 51, 52, 53] + [i for _, _, i in DEVICE_SET])
    finally:
        hs.set_build_option("mixed_rose", 0)
    assert db.info().runtime_impl == 0 and db.info().engine_count == 1
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    for name, got in _device_paths(hs, db, blocks).items():
        assert got == want, name


@pytest.mark.gpu
@pytest.mark.parametrize("seg", [16, 64, 1000])
@pytest.mark.parametrize("dfa", [1, 0])
def test_device_segment_seams_inside_characters(hs, ref, seg, dfa):
    """forced engine_segment lengths: 2-, 3- and 4-byte characters planted so that seams fall after their first,
    second and third bytes"""
    from test_gpu_engine_segments import _device
    db = _set_db(hs, dfa)
    blocks = [bytearray(b) for b in _utf8_blocks(9 + seg, [6000, 3000])]
    for b in blocks:
        k = 1
        for ch in ("é", "€", "😀", "😀", "€", "😀"):
            enc = ch.encode()
            for cut in range(1, len(enc)):
                at = k * seg - cut
                if at + len(enc) + 2 < len(b):
                    b[at - 1:at + len(enc) + 1] = b"a" + enc + b"x"
                k += 1
    blocks = [bytes(b) for b in blocks]
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    assert _device(hs, db, blocks, -1) == want
    got, st = _device(hs, db, blocks, seg, stats=True)
    assert got == want and st["segments"] > len(blocks)
