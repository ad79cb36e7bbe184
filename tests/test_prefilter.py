"""Prefilter mode (HS_FLAG_PREFILTER): an expression is rewritten into one whose matches are a superset of its own
(regex_nfa.cpp; the reference's src/parser/prefilter.cpp), and reduced until its automaton fits an engine.

CPU half: the rewrites give byte for byte the database of the hand-rewritten expression; the UNMODIFIED reference
hs_scan on the prefiltered databases reports every match end Python's re finds for the original expression (and
exactly those where the expression has nothing to rewrite); large repeats compile and stay supersets; the errors
and hs_expression_info rows.  GPU half: the device equals the reference on prefiltered sets of every database shape
and through every scan entry point."""
import base64
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from test_expr_info import Info

PREFILTER, CASELESS, DOTALL, SINGLE, SOM, COMBINATION = 128, 1, 2, 8, 256, 512
INF = 0xffffffff
HERE = os.path.dirname(os.path.abspath(__file__))
ENGINE = rb"zq+y"   # a companion expression that is no finite set of literals: the set takes the regex route


def _ends(pat, data, flags=0):
    """every end e such that the expression matches some data[s:e] in the context of the whole data"""
    fl = (re.I if flags & CASELESS else 0) | (re.S if flags & DOTALL else 0)
    out = []
    for e in range(1, len(data) + 1):
        rx = re.compile(b"(?:" + pat + b")(?<=(?s:\\A.{%d}))" % e, fl)
        if any(rx.match(data, s) for s in range(e)):
            out.append(e)
    return out


def _ref_ends(ref, db, data, block_ids=None):
    a = np.frombuffer(data, dtype=np.uint8) if data else np.zeros(0, np.uint8)
    r = ref.scan_sorted(db.ptr, a, np.array([0], np.uint64), np.array([len(data)], np.uint32))
    return [(int(x["id"]), int(x["to"])) for x in r]


# ---- rewrites, by bytes ----------------------------------------------------------------------------------------------

REWRITES = [
    (rb"(a)\1", rb"(a)a"), (rb"(ab)\1c", rb"(ab)[\x00-\xff]*c"), (rb"foo(?!bar)x", rb"foox"), (rb"(?>a+)b", rb"(a+)b"),
    (rb"a++b", rb"a+b"), (rb"(a)?(?(1)b|c)", rb"(a)?(b|c)"),
    # named groups and every spelling of a back-reference
    (rb"(?<n>a)\k<n>", rb"(a)a"), (rb"(?'n'a)\k'n'x", rb"(a)ax"), (rb"(?P<n>[ab])(?P=n)", rb"([ab])[ab]"),
    (rb"(?<n>a)\k{n}", rb"(a)a"), (rb"(?<n>a)\g{n}", rb"(a)a"), (rb"(a)\g1", rb"(a)a"), (rb"(a)\g{1}", rb"(a)a"),
    (rb"(a)(b)\g{-2}", rb"(a)(b)a"), (rb"(a)(b)\g-1", rb"(a)(b)b"), (rb"\2(a)(bc)", rb"[\x00-\xff]*(a)(bc)"),
    (rb"(a)(b)(c)(d)(e)(f)(g)(h)(i)(j)(k)\11", rb"(a)(b)(c)(d)(e)(f)(g)(h)(i)(j)(k)k"),
    (rb"(a)\12x", rb"(a)\nx"), (rb"(a+)\1", rb"(a+)a+"), (rb"(a{2})\1", rb"(a{2})[\x00-\xff]*"),
    (rb"(a|b)\1", rb"(a|b)[\x00-\xff]*"), (rb"(a\1)b", rb"(a[\x00-\xff]*)b"),
    # look-around, atomic groups, possessive quantifiers, conditionals
    (rb"x(?<=a)y(?<!b)z(?=c)", rb"xyz"), (rb"a?+b{2,3}+c*+", rb"a?b{2,3}c*"), (rb"(?>ab|a)c", rb"(ab|a)c"),
    (rb"(a)?(?(1)b)c", rb"(a)?(b|)c"), (rb"(?<q>a)?(?(<q>)b|c)d", rb"(a)?(b|c)d"), (rb"(?'q'a)?(?('q')b|c)d", rb"(a)?(b|c)d"),
    (rb"(?<q>a)?(?(q)b|c)", rb"(a)?(b|c)"), (rb"x(?(?=a)ab|cd)", rb"x(ab|cd)"), (rb"x(?(?<!a)ab|cd)", rb"x(ab|cd)"),
    (rb"(a)x(?(1))y", rb"(a)xy"), (rb"(?(DEFINE)a)bc", rb"(a|)bc"), (rb"(?=(a))\1b", rb"ab"),
]


def _db_bytes(hs, pat, flags):
    return hs.compile_multi([pat, ENGINE], [flags, 0], [1, 2]).serialize()


@pytest.mark.parametrize("pat,plain", REWRITES, ids=[str(i) for i in range(len(REWRITES))])
def test_rewrite_is_the_hand_rewritten_expression(hs, pat, plain):
    """with an expression beside it that needs an engine, the set's one automaton holds the rewritten expression"""
    assert _db_bytes(hs, pat, PREFILTER) == _db_bytes(hs, plain, 0), pat


def test_rewrite_alone_and_in_utf8_mode(hs):
    assert hs.compile_multi([rb"(a)\1b+"], [PREFILTER], [1]).serialize() == \
        hs.compile_multi([rb"(a)ab+"], [0], [1]).serialize()
    UTF8 = 32
    for pat, plain in [("(é)\\1x+", "(é)[\\x00-\\xff]*x+"), ("\\Xz", "(?s:.+)z"), ("(?<=é)ab+", "ab+")]:
        a = hs.compile_multi([pat.encode()], [PREFILTER | UTF8], [1]).serialize()
        b = hs.compile_multi([plain.encode()], [UTF8], [1]).serialize() if "\\x00" not in plain else \
            hs.compile_multi([b"(\xc3\xa9)\\C*x+"], [UTF8], [1]).serialize()
        assert a == b, pat


def test_named_groups_without_the_flag(hs):
    for pat, plain in [(rb"(?<n>ab+)c", rb"(ab+)c"), (rb"(?'n'a)(?P<m>b+)", rb"(a)(b+)")]:
        assert hs.compile_multi([pat], [0], [1]).serialize() == hs.compile_multi([plain], [0], [1]).serialize()


def test_expressions_without_the_constructs_keep_their_bytes(hs):
    """every expression of the hscollider fixture that compiles without the flag compiles to the same bytes with it"""
    with open(os.path.join(HERE, "golden", "hscollider_regex.json")) as f:
        cases = json.load(f)["cases"]
    n = 0
    for case in cases:
        pat, fl, ext = base64.b64decode(case["pattern"]), case["hs_flags"], case["ext"]
        if fl & (PREFILTER | SOM):
            continue
        try:
            plain = hs.compile_ext_multi([pat], [fl], [1], [ext]).serialize()
        except hs.HsError:
            continue
        assert hs.compile_ext_multi([pat], [fl | PREFILTER], [1], [ext]).serialize() == plain, pat
        n += 1
    assert n >= 200


# ---- superset on the reference runtime --------------------------------------------------------------------------------

class _Gen:
    """seeded random expressions over "abc": back-references (numbered and named, in the spellings Python's re also
    reads), the four look-arounds, atomic groups, possessive quantifiers and conditionals mixed with classes,
    groups, alternation and repeats; `kinds` names the constructs an expression has"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.groups = 0
        self.closed = []   # (number, name or None)
        self.kinds = set()

    def pick(self, *xs):
        return xs[int(self.rng.integers(0, len(xs)))]

    def atom(self, depth):
        r = self.rng.random()
        if r < 0.35 or depth > 2:
            return self.pick(b"a", b"b", b"c", b"[ab]", b"[^a]", b".")
        if r < 0.5:
            self.groups += 1
            g = self.groups
            name = b"g%d" % g if self.rng.random() < 0.4 else None
            body = self.alt(depth + 1)
            self.closed.append((g, name))
            return (b"(?P<" + name + b">" if name else b"(") + body + b")"
        if r < 0.6 and self.closed:
            g, name = self.pick(*self.closed)
            if name and (g > 7 or self.rng.random() < 0.6):
                self.kinds.add("named reference")
                return b"(?P=" + name + b")"
            if g <= 7:   # (the reference reads \\8 and \\9 as the digits, where Python's re reads a reference)
                self.kinds.add("numbered reference")
                return b"\\%d" % g
            return b"c"
        if r < 0.7:
            self.kinds.add("look-ahead")
            look = self.pick(b"(?=", b"(?!")
            return look + self.alt(depth + 1) + b")"
        if r < 0.76:
            self.kinds.add("look-behind")
            return self.pick(b"(?<=", b"(?<!") + self.pick(b"a", b"b", b"[bc]", b"ab", b"c.") + b")"
        if r < 0.86:
            self.kinds.add("atomic group")
            return b"(?>" + self.alt(depth + 1) + b")"
        if self.closed:
            self.kinds.add("conditional")
            g, _ = self.pick(*self.closed)
            no = self.pick(b"", b"|" + self.seq(depth + 1))
            return b"(?(%d)" % g + self.seq(depth + 1) + no + b")"
        return b"b"

    def seq(self, depth):
        out = b""
        for _ in range(int(self.rng.integers(1, 4))):
            a = self.atom(depth)
            if a[:1] == b"(" and (b"*" in a or b"+" in a):   # no nested unbounded repeats: re backtracks for ever
                q = self.pick(b"", b"", b"?", b"{2}")
            else:
                q = self.pick(b"", b"", b"", b"?", b"*", b"+", b"{1,2}", b"{2}")
            if q and self.rng.random() < 0.3:
                q += b"+"
                self.kinds.add("possessive")
            out += a + q
        return out

    def alt(self, depth):
        s = self.seq(depth)
        if self.rng.random() < 0.25:
            s += b"|" + self.seq(depth)
        return s


def _cases(n, seed0):
    out = []
    for i in range(n):
        g = _Gen(seed0 + i)
        pat = g.alt(0)
        try:
            re.compile(pat)
        except re.error:
            continue
        out.append((pat, g.kinds, seed0 + i))
    return out


KINDS = ("numbered reference", "named reference", "look-ahead", "look-behind", "atomic group", "conditional", "possessive")


@pytest.mark.parametrize("part", range(6))
def test_superset_on_the_reference_runtime(hs, ref, part):
    """4 200 seeded expressions in six parts (those Python's re reads and that match more than the empty buffer
    once rewritten are checked); the first violation fails the part, and every construct is checked in every part"""
    checked = exact = 0
    per_kind = dict.fromkeys(KINDS, 0)
    for pat, kinds, seed in _cases(700, 10000 + 1000 * part):
        try:
            db = hs.compile_multi([pat], [PREFILTER], [7])
        except hs.HsError as e:
            assert "empty buffer" in str(e) or "can never match" in str(e), (pat, str(e))
            continue
        rng = np.random.default_rng(seed)
        data = bytes(np.frombuffer(b"abc\n", np.uint8)[rng.integers(0, 4, size=24)])
        want = _ends(pat, data)
        got = [e for _, e in _ref_ends(ref, db, data)]
        assert set(want) <= set(got), (pat, data, want, got)
        if not kinds:
            assert got == want, (pat, data)
            exact += 1
        for k in kinds:
            per_kind[k] += 1
        checked += 1
    assert checked > 250 and exact > 20 and min(per_kind.values()) >= 15, (checked, exact, per_kind)


def _pcre():
    with open(os.path.join(HERE, "golden", "hscollider_prefilter.json")) as f:
        return json.load(f)


_PCRE_IDS = [c["id"] for c in _pcre()["cases"]]


def test_pcre_fixture_summary():
    """the generator kept the lines only prefilter mode compiles and counted why it skipped the others"""
    d = _pcre()
    assert d["kept"] == len(d["cases"]) >= 70 and d["kept_flagged_P"] >= 40 and d["flagged_P"] >= 41
    assert d["kept"] + sum(d["skipped"].values()) == d["lines"]


@pytest.mark.parametrize("ci", range(len(_PCRE_IDS)), ids=[str(i) for i in _PCRE_IDS])
def test_recorded_pcre_offsets_are_reported(hs, ref, ci):
    """every offset PCRE recorded for the reference's own test expressions is among the reference runtime's
    offsets on the prefiltered database compiled here"""
    case = _pcre()["cases"][ci]
    db = hs.compile_multi([base64.b64decode(case["pattern"])], [case["hs_flags"]], [case["id"]])
    for c in case["corpora"]:
        got = {e for _, e in _ref_ends(ref, db, base64.b64decode(c["data"]))}
        assert set(c["ends"]) <= got, c


# ---- size reduction ---------------------------------------------------------------------------------------------------

def _long_ends(pat, data, last):
    """ends of an expression without look-around, only where the data has `last` (the byte every match ends with)"""
    rx = re.compile(b"(?:" + pat + b")\\Z")
    return [e for e in range(1, len(data) + 1) if data[e - 1] == last and rx.search(data[:e])]


def _plant(seed, n, parts):
    rng = np.random.default_rng(seed)
    data = bytearray(np.frombuffer(b"abcdq\nxz", np.uint8)[rng.integers(0, 8, size=n)])
    for at, s in parts:
        data[at:at + len(s)] = s
    return bytes(data)


LARGE = [
    (rb"q[a-d]{600}z", b"z", [(10, b"q" + b"abcd" * 150 + b"z"), (700, b"q" + b"ab" * 200 + b"z"), (1200, b"q" + b"a" * 599 + b"z")]),
    (rb"[^\n]{300,}x", b"x", [(0, b"a" * 400 + b"x"), (900, b"\n" + b"b" * 250 + b"x")]),
    (rb"(a{40}){40}b+", b"b", [(0, b"a" * 1600 + b"bbb"), (1700, b"a" * 100 + b"b")]),
    (rb"(?:[ab]c){255}", b"c", [(0, b"ac" * 255), (600, b"bc" * 200)]),   # exactly 510 positions: no reduction
    (rb"(?:[ab]c){256}", b"c", [(0, b"ac" * 256), (600, b"bc" * 200)]),   # one position over
    (rb"x[^y]{60000}", b"", []),                                          # beyond the repeats that unroll
]


@pytest.mark.parametrize("pi", range(len(LARGE)))
def test_large_repeats_compile_and_stay_supersets(hs, ref, pi):
    pat, last, parts = LARGE[pi]
    db = hs.compile_multi([pat], [PREFILTER], [7])
    if not parts:
        return
    data = _plant(pi, 2400, parts)
    want = _long_ends(pat, data, last[0])
    got = [e for _, e in _ref_ends(ref, db, data)]
    assert want and set(want) <= set(got), pat


def test_large_repeats_without_the_flag_keep_their_errors(hs):
    for pat, msg in [(rb"q[a-d]{600}z", "too large"), (rb"(a{40}){40}b+", "too large"), (rb"[a-z]{600}x+", "too large"),
                     (rb"(?:[ab]c){256}", "too large")]:
        with pytest.raises(hs.HsError) as e:
            hs.compile_multi([pat], [0], [1])
        assert msg in str(e.value).lower()
    assert hs.compile_multi([rb"(?:[ab]c){255}"], [PREFILTER], [1]).serialize() == \
        hs.compile_multi([rb"(?:[ab]c){255}"], [0], [1]).serialize()


def test_min_length_beyond_the_model(hs, ref):
    ext = [{"min_length": 600}]
    with pytest.raises(hs.HsError):
        hs.compile_ext_multi([rb"a.{600}b"], [0], [1], ext)
    db = hs.compile_ext_multi([rb"a.{600}b"], [PREFILTER], [1], ext)
    data = _plant(5, 1500, [(3, b"a" + b"c" * 600 + b"b"), (800, b"a" + b"d" * 599 + b"b")])
    want = _long_ends(rb"a.{600}b", data, ord("b"))
    assert want and set(want) <= {e for _, e in _ref_ends(ref, db, data)}
    # a min_length that fits is kept, as without the flag
    small = [{"min_length": 6}]
    assert hs.compile_ext_multi([rb"a.*d"], [PREFILTER], [1], small).serialize() == \
        hs.compile_ext_multi([rb"a.*d"], [0], [1], small).serialize()


def test_referents_that_would_not_be_supersets(hs, ref):
    """a group that is one assertion is no referent, and a copy under HS_FLAG_CASELESS at the reference is folded:
    copied as they are, these would miss PCRE's matches"""
    for pat, data, ends in [(rb"(\b)a\1", b" ab", {2}), (rb"(^)a\1", b"ab", {1, 2}), (rb"(a)(?i)\1x+", b"aAx", {3})]:
        db = hs.compile_multi([pat], [PREFILTER], [1])
        assert ends <= {e for _, e in _ref_ends(ref, db, data)}, pat
        if b"(?i)" not in pat:   # (Python's re takes options at the start only; PCRE matches "aAx" at 3)
            assert set(_ends(pat, data)) <= ends, pat


def test_nested_repeats_of_nothing_stay_bounded(hs):
    """look-arounds and references have no positions; their copies still count toward the unrolling limit"""
    db = hs.compile_multi([rb"(?:(?:(?=a)){65535}){65535}b"], [PREFILTER], [1])
    assert db.serialize() == hs.compile_multi([rb"(?:(?:)+)+b"], [0], [1]).serialize()   # both widened to x{1,}


# ---- errors and expression info ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("pat,flags,msg", [
    (rb"(a)\1", PREFILTER | SOM, "HS_FLAG_PREFILTER is not supported in combination with HS_FLAG_SOM_LEFTMOST."),
    (rb"(abc)\2", PREFILTER, "Invalid back reference to expression 2."),
    (rb"(?<n>a)\k<m>", PREFILTER, "Invalid back reference to label 'm'."),
    (rb"(a)\g{-2}", PREFILTER, "Invalid reference."),
    (rb"a\g{0}", PREFILTER, "Numbered reference cannot be zero."),
    (rb"a\gx", PREFILTER, "Invalid reference after \\g."),
    (rb"a\g{12abc}", PREFILTER, "Invalid back reference to label '12abc'."),
    (rb"(a)\g{1234}", PREFILTER, "Invalid back reference to label '1234'."),
    (rb"abc(?(1)def|ghi)", PREFILTER, "Invalid conditional reference to expression 1."),
    (rb"abc(?(<blah>)def|ghi)", PREFILTER, "Invalid conditional reference to label 'blah'."),
    (rb"(a)(?(1)b|c|d)", PREFILTER, "Conditional with more than two branches."),
    (rb"(?(DEFINE)foo|bar)", PREFILTER, "DEFINE conditional group with more than one branch."),
    (rb"abc((def)?(?(R)bar))+", PREFILTER, "Pattern recursion not supported."),
    (rb"(?P<d>foo).*(?P<d>bar)", 0, "Two named subpatterns use the name 'd'."),
    (rb"(?P<d>foo).*(?P<d>bar)", PREFILTER, "Two named subpatterns use the name 'd'."),
    (rb"(?<1name>group)", 0, "Group name cannot begin with a digit."),
    (rb"(a|b)\1", 0, "Escape sequence \\1 is not supported."),
    (rb"(?=a)b", 0, "Look-around"), (rb"a++b", 0, "Possessive"), (rb"(?>a)b", 0, "Look-around"),
])
def test_errors(hs, pat, flags, msg):
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi([pat], [flags], [1])
    assert msg in str(e.value), str(e.value)


def test_prefilter_stays_refused_in_combinations_and_the_literal_api(hs):
    with pytest.raises(hs.HsError) as e:
        hs.compile_multi([rb"(a)\1b+", rb"ab+", rb"1 & 2"], [PREFILTER, 0, COMBINATION], [1, 2, 3])
    assert "Have PREFILTER flag in sub-expression." in str(e.value)
    with pytest.raises(hs.HsError) as e:
        hs.compile_lit_multi([b"abc"], [PREFILTER], [1])
    assert "literal API" in str(e.value)


def _info(hs, pat, flags):
    L = hs.lib()
    out = C.POINTER(Info)()
    err = C.POINTER(hs.CompileError)()
    L.hs_expression_info.argtypes = [C.c_char_p, C.c_uint, C.c_void_p, C.c_void_p]
    rc = L.hs_expression_info(pat, flags, C.byref(out), C.byref(err))
    assert rc == 0, pat
    i = out.contents
    got = (i.min_width, i.max_width) + tuple(ord(x) for x in (i.unordered_matches, i.matches_at_eod, i.matches_only_at_eod))
    C.CDLL(None).free(C.cast(out, C.c_void_p))
    return got


@pytest.mark.parametrize("pat,want", [
    (rb"foo(?=bar)", (3, 3, 0, 0, 0)), (rb"(ab)\1", (2, INF, 0, 0, 0)), (rb"(a)\1", (2, 2, 0, 0, 0)),
    (rb"(a)?\1b", (2, 3, 0, 0, 0)), (rb"x(?<!y)z", (2, 2, 0, 0, 0)), (rb"(?>ab|c)d", (2, 3, 0, 0, 0)),
    (rb"a{2,3}+b", (3, 4, 0, 0, 0)), (rb"(a)?(?(1)bc|d)", (1, 3, 0, 0, 0)), (rb"(a)(?(1)bc)", (1, 3, 0, 0, 0)),
    (rb"q[a-d]{600}z", (510, INF, 0, 0, 0)), (rb"a(?=b)$", (1, 1, 1, 1, 1)), (rb"(?<n>a+)\k<n>\b", (2, INF, 1, 1, 0)),
])
def test_expression_info(hs, pat, want):
    """worked out by hand on the rewritten, reduced expression"""
    assert _info(hs, pat, PREFILTER) == want, pat


# ---- device -----------------------------------------------------------------------------------------------------------

DEVICE_SET = [(rb"(['\"]).*?\1", 1), (rb"foo(?!bar)\w+", 2), (rb"(?<=a)b{2,}+c", 3), (rb"(?>x+)y", 4),
              (rb"(q)?(?(1)r|s)t", 5), (rb"(?P<w>[ab])(?P=w)c", 6), (rb"[^\n]{30,}!", 7), (rb"(a|b)\1z", 8)]


def _blocks(seed, lengths):
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(b"abcfoqrstxyz'\"!\n w", np.uint8)
    return [bytes(alpha[rng.integers(0, alpha.size, size=n)]) + b" 'ab' foobaz abbc xxy qrt st aac bbz" for n in lengths]


def _compile(hs, exprs, dfa=1, mixed=0):
    hs.set_build_option("regex_dfa", dfa)
    hs.set_build_option("mixed_rose", mixed)
    try:
        return hs.compile_multi([p for p, _ in exprs], [PREFILTER if b"(" in p or b"{" in p else 0 for p, _ in exprs],
                                [i for _, i in exprs])
    finally:
        hs.set_build_option("reset", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("dfa", [1, 0])
def test_device_single_outfix(hs, ref, dfa):
    from test_utf8 import _device_paths
    from test_mixed_rose import _ref_per_block
    exprs = DEVICE_SET if not dfa else [x for x in DEVICE_SET if x[1] != 7]   # [^\n]{30,}! keeps it out of a DFA
    db = _compile(hs, exprs, dfa)
    assert db.info().runtime_impl == 2 and db.info().engine_id in ((6, 7) if dfa else (0, 1, 2, 3, 5))
    blocks = _blocks(1 + dfa, [0, 1, 3, 17, 64, 100, 300, 1000, 40])
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    for name, got in _device_paths(hs, db, blocks).items():
        assert got == want, name


@pytest.mark.gpu
def test_device_split_set_and_literals_beside_an_engine(hs, ref):
    from test_utf8 import _device_paths
    from test_mixed_rose import _ref_per_block
    big = [(b"%s[^\\n]{%d}%s(?!%s)" % (c, 400 + k, c, c), 100 + k) for k, c in enumerate([b"a", b"b", b"q", b"x"])]
    db = _compile(hs, big + DEVICE_SET)
    assert db.info().runtime_impl == 0 and db.info().engine_count >= 2
    blocks = _blocks(5, [200, 900, 0, 50, 2000])
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    assert _device_paths(hs, db, blocks)["fetch"] == want
    db = _compile(hs, [(b"foobaz", 50), (b"qrt", 51), (b"xxy", 52)] + DEVICE_SET, mixed=1)
    assert db.info().runtime_impl == 0 and db.info().engine_count == 1
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    for name, got in _device_paths(hs, db, blocks).items():
        assert got == want, name


@pytest.mark.gpu
@pytest.mark.parametrize("seg", [16, 64, 1000])
@pytest.mark.parametrize("dfa", [1, 0])
def test_device_long_buffer_forced_segments(hs, ref, seg, dfa):
    """back-references as any-byte runs and widened repeats keep states live across every seam"""
    from test_gpu_engine_segments import _device
    from test_mixed_rose import _ref_per_block
    db = _compile(hs, DEVICE_SET + [(rb"q[a-d]{600}z", 9)], dfa)
    blocks = _blocks(9 + seg, [6000, 3000])
    blocks[0] = blocks[0][:100] + b"q" + b"abcd" * 150 + b"z" + blocks[0][702:]
    want = _ref_per_block(ref, db, blocks)
    assert sum(map(len, want)) > 50
    assert _device(hs, db, blocks, -1) == want
    got, st = _device(hs, db, blocks, seg, stats=True)
    assert got == want and st["segments"] > len(blocks)


