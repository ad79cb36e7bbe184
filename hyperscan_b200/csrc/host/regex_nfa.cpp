/* regex_nfa.cpp -- see regex_nfa.h */
#include "regex_nfa.h"

#include <algorithm>
#include <bitset>
#include <cstring>
#include <map>
#include <memory>
#include <tuple>

#include "../../../include/hs_b200.h"

namespace hsb {

namespace {

typedef std::bitset<256> CharSet;

struct Node {
    enum Kind { CLASS, CAT, ALT, STAR, PLUS, OPT, EMPTY, ASSERT } kind = EMPTY;
    int assertKind = 0;    /* ASSERT: one of the A_* bits below */
    bool unit = false;     /* the byte automaton of one UTF-8 character set: never split into top-level arms */
    unsigned ref = 0;      /* EMPTY standing for a back-reference (HS_FLAG_PREFILTER) to this group number ... */
    std::string refName;   /* ... or to this group name, until Parser::resolve replaces it */
    bool caseless = false; /* that back-reference is under HS_FLAG_CASELESS */
    CharSet cls;
    std::vector<std::shared_ptr<Node>> kids;
};
/* zero-width assertions; a path through several of them carries the union of their bits */
enum {
    A_WORD_B = 1,      /* \\b */
    A_NOT_WORD_B = 2,  /* \\B */
    A_BEGIN = 4,       /* \\A, "^": offset 0 */
    A_BEGIN_LINE = 8,  /* "^" under HS_FLAG_MULTILINE: offset 0 or right after a newline */
    A_END = 16,        /* \\z: end of the data */
    A_END_LF = 32,     /* "$", \\Z: end of the data, or before a newline that ends the data */
    A_END_LINE = 64,   /* "$" under HS_FLAG_MULTILINE: end of the data or before any newline */
    A_BOUNDARY = A_WORD_B | A_NOT_WORD_B,
    A_STARTS = A_BEGIN | A_BEGIN_LINE,
    A_ENDS = A_END | A_END_LF | A_END_LINE,
    A_ALL = 127
};
typedef std::shared_ptr<Node> NodeP;

NodeP mk(Node::Kind k) {
    NodeP n = std::make_shared<Node>();
    n->kind = k;
    return n;
}

NodeP clone(const NodeP &n) {
    NodeP c = std::make_shared<Node>(*n);
    for (NodeP &k : c->kids) {
        k = clone(k);
    }
    return c;
}

/* ---- UTF-8 mode ------------------------------------------------------------------------------
 * A set of code points is a sorted list of disjoint inclusive ranges.  It becomes a byte automaton:
 * every range is cut into runs whose UTF-8 encodings are a product of byte ranges (one range per
 * byte, 1 to 4 bytes), and those byte-range sequences form a tree that shares common suffixes,
 * whose leaves are ordinary character positions of the Glushkov construction. */
const u32 MAX_UNICODE = 0x10ffff;
typedef std::vector<std::pair<u32, u32>> Cps;

Cps cpsNorm(Cps s) {
    std::sort(s.begin(), s.end());
    Cps out;
    for (const auto &r : s) {
        if (!out.empty() && r.first <= out.back().second + 1) {
            out.back().second = std::max(out.back().second, r.second);
        } else {
            out.push_back(r);
        }
    }
    return out;
}

Cps cpsFlip(const Cps &in) { /* over [0, 0x10ffff], surrogates included, as the reference's CodePointSet::flip */
    const Cps s = cpsNorm(in);
    Cps out;
    u32 next = 0;
    for (const auto &r : s) {
        if (r.first > next) {
            out.push_back({next, r.first - 1});
        }
        next = r.second + 1;
    }
    if (next <= MAX_UNICODE) {
        out.push_back({next, MAX_UNICODE});
    }
    return out;
}

Cps cpsOf(const CharSet &c) {
    Cps s;
    for (u32 b = 0; b < 256; b++) {
        if (c[b]) s.push_back({b, b});
    }
    return cpsNorm(s);
}

typedef std::vector<std::pair<u8, u8>> ByteSeq; /* one inclusive byte range per byte of the encoding */

void utf8Encode(u32 c, u8 *out, int len) {
    static const u8 head[] = {0, 0, 0xc0, 0xe0, 0xf0};
    for (int i = len - 1; i > 0; i--) {
        out[i] = (u8)(0x80 | (c & 0x3f));
        c >>= 6;
    }
    out[0] = (u8)(len == 1 ? c : (head[len] | c));
}

/* the runs of [lo, hi] whose encodings are products of byte ranges */
void utf8Runs(u32 lo, u32 hi, std::vector<ByteSeq> *out) {
    static const u32 lim[] = {0x7f, 0x7ff, 0xffff};
    for (u32 l : lim) {
        if (lo <= l && hi > l) {
            utf8Runs(lo, l, out);
            utf8Runs(l + 1, hi, out);
            return;
        }
    }
    const int len = lo <= 0x7f ? 1 : lo <= 0x7ff ? 2 : lo <= 0xffff ? 3 : 4;
    for (int i = 1; i < len; i++) {
        const u32 m = (1u << (6 * i)) - 1;
        if ((lo & ~m) != (hi & ~m)) {
            if (lo & m) {
                utf8Runs(lo, lo | m, out);
                utf8Runs((lo | m) + 1, hi, out);
                return;
            }
            if ((hi & m) != m) {
                utf8Runs(lo, (hi & ~m) - 1, out);
                utf8Runs(hi & ~m, hi, out);
                return;
            }
        }
    }
    u8 a[4], b[4];
    utf8Encode(lo, a, len);
    utf8Encode(hi, b, len);
    ByteSeq s;
    for (int i = 0; i < len; i++) {
        s.push_back({a[i], b[i]});
    }
    out->push_back(s);
}

NodeP byteLeaf(u32 lo, u32 hi) {
    NodeP l = mk(Node::CLASS);
    for (u32 b = lo; b <= hi; b++) {
        l->cls[b] = true;
    }
    return l;
}

/* alternation of byte-range sequences (all non-empty), sharing common suffixes: the sequences are grouped by their
 * last byte range, and the ones whose prefix is used up merge into one position */
NodeP suffixTree(const std::vector<ByteSeq> &seqs) {
    std::map<std::pair<u8, u8>, std::vector<ByteSeq>> byLast;
    for (ByteSeq s : seqs) {
        const auto last = s.back();
        s.pop_back();
        byLast[last].push_back(s);
    }
    NodeP alt = mk(Node::ALT);
    NodeP single; /* the last byte of a sequence that has no prefix left */
    for (const auto &g : byLast) {
        std::vector<ByteSeq> rest;
        bool ends = false;
        for (const ByteSeq &s : g.second) {
            if (s.empty()) {
                ends = true;
            } else {
                rest.push_back(s);
            }
        }
        if (ends && rest.empty()) {
            if (!single) {
                single = mk(Node::CLASS);
                alt->kids.push_back(single);
            }
            single->cls |= byteLeaf(g.first.first, g.first.second)->cls;
            continue;
        }
        NodeP pre = suffixTree(rest);
        if (ends) {
            NodeP o = mk(Node::OPT);
            o->kids.push_back(pre);
            pre = o;
        }
        NodeP cat = mk(Node::CAT);
        cat->kids = {pre, byteLeaf(g.first.first, g.first.second)};
        alt->kids.push_back(cat);
    }
    return alt->kids.size() == 1 ? alt->kids[0] : alt;
}

} // namespace

bool validUtf8(const char *s, size_t len) {
    const u8 *p = (const u8 *)s;
    size_t i = 0;
    while (i < len) {
        const u8 c = p[i];
        const int n = c < 0x80 ? 1 : (c & 0xe0) == 0xc0 ? 2 : (c & 0xf0) == 0xe0 ? 3 : (c & 0xf8) == 0xf0 ? 4 : 0;
        if (!n || i + n > len) {
            return false;
        }
        u32 v = n == 1 ? c : c & (0x7f >> n);
        for (int k = 1; k < n; k++) {
            if ((p[i + k] & 0xc0) != 0x80) {
                return false;
            }
            v = (v << 6) | (p[i + k] & 0x3f);
        }
        static const u32 least[] = {0, 0, 0x80, 0x800, 0x10000};
        if (v < least[n] || v > MAX_UNICODE || (v >= 0xd800 && v <= 0xdfff)) {
            return false; /* overlong, beyond Unicode, or a surrogate */
        }
        i += n;
    }
    return true;
}

namespace {

/* HS_FLAG_PREFILTER: a bounded repeat the size reduction may widen, in parse order */
struct Repeat {
    size_t positions; /* what its copies contribute */
    unsigned lo;
};

class Parser {
public:
    /* widen (HS_FLAG_PREFILTER): per Repeat in parse order, -1 or the m' that x{m,n} becomes x{m',} with */
    Parser(const char *re_in, unsigned flags_in, const std::vector<long> *widen_in = nullptr)
        : re(re_in), n(strlen(re_in)), flags(flags_in), utf8(flags_in & HS_FLAG_UTF8),
          prefilter(flags_in & HS_FLAG_PREFILTER), widen(widen_in) {}

    std::vector<Repeat> repeats; /* HS_FLAG_PREFILTER: the repeats the reduction may widen */
    bool overflow = false;       /* HS_FLAG_PREFILTER: unrolling stopped early, the tree is too large */

    NodeP parse() {
        if (flags & HS_FLAG_UCP) {
            fail("HS_FLAG_UCP is not supported: Unicode character classes need the reference's Unicode property "
                 "tables.");
        }
        if (utf8 && !validUtf8(re, n)) {
            fail("Expression is not valid UTF-8.");
        }
        if (flags & HS_FLAG_SOM_LEFTMOST) {
            fail("HS_FLAG_SOM_LEFTMOST is not supported.");
        }
        NodeP r = alt();
        if (pos != n) {
            fail("Unmatched parentheses.");
        }
        /* references are checked once every group is known, as the reference's checkReferences does */
        for (unsigned c : condNums) {
            if (c >= groups) {
                fail("Invalid conditional reference to expression " + std::to_string(c) + ".");
            }
        }
        for (const std::string &c : condNames) {
            if (c != "DEFINE" && !names.count(c)) {
                fail("Invalid conditional reference to label '" + c + "'.");
            }
        }
        resolve(r);
        /* anchors only where the reference takes them (ComponentBoundary::checkEmbeddedStartAnchor / EndAnchor,
         * src/parser/ComponentBoundary.cpp:162-185, and the callers' rules in ComponentSequence / Alternation / Repeat) */
        embeddedStart(r, true);
        embeddedEnd(r, true);
        return r;
    }

private:
    const char *re;
    size_t n, pos = 0;
    unsigned flags;
    const bool utf8;      /* HS_FLAG_UTF8: characters are code points, encoded in 1 to 4 bytes */
    const bool prefilter; /* HS_FLAG_PREFILTER: back-references, look-around, atomic and conditional groups and
                           * possessive quantifiers are rewritten into a superset (src/parser/prefilter.cpp) */
    const std::vector<long> *widen;
    size_t unrolled = 0;  /* positions made by unrolling bounded repeats so far */
    bool quoting = false; /* between \\Q and \\E: every byte is a literal */
    unsigned groups = 1;  /* the number the next capturing group gets */
    std::vector<NodeP> referent = {nullptr}; /* per group: a copy of it when it is one position, else null */
    std::map<std::string, unsigned> names;   /* named groups */
    size_t refsSeen = 0;  /* back-references and conditionals so far: a group with one is no safe referent */
    std::vector<unsigned> condNums;
    std::vector<std::string> condNames;

    /* a back-reference becomes a copy of its group when that group is a single character position
     * (MAX_REFERENT_POSITIONS = 1 in the reference), else any byte sequence -- the reference's ".*" with DOTALL,
     * which under HS_FLAG_UTF8 is any sequence of whole characters.  Unlike the reference, a group that is one
     * assertion (its copy would assert again where PCRE asserts nothing) is no referent, and a copy under
     * HS_FLAG_CASELESS at the reference is folded (PCRE then compares the text caselessly), so the result is
     * always a superset. */
    void resolve(NodeP &x) {
        if (x->kind == Node::EMPTY && (x->ref || !x->refName.empty())) {
            unsigned g = x->ref;
            if (g && g >= groups) {
                fail("Invalid back reference to expression " + std::to_string(g) + ".");
            }
            if (!g) {
                const auto it = names.find(x->refName);
                if (it == names.end()) {
                    fail("Invalid back reference to label '" + x->refName + "'.");
                }
                g = it->second;
            }
            if (referent[g]) {
                NodeP copy = clone(referent[g]);
                if (x->caseless) {
                    foldTree(copy);
                }
                x = copy;
            } else {
                CharSet any;
                x = repeat(leaf(any.set()), 0, -1);
            }
            return;
        }
        for (NodeP &k : x->kids) {
            resolve(k);
        }
    }

    void foldTree(const NodeP &x) {
        const unsigned saved = flags;
        flags |= HS_FLAG_CASELESS;
        if (x->kind == Node::CLASS) {
            x->cls = fold(x->cls);
        }
        for (const NodeP &k : x->kids) {
            foldTree(k);
        }
        flags = saved;
    }

    NodeP backRef(unsigned g, const std::string &name = std::string()) {
        refsSeen++;
        NodeP b = mk(Node::EMPTY);
        b->ref = g;
        b->refName = name;
        b->caseless = flags & HS_FLAG_CASELESS;
        return b;
    }

    /* [A-Za-z0-9_]+ and then `term` at pos (pos moves past the terminator); false and pos unchanged if not */
    bool readName(char term, std::string *out) {
        size_t q = pos;
        while (q < n && (isalnum((unsigned char)re[q]) || re[q] == '_')) q++;
        if (q == pos || q >= n || re[q] != term) {
            return false;
        }
        out->assign(re + pos, q - pos);
        pos = q + 1;
        return true;
    }

    /* up to three decimal digits at pos */
    bool readNumber(unsigned *v) {
        size_t q = pos;
        unsigned x = 0;
        while (q < n && q < pos + 3 && isdigit((unsigned char)re[q])) x = x * 10 + (unsigned)(re[q++] - '0');
        if (q == pos) {
            return false;
        }
        pos = q;
        *v = x;
        return true;
    }

    /* HS_FLAG_PREFILTER, an escape at pos that is a back-reference (\\1..\\99 as PCRE reads them, \\g, \\k) or
     * \\X: its node; null (pos unchanged) for every other escape */
    NodeP prefilterEscape() {
        const size_t at0 = pos;
        const char e = re[pos + 1];
        if (e == 'X') { /* an extended grapheme cluster: one or more of any character */
            pos += 2;
            CharSet any;
            return repeat(utf8 ? unit({{0, MAX_UNICODE}}) : leaf(any.set()), 1, -1);
        }
        if (e >= '1' && e <= '9') {
            size_t q = pos + 1;
            u64 v = 0;
            while (q < n && isdigit((unsigned char)re[q])) v = std::min<u64>(v * 10 + (u64)(re[q++] - '0'), 1u << 20);
            if (q == pos + 2) { /* one digit: \\1..\\7 refer to a group, forward ones too; \\8 \\9 are not read here */
                if (e > '7') {
                    return nullptr;
                }
                pos = q;
                return backRef((unsigned)v);
            }
            if (v < groups) {
                pos = q;
                return backRef((unsigned)v);
            }
            /* not that many groups yet: up to three octal digits, then literal digits */
            pos++;
            u32 oct = 0;
            int digits = 0;
            while (digits < 3 && pos < q && re[pos] <= '7') oct = oct * 8 + (u32)(re[pos++] - '0'), digits++;
            NodeP s = mk(Node::CAT);
            auto lit = [&](u32 c) {
                CharSet one;
                one[c & 0xff] = true;
                s->kids.push_back(utf8 ? unit(foldU(c, c)) : leaf(fold(one)));
            };
            if (digits) lit(oct);
            while (pos < q) lit((u32)re[pos++]);
            return s;
        }
        std::string name;
        unsigned v = 0;
        if (e == 'g') {
            pos += 2;
            const bool brace = at('{');
            if (brace) pos++;
            const bool neg = at('-');
            if (neg) pos++;
            const size_t digits = pos;
            if (readNumber(&v) && (!brace || at('}'))) {
                pos += brace;
                if (v == 0) {
                    fail("Numbered reference cannot be zero.");
                }
                if (neg) {
                    if (v >= groups) {
                        fail("Invalid reference.");
                    }
                    v = groups - v;
                }
                return backRef(v);
            }
            pos = digits; /* \\g{name}: the name may begin with digits, as "12abc" */
            if (brace && !neg && readName('}', &name)) {
                return backRef(0, name);
            }
            pos = at0;
            fail("Invalid reference after \\g.");
        }
        if (e == 'k' && pos + 2 < n && strchr("<'{", re[pos + 2])) {
            pos += 3;
            const char open = re[pos - 1];
            if (readName(open == '<' ? '>' : open == '{' ? '}' : '\'', &name)) {
                return backRef(0, name);
            }
            pos = at0;
        }
        return nullptr;
    }

    /* HS_FLAG_PREFILTER, "(?(" at pos: a conditional group becomes the alternation of its branches (one branch
     * only: that branch or nothing) */
    NodeP conditional(unsigned saved) {
        pos += 2;
        refsSeen++;
        if (at('R') && pos + 1 < n && (isdigit((unsigned char)re[pos + 1]) || re[pos + 1] == '&' || re[pos + 1] == ')')) {
            fail("Pattern recursion not supported.");
        }
        std::string name;
        unsigned v = 0;
        bool define = false;
        if (isdigit((unsigned char)re[pos])) {
            size_t q = pos;
            while (q < n && isdigit((unsigned char)re[q])) v = std::min(v * 10 + (unsigned)(re[q++] - '0'), 1u << 20);
            if (q >= n || re[q] != ')') {
                fail("Conditional subpattern unsupported.");
            }
            if (v == 0) {
                fail("Numbered reference cannot be zero.");
            }
            pos = q + 1;
            condNums.push_back(v);
        } else if (at('?') && pos + 1 < n && (strchr("=!", re[pos + 1]) || (re[pos + 1] == '<' && pos + 2 < n && strchr("=!", re[pos + 2])))) {
            pos += re[pos + 1] == '<' ? 3 : 2; /* an assertion as the condition: it asserts nothing here */
            alt();
            if (!at(')')) {
                fail("Missing close parenthesis.");
            }
            pos++;
        } else {
            /* (?(<name>)...), (?('name')...), (?(name)...) */
            const char open = re[pos];
            const char close = open == '<' ? '>' : open == '\'' ? '\'' : ')';
            if (close != ')') pos++;
            if (!readName(close, &name) || (close != ')' && !at(')'))) {
                fail("Conditional subpattern unsupported.");
            }
            if (close != ')') pos++;
            define = name == "DEFINE";
            condNames.push_back(name);
        }
        std::vector<NodeP> arms = {seq()};
        while (at('|')) {
            pos++;
            arms.push_back(seq());
        }
        if (arms.size() > 2) {
            fail("Conditional with more than two branches.");
        }
        if (define && arms.size() == 2) {
            fail("DEFINE conditional group with more than one branch.");
        }
        if (!at(')')) {
            fail("Missing close parenthesis.");
        }
        pos++;
        flags = saved;
        if (arms.size() == 1 && arms[0]->kids.empty()) {
            return mk(Node::EMPTY);
        }
        if (arms.size() == 1) {
            arms.push_back(mk(Node::CAT));
        }
        NodeP a = mk(Node::ALT);
        a->kids = arms;
        return a;
    }

    [[noreturn]] void fail(const std::string &m) const { throw RegexError{m}; }
    bool at(char c) const { return pos < n && re[pos] == c; }

    /* the (validated) UTF-8 character at pos; pos moves past it */
    u32 readChar() {
        const u8 c = (u8)re[pos];
        const int len = c < 0x80 ? 1 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : 4;
        u32 v = len == 1 ? c : c & (0x7f >> len);
        for (int k = 1; k < len; k++) {
            v = (v << 6) | ((u8)re[pos + k] & 0x3f);
        }
        pos += len;
        return v;
    }

    /* UTF-8 mode, a character or range written in the expression under HS_FLAG_CASELESS: ASCII letters take their
     * other case, and "k" / "s" also the two non-ASCII characters that fold to them, KELVIN SIGN (U+212A) and LATIN
     * SMALL LETTER LONG S (U+017F), as the reference's case folding does.  Non-ASCII case folding needs Unicode
     * tables this compiler does not have. */
    Cps foldU(u32 lo, u32 hi) const {
        Cps s = {{lo, hi}};
        if (!(flags & HS_FLAG_CASELESS)) {
            return s;
        }
        if (hi >= 0x80) {
            fail("HS_FLAG_CASELESS on a non-ASCII character is not supported under HS_FLAG_UTF8: it needs Unicode "
                 "case folding.");
        }
        for (u32 c = lo; c <= hi; c++) {
            const u32 l = c | 0x20;
            if (l >= 'a' && l <= 'z') {
                s.push_back({l, l});
                s.push_back({l - 32, l - 32});
                if (l == 'k') s.push_back({0x212a, 0x212a});
                if (l == 's') s.push_back({0x17f, 0x17f});
            }
        }
        return cpsNorm(s);
    }

    /* a set of code points as a node: ASCII only, one position; else the byte automaton of the UTF-8 encodings */
    NodeP unit(const Cps &in) {
        const Cps s = cpsNorm(in);
        if (s.empty()) {
            fail("Empty character class.");
        }
        CharSet ascii;
        std::vector<ByteSeq> multi;
        for (const auto &r : s) {
            for (u32 c = r.first; c <= std::min<u32>(r.second, 0x7f); c++) {
                ascii[c] = true;
            }
            if (r.second >= 0x80) {
                utf8Runs(std::max<u32>(r.first, 0x80), r.second, &multi);
            }
        }
        if (multi.empty()) {
            return leaf(ascii);
        }
        NodeP m = suffixTree(multi);
        NodeP u = m;
        if (ascii.any()) {
            u = mk(Node::ALT);
            NodeP a = mk(Node::CLASS);
            a->cls = ascii;
            u->kids = {a, m};
        }
        u->unit = true;
        return u;
    }

    /* \\h / \\v under HS_FLAG_UTF8: PCRE's horizontal and vertical white space */
    static Cps spaceU(bool vertical) {
        if (vertical) {
            return {{0x0a, 0x0d}, {0x85, 0x85}, {0x2028, 0x2029}};
        }
        return {{0x09, 0x09}, {0x20, 0x20}, {0xa0, 0xa0}, {0x1680, 0x1680}, {0x180e, 0x180e},
                {0x2000, 0x200a}, {0x202f, 0x202f}, {0x205f, 0x205f}, {0x3000, 0x3000}};
    }

    /* an escape under HS_FLAG_UTF8: either one code point (*single) or a set; pos is at the backslash */
    Cps escapeU(bool inClass, long *single) {
        *single = -1;
        if (pos + 1 >= n) {
            fail("Unterminated escape at end of pattern.");
        }
        const unsigned char e = (unsigned char)re[pos + 1];
        switch (e) {
        case 'p': case 'P':
            fail("\\p / \\P (Unicode properties) are not supported: they need the reference's Unicode property "
                 "tables.");
        case 'X':
            fail("\\X (an extended grapheme cluster) is not supported: it needs the reference's Unicode property "
                 "tables.");
        case 'd': case 'D': case 'w': case 'W': case 's': case 'S': {
            pos += 2;
            const Cps s = cpsOf(classEscape((char)(e | 0x20)));
            return e >= 'a' ? s : cpsFlip(s);
        }
        case 'h': case 'H': case 'v': case 'V': {
            pos += 2;
            const Cps s = spaceU((e | 0x20) == 'v');
            return e >= 'a' ? s : cpsFlip(s);
        }
        case 'N':
            pos += 2;
            return cpsFlip({{'\n', '\n'}});
        case 'x': case 'o': {
            pos += 2;
            const bool hex = e == 'x';
            if (hex && !at('{')) { /* \\x and up to two hexadecimal digits */
                u32 v = 0;
                for (int k = 0; k < 2 && pos < n && hexval(re[pos]) >= 0; k++) {
                    v = v * 16 + (u32)hexval(re[pos++]);
                }
                *single = v;
                return {{v, v}};
            }
            size_t q = pos + 1;
            u64 v = 0;
            while (q < n && (hex ? hexval(re[q]) >= 0 : (re[q] >= '0' && re[q] <= '7'))) {
                v = std::min<u64>(v * (hex ? 16 : 8) + (u64)(hex ? hexval(re[q]) : re[q] - '0'), MAX_UNICODE + 1);
                q++;
            }
            if (!at('{') || q == pos + 1 || q >= n || re[q] != '}') {
                fail(hex ? "Value in \\x{...} sequence is non-hex or missing }"
                         : "Value in \\o{...} sequence is non-octal or missing braces");
            }
            if (v > MAX_UNICODE) {
                fail(hex ? "Value in \\x{...} sequence is too large" : "Value in \\o{...} sequence is too large");
            }
            pos = q + 1;
            *single = (long)v;
            return {{(u32)v, (u32)v}};
        }
        default:
            break;
        }
        if (inClass && e >= '1' && e <= '7') { /* octal, up to three digits: a code point up to \\777 */
            pos += 2;
            u32 v = e - '0';
            for (int k = 0; k < 2 && pos < n && re[pos] >= '0' && re[pos] <= '7'; k++) {
                v = v * 8 + (u32)(re[pos++] - '0');
            }
            *single = v;
            return {{v, v}};
        }
        if (e >= 0x80) { /* an escaped non-ASCII character is that character */
            pos++;
            const u32 v = readChar();
            *single = v;
            return {{v, v}};
        }
        int b;
        escape(inClass, &b); /* the rest name ASCII characters */
        *single = b;
        return {{(u32)b, (u32)b}};
    }

    Cps charClassU() {
        pos++; /* [ */
        bool negate = false;
        if (at('^')) {
            negate = true;
            pos++;
        }
        Cps set;
        bool first = true;   /* no member yet: a "]" is a literal */
        bool quoted = false; /* between \\Q and \\E */
        long prev = -1;
        auto add = [&](const Cps &s) { set.insert(set.end(), s.begin(), s.end()); };
        for (;;) {
            if (pos >= n) {
                fail("Unterminated character class.");
            }
            const unsigned char c = (unsigned char)re[pos];
            if (c == '\\' && pos + 1 < n && (re[pos + 1] == 'E' || (re[pos + 1] == 'Q' && !quoted))) {
                quoted = re[pos + 1] == 'Q';
                pos += 2;
                continue;
            }
            if (quoted) {
                prev = readChar();
                add(foldU((u32)prev, (u32)prev));
                first = false;
                continue;
            }
            if (c == ']' && !first) {
                pos++;
                break;
            }
            first = false;
            if (c == '[' && pos + 1 < n && re[pos + 1] == ':') {
                const char *close = strstr(re + pos + 2, ":]");
                if (!close) {
                    fail("Unterminated POSIX character class.");
                }
                std::string name(re + pos + 2, close);
                bool neg = false;
                if (!name.empty() && name[0] == '^') {
                    neg = true;
                    name.erase(0, 1);
                }
                CharSet pc;
                if (!posixClass(name, &pc)) {
                    fail("Unknown POSIX character class.");
                }
                const Cps s = cpsOf(fold(pc)); /* ASCII classes: ASCII case folding only */
                add(neg ? cpsFlip(s) : s);
                pos = (size_t)(close - re) + 2;
                prev = -1;
                continue;
            }
            if (c == '[' && pos + 1 < n && (re[pos + 1] == '.' || re[pos + 1] == '=')) {
                fail("POSIX collating elements are not supported.");
            }
            if (c == '-' && prev >= 0 && pos + 1 < n && re[pos + 1] != ']') {
                pos++;
                long hi;
                if (re[pos] == '[' && pos + 1 < n && strchr(":.=", re[pos + 1])) {
                    fail("Invalid range in character class.");
                }
                if (re[pos] == '\\') {
                    if (pos + 1 < n && (re[pos + 1] == 'Q' || re[pos + 1] == 'E')) {
                        fail("\\Q / \\E as the end of a range is not supported.");
                    }
                    escapeU(true, &hi);
                    if (hi < 0) {
                        fail("Invalid range in character class.");
                    }
                } else {
                    hi = readChar();
                }
                if (hi < prev) {
                    fail("Invalid range in character class.");
                }
                add(foldU((u32)prev, (u32)hi));
                prev = -1;
                continue;
            }
            if (c == '\\') {
                long single;
                const Cps e = escapeU(true, &single);
                add(single >= 0 ? foldU((u32)single, (u32)single) : e);
                prev = single;
            } else {
                prev = readChar();
                add(foldU((u32)prev, (u32)prev));
            }
        }
        return negate ? cpsFlip(set) : cpsNorm(set);
    }

    /* one atom under HS_FLAG_UTF8 that is not a group, a class, an assertion or an option: pos is at it */
    NodeP atomU() {
        const unsigned char c = (unsigned char)re[pos];
        if (quoting) {
            const u32 v = readChar();
            return unit(foldU(v, v));
        }
        if (c == '\\') {
            if (pos + 1 < n && re[pos + 1] == 'C') { /* \\C: one byte, whatever it is */
                pos += 2;
                CharSet any;
                return leaf(any.set());
            }
            long single;
            const Cps s = escapeU(false, &single);
            return unit(single >= 0 ? foldU((u32)single, (u32)single) : s);
        }
        if (c == '.') {
            pos++;
            return unit(flags & HS_FLAG_DOTALL ? Cps{{0, MAX_UNICODE}} : cpsFlip({{'\n', '\n'}}));
        }
        if (strchr("*+?", c) || (c == '{' && startsRepeat(pos))) {
            fail("Invalid repeat: nothing to repeat.");
        }
        const u32 v = readChar();
        return unit(foldU(v, v));
    }

    CharSet fold(CharSet s) const {
        if (flags & HS_FLAG_CASELESS) {
            for (int c = 'a'; c <= 'z'; c++) {
                if (s[c] || s[c - 32]) {
                    s[c] = s[c - 32] = true;
                }
            }
        }
        return s;
    }

    NodeP alt() {
        std::vector<NodeP> arms;
        arms.push_back(seq());
        while (at('|')) {
            pos++;
            arms.push_back(seq());
        }
        if (arms.size() == 1) {
            return arms[0];
        }
        NodeP a = mk(Node::ALT);
        a->kids = arms;
        return a;
    }

    NodeP seq() {
        NodeP s = mk(Node::CAT);
        while (pos < n && (quoting || (re[pos] != '|' && re[pos] != ')'))) {
            NodeP a = atom();
            a = quantified(a);
            s->kids.push_back(a);
        }
        return s;
    }

    /* may the match still start here (nothing consumed before on any way to this node)?  A start anchor
     * anywhere else is refused, as the reference does. */
    static bool embeddedStart(const NodeP &x, bool atStart) {
        switch (x->kind) {
        case Node::CLASS:
            return false;
        case Node::EMPTY:
            return atStart;
        case Node::ASSERT:
            if (x->assertKind & A_BOUNDARY) {
                return false;
            }
            if ((x->assertKind & A_STARTS) && !atStart) {
                throw RegexError{"Embedded start anchors not supported."};
            }
            return atStart;
        case Node::CAT:
            for (const NodeP &k : x->kids) {
                atStart = embeddedStart(k, atStart);
            }
            return atStart;
        case Node::ALT: {
            bool rv = true;
            for (const NodeP &k : x->kids) {
                rv &= embeddedStart(k, atStart);
            }
            return rv;
        }
        case Node::STAR:
        case Node::PLUS:
            atStart = embeddedStart(x->kids[0], atStart);
            return embeddedStart(x->kids[0], atStart);
        case Node::OPT:
            return embeddedStart(x->kids[0], atStart);
        }
        return false;
    }
    static bool embeddedEnd(const NodeP &x, bool atEnd) {
        switch (x->kind) {
        case Node::CLASS:
            return false;
        case Node::EMPTY:
            return atEnd;
        case Node::ASSERT:
            if (x->assertKind & A_BOUNDARY) {
                return false;
            }
            if ((x->assertKind & A_ENDS) && !atEnd) {
                throw RegexError{"Embedded end anchors not supported."};
            }
            return atEnd;
        case Node::CAT:
            for (auto k = x->kids.rbegin(); k != x->kids.rend(); ++k) {
                atEnd = embeddedEnd(*k, atEnd);
            }
            return atEnd;
        case Node::ALT: {
            bool rv = true;
            for (const NodeP &k : x->kids) {
                rv &= embeddedEnd(k, atEnd);
            }
            return rv;
        }
        case Node::STAR:
        case Node::PLUS:
            atEnd = embeddedEnd(x->kids[0], atEnd);
            return embeddedEnd(x->kids[0], atEnd);
        case Node::OPT:
            return embeddedEnd(x->kids[0], atEnd);
        }
        return false;
    }

    static bool hasAssert(const NodeP &x) {
        if (x->kind == Node::ASSERT) {
            return true;
        }
        for (const NodeP &k : x->kids) {
            if (hasAssert(k)) return true;
        }
        return false;
    }

    static size_t leaves(const NodeP &x) {
        size_t c = x->kind == Node::CLASS || x->kind == Node::ASSERT;
        for (const NodeP &k : x->kids) {
            c += leaves(k);
        }
        return c;
    }

    NodeP repeat(const NodeP &a, unsigned lo, long hi /* -1 = unbounded */) {
        const size_t copies = hi < 0 ? std::max<size_t>(lo, 1) : (size_t)hi;
        if (prefilter && copies > 1) { /* the size reduction may widen this one to x{m',} */
            const size_t i = repeats.size();
            repeats.push_back({leaves(a) * copies, lo});
            if (widen && i < widen->size() && (*widen)[i] >= 0) {
                lo = (unsigned)(*widen)[i];
                hi = -1;
            }
        }
        /* repeats are unrolled: refuse before copying what cannot fit the largest model anyway */
        /* (under HS_FLAG_PREFILTER a copy without positions, of a look-around or a reference, still costs a node:
         * the repeats may be 65 535 long there) */
        unrolled += std::max<size_t>(leaves(a), prefilter) * std::max<size_t>(hi < 0 ? lo + 1 : (size_t)hi, 1);
        if (unrolled > 4 * MAX_NFA_STATES) {
            if (prefilter) { /* the reduction widens repeats until the expression fits */
                overflow = true;
                return mk(Node::EMPTY);
            }
            fail("Pattern is too large.");
        }
        NodeP s = mk(Node::CAT);
        for (unsigned i = 0; i < lo; i++) {
            s->kids.push_back(clone(a));
        }
        if (hi < 0) {
            if (lo == 0) {
                NodeP st = mk(Node::STAR);
                st->kids.push_back(clone(a));
                s->kids.push_back(st);
            } else { /* x{n,} = x^(n-1) x+ */
                NodeP pl = mk(Node::PLUS);
                pl->kids.push_back(s->kids.back());
                s->kids.back() = pl;
            }
        } else {
            for (long i = lo; i < hi; i++) { /* x{n,m}: m - n optional copies (same language as the nested form) */
                NodeP o = mk(Node::OPT);
                o->kids.push_back(clone(a));
                s->kids.push_back(o);
            }
        }
        return s;
    }

    /* "{n}", "{n,}", "{n,m}" at q?  (anything else that starts with a brace is literal text) */
    bool startsRepeat(size_t q) const {
        if (q >= n || re[q] != '{') {
            return false;
        }
        size_t k = q + 1;
        while (k < n && isdigit((unsigned char)re[k])) k++;
        if (k == q + 1) {
            return false;
        }
        if (k < n && re[k] == ',') {
            k++;
            while (k < n && isdigit((unsigned char)re[k])) k++;
        }
        return k < n && re[k] == '}';
    }

    NodeP quantified(NodeP a) {
        while (pos + 1 < n && re[pos] == '\\' && re[pos + 1] == 'E') { /* "\\Qab\\E+": the quantifier binds to the "b" */
            quoting = false;
            pos += 2;
        }
        if (pos >= n || quoting) {
            return a;
        }
        const char c = re[pos];
        if (a->kind == Node::ASSERT && (c == '*' || c == '+' || c == '?' || c == '{')) {
            fail("A quantifier on an assertion is not supported.");
        }
        unsigned lo = 1;
        long hi = 1;
        if (c == '*') {
            pos++;
            lo = 0;
            hi = -1;
        } else if (c == '+') {
            pos++;
            lo = 1;
            hi = -1;
        } else if (c == '?') {
            pos++;
            lo = 0;
            hi = 1;
        } else if (c == '{') {
            size_t q = pos + 1;
            unsigned long x = 0, y = 0;
            bool haveX = false, haveY = false, comma = false;
            while (q < n && isdigit((unsigned char)re[q])) {
                x = std::min(x * 10 + (unsigned long)(re[q++] - '0'), 100000ul);
                haveX = true;
            }
            if (q < n && re[q] == ',') {
                comma = true;
                q++;
                while (q < n && isdigit((unsigned char)re[q])) {
                    y = std::min(y * 10 + (unsigned long)(re[q++] - '0'), 100000ul);
                    haveY = true;
                }
            }
            if (!haveX || q >= n || re[q] != '}') {
                return a; /* not a quantifier: the brace is a literal (atom() reads it next) */
            }
            if (comma && haveY && y < x) {
                fail("Bounded repeat is invalid: min > max.");
            }
            const unsigned long most = prefilter ? 65535 : 1000; /* PCRE's own limit, when repeats can be widened */
            if (x > most || (haveY && y > most)) {
                fail("Pattern is too large.");
            }
            pos = q + 1;
            lo = (unsigned)x;
            hi = !comma ? (long)x : haveY ? (long)y : -1;
        } else {
            return a;
        }
        if (pos < n && re[pos] == '?') {
            pos++; /* lazy: same set of match ends */
        } else if (pos < n && re[pos] == '+') {
            if (!prefilter) {
                fail("Possessive quantifiers are not supported.");
            }
            pos++; /* the greedy form: the same match ends and more */
        }
        if (lo == 1 && hi == 1) {
            return a;
        }
        if (lo == 0 && hi == 0) {
            return mk(Node::EMPTY);
        }
        return repeat(a, lo, hi);
    }

    static int hexval(char c) {
        if (c >= '0' && c <= '9') return c - '0';
        if (c >= 'a' && c <= 'f') return c - 'a' + 10;
        if (c >= 'A' && c <= 'F') return c - 'A' + 10;
        return -1;
    }

    static CharSet classEscape(char e) {
        CharSet s;
        switch (e | 0x20) {
        case 'd':
            for (int c = '0'; c <= '9'; c++) s[c] = true;
            break;
        case 'w':
            for (int c = '0'; c <= '9'; c++) s[c] = true;
            for (int c = 'a'; c <= 'z'; c++) s[c] = s[c - 32] = true;
            s['_'] = true;
            break;
        case 's': /* PCRE 8.41 \s: space, \t \n \v \f \r */
            s[' '] = s['\t'] = s['\n'] = s[0x0b] = s['\f'] = s['\r'] = true;
            break;
        }
        return (e >= 'A' && e <= 'Z') ? ~s : s;
    }

    static bool posixClass(const std::string &name, CharSet *out) { /* C locale, as PCRE */
        static const struct { const char *n; int (*f)(int); } tab[] = {
            {"alpha", isalpha}, {"digit", isdigit}, {"alnum", isalnum}, {"upper", isupper}, {"lower", islower},
            {"space", isspace}, {"punct", ispunct}, {"print", isprint}, {"graph", isgraph}, {"cntrl", iscntrl},
            {"xdigit", isxdigit}, {"blank", isblank}};
        for (const auto &t : tab) {
            if (name == t.n) {
                for (int c = 0; c < 128; c++) {
                    if (t.f(c)) (*out)[(size_t)c] = true;
                }
                return true;
            }
        }
        if (name == "word") {
            *out = classEscape('w');
            return true;
        }
        if (name == "ascii") {
            for (int c = 0; c < 128; c++) (*out)[(size_t)c] = true;
            return true;
        }
        return false;
    }

    /* an escape: either one character (*single) or a class */
    CharSet escape(bool inClass, int *single) {
        *single = -1;
        if (++pos >= n) {
            fail("Unterminated escape at end of pattern.");
        }
        const unsigned char e = (unsigned char)re[pos++];
        CharSet s;
        switch (e) {
        case 'n': *single = '\n'; break;
        case 't': *single = '\t'; break;
        case 'r': *single = '\r'; break;
        case 'f': *single = '\f'; break;
        case 'a': *single = '\a'; break;
        case 'e': *single = 0x1b; break;
        case 'd': case 'D': case 'w': case 'W': case 's': case 'S':
            return classEscape((char)e);
        case 'h': case 'H': /* horizontal white space, 8-bit: \t, space, 0xa0 */
            s['\t'] = s[' '] = s[0xa0] = true;
            return e == 'H' ? ~s : s;
        case 'v': case 'V': /* vertical white space, 8-bit: \n \v \f \r, 0x85 */
            s['\n'] = s[0x0b] = s['\f'] = s['\r'] = s[0x85] = true;
            return e == 'V' ? ~s : s;
        case 'N': /* not a newline, whatever HS_FLAG_DOTALL says */
            s.set();
            s['\n'] = false;
            return s;
        case 'x': {
            if (pos < n && re[pos] == '{') { /* \x{h..h} */
                size_t q = pos + 1;
                unsigned long v = 0;
                while (q < n && hexval(re[q]) >= 0) {
                    v = std::min(v * 16 + (unsigned long)hexval(re[q]), 0x10000ul);
                    q++;
                }
                if (q == pos + 1 || q >= n || re[q] != '}') {
                    fail("Invalid hex escape: \\x{ without hexadecimal digits and a closing brace.");
                }
                if (v > 0xff) {
                    fail("Hexadecimal value is greater than \\xFF.");
                }
                pos = q + 1;
                *single = (int)v;
                break;
            }
            int v = 0; /* \x followed by up to two hexadecimal digits (none: a NUL byte) */
            for (int k = 0; k < 2 && pos < n && hexval(re[pos]) >= 0; k++) {
                v = v * 16 + hexval(re[pos++]);
            }
            *single = v;
            break;
        }
        case 'c': { /* control character: the next byte, upper-cased, with bit 6 flipped */
            if (pos >= n) {
                fail("\\c at end of pattern.");
            }
            const unsigned char x = (unsigned char)re[pos++];
            if (x >= 128) {
                fail("\\c must be followed by an ASCII character.");
            }
            *single = toupper(x) ^ 0x40;
            break;
        }
        case '0': { /* \0 and up to two more octal digits */
            int v = 0;
            for (int k = 0; k < 2 && pos < n && re[pos] >= '0' && re[pos] <= '7'; k++) {
                v = v * 8 + (re[pos++] - '0');
            }
            *single = v;
            break;
        }
        default:
            if (inClass && e == 'b') {
                *single = 0x08;
            } else if (inClass && e >= '1' && e <= '7') { /* no back-references in a class: octal, up to three digits */
                int v = e - '0';
                for (int k = 0; k < 2 && pos < n && re[pos] >= '0' && re[pos] <= '7'; k++) {
                    v = v * 8 + (re[pos++] - '0');
                }
                *single = v & 0xff;
            } else if (isalnum(e)) {
                fail(std::string("Escape sequence \\") + (char)e + " is not supported.");
            } else {
                *single = e;
            }
        }
        s[(size_t)*single] = true;
        return s;
    }

    CharSet charClass() {
        pos++; /* [ */
        bool negate = false;
        if (at('^')) {
            negate = true;
            pos++;
        }
        CharSet set;
        bool first = true;   /* no member yet: a "]" is a literal */
        bool quoted = false; /* between \\Q and \\E */
        int prev = -1;
        for (;;) {
            if (pos >= n) {
                fail("Unterminated character class.");
            }
            const unsigned char c = (unsigned char)re[pos];
            if (c == '\\' && pos + 1 < n && (re[pos + 1] == 'E' || (re[pos + 1] == 'Q' && !quoted))) {
                quoted = re[pos + 1] == 'Q';
                pos += 2;
                continue;
            }
            if (quoted) {
                set[c] = true;
                prev = c;
                pos++;
                first = false;
                continue;
            }
            if (c == ']' && !first) {
                pos++;
                break;
            }
            first = false;
            if (c == '[' && pos + 1 < n && re[pos + 1] == ':') {
                const char *close = strstr(re + pos + 2, ":]");
                if (!close) {
                    fail("Unterminated POSIX character class.");
                }
                std::string name(re + pos + 2, close);
                bool neg = false;
                if (!name.empty() && name[0] == '^') {
                    neg = true;
                    name.erase(0, 1);
                }
                CharSet pc;
                if (!posixClass(name, &pc)) {
                    fail("Unknown POSIX character class.");
                }
                pc = fold(pc); /* under CASELESS [:upper:] and [:lower:] are all letters, THEN the "^" applies */
                set |= neg ? ~pc : pc;
                pos = (size_t)(close - re) + 2;
                prev = -1;
                continue;
            }
            if (c == '[' && pos + 1 < n && (re[pos + 1] == '.' || re[pos + 1] == '=')) {
                fail("POSIX collating elements are not supported.");
            }
            if (c == '-' && prev >= 0 && pos + 1 < n && re[pos + 1] != ']') {
                pos++;
                int hi;
                if (re[pos] == '[' && pos + 1 < n && strchr(":.=", re[pos + 1])) {
                    fail("Invalid range in character class.");
                }
                if (re[pos] == '\\') {
                    if (pos + 1 < n && (re[pos + 1] == 'Q' || re[pos + 1] == 'E')) {
                        fail("\\Q / \\E as the end of a range is not supported.");
                    }
                    escape(true, &hi);
                    if (hi < 0) {
                        fail("Invalid range in character class.");
                    }
                } else {
                    hi = (unsigned char)re[pos++];
                }
                if (hi < prev) {
                    fail("Invalid range in character class.");
                }
                for (int v = prev; v <= hi; v++) {
                    set[(size_t)v] = true;
                }
                prev = -1;
                continue;
            }
            if (c == '\\') {
                int single;
                const CharSet e = escape(true, &single);
                set |= e;
                prev = single;
            } else {
                set[c] = true;
                prev = c;
                pos++;
            }
        }
        set = fold(set);
        return negate ? ~set : set;
    }

    NodeP leaf(const CharSet &s) {
        if (s.none()) {
            fail("Empty character class.");
        }
        NodeP l = mk(Node::CLASS);
        l->cls = s;
        return l;
    }

    NodeP atom() {
        /* \\Q ... \\E: literal bytes (an \\E without \\Q is ignored) */
        while (pos + 1 < n && re[pos] == '\\' && (re[pos + 1] == 'E' || (re[pos + 1] == 'Q' && !quoting))) {
            quoting = re[pos + 1] == 'Q';
            pos += 2;
        }
        if (pos >= n || (!quoting && (re[pos] == '|' || re[pos] == ')'))) {
            return mk(Node::EMPTY);
        }
        const unsigned char c = (unsigned char)re[pos];
        if (quoting && utf8) {
            return atomU();
        }
        if (quoting) {
            pos++;
            CharSet s;
            s[c] = true;
            return leaf(fold(s));
        }
        if (c == '(') {
            pos++;
            const unsigned saved = flags; /* an option change lasts to the end of the group it is in */
            unsigned capture = 0;         /* the group's number; 0: not a capturing group */
            bool lookAround = false;
            std::string name;
            const char q1 = pos + 1 < n ? re[pos + 1] : 0, q2 = pos + 2 < n ? re[pos + 2] : 0;
            if (at('?') && (q1 == '\'' || (q1 == '<' && q2 != '=' && q2 != '!') || (q1 == 'P' && q2 == '<'))) {
                /* a named group, (?<name>...), (?'name'...), (?P<name>...): a capturing group in every mode */
                const size_t start = pos - 1;
                pos += q1 == 'P' ? 3 : 2;
                if (!readName(q1 == '\'' ? '\'' : '>', &name)) {
                    fail("Look-around, named groups, comments and the other (?...) groups are not supported.");
                }
                if (isdigit((unsigned char)name[0])) {
                    pos = start;
                    fail("Group name cannot begin with a digit.");
                }
                if (!names.emplace(name, groups).second) {
                    fail("Two named subpatterns use the name '" + name + "'.");
                }
                capture = groups++;
            } else if (prefilter && at('?') && (q1 == '=' || q1 == '!' || (q1 == '<' && (q2 == '=' || q2 == '!')))) {
                pos += q1 == '<' ? 3 : 2; /* look-around: an empty sequence */
                lookAround = true;
            } else if (prefilter && at('?') && q1 == '>') {
                pos += 2; /* an atomic group: a plain group */
            } else if (prefilter && at('?') && q1 == '(') {
                return conditional(saved);
            } else if (prefilter && at('?') && q1 == 'P' && q2 == '=') {
                pos += 3;
                if (!readName(')', &name)) {
                    fail("Look-around, named groups, comments and the other (?...) groups are not supported.");
                }
                return backRef(0, name);
            } else if (!at('?')) {
                capture = groups++;
            } else {
                /* (?ims-ims) and (?ims-ims: ... ) */
                size_t q = pos + 1;
                unsigned on = 0, off = 0;
                bool neg = false, any = false;
                for (; q < n && strchr("ims-", re[q]); q++) {
                    if (re[q] == '-') {
                        neg = true;
                        continue;
                    }
                    const unsigned f = re[q] == 'i' ? HS_FLAG_CASELESS : re[q] == 's' ? HS_FLAG_DOTALL : HS_FLAG_MULTILINE;
                    (neg ? off : on) |= f;
                    any = true;
                }
                if (q < n && re[q] == ')' && any) {
                    flags = (flags | on) & ~off;
                    pos = q + 1;
                    if (pos < n && (strchr("*+?", re[pos]) || startsRepeat(pos))) {
                        fail("Invalid repeat.");
                    }
                    return mk(Node::EMPTY);
                }
                if (q < n && re[q] == ':') {
                    flags = (flags | on) & ~off;
                    pos = q + 1;
                } else {
                    fail("Look-around, named groups, comments and the other (?...) groups are not supported.");
                }
            }
            if (capture) {
                referent.push_back(nullptr);
            }
            const size_t refsBefore = refsSeen;
            NodeP r = alt();
            if (!at(')')) {
                fail("Missing close parenthesis.");
            }
            pos++;
            flags = saved;
            if (capture && refsSeen == refsBefore && leaves(r) <= 1 && !hasAssert(r)) {
                referent[capture] = clone(r);
            }
            return lookAround ? mk(Node::EMPTY) : r;
        }
        if (c == '[') {
            /* "[:name:]", "[.x.]", "[=x=]" where a class should start: PCRE's check_posix_syntax */
            if (pos + 1 < n && strchr(":.=", re[pos + 1])) {
                const char term = re[pos + 1];
                for (size_t q = pos + 2; q < n; q++) {
                    if (re[q] == '\\' && q + 1 < n && (re[q + 1] == ']' || re[q + 1] == '\\')) {
                        q++;
                    } else if ((re[q] == '[' && q + 1 < n && re[q + 1] == term) || re[q] == ']') {
                        break;
                    } else if (re[q] == term && q + 1 < n && re[q + 1] == ']') {
                        fail(term == ':' ? "POSIX named classes are only supported inside a class."
                                         : "Unsupported POSIX collating element.");
                    }
                }
            }
            return utf8 ? unit(charClassU()) : leaf(charClass());
        }
        if (c == '\\' && pos + 1 < n && strchr("bBAzZ", re[pos + 1])) {
            NodeP a = mk(Node::ASSERT);
            const char e = re[pos + 1];
            a->assertKind = e == 'b' ? A_WORD_B : e == 'B' ? A_NOT_WORD_B : e == 'A' ? A_BEGIN : e == 'z' ? A_END : A_END_LF;
            pos += 2;
            return a;
        }
        if (c == '^' || c == '$') {
            NodeP a = mk(Node::ASSERT);
            const bool ml = flags & HS_FLAG_MULTILINE;
            a->assertKind = c == '^' ? (ml ? A_BEGIN_LINE : A_BEGIN) : (ml ? A_END_LINE : A_END_LF);
            pos++;
            return a;
        }
        if (prefilter && c == '\\' && pos + 1 < n) {
            if (NodeP b = prefilterEscape()) {
                return b;
            }
        }
        if (utf8) {
            return atomU();
        }
        if (c == '\\') {
            int single;
            CharSet s = escape(false, &single);
            return leaf(single >= 0 ? fold(s) : s);
        }
        if (c == '.') {
            pos++;
            CharSet s;
            s.set();
            if (!(flags & HS_FLAG_DOTALL)) {
                s['\n'] = false;
            }
            return leaf(s);
        }
        if (strchr("*+?", c) || (c == '{' && startsRepeat(pos))) {
            fail("Invalid repeat: nothing to repeat.");
        }
        pos++;
        CharSet s;
        s[c] = true;
        return leaf(fold(s));
    }
};

/* Glushkov: positions, nullable / first / last / follow */
struct Glushkov {
    std::vector<CharSet> cls;         /* per position */
    std::vector<StateSet> follow;     /* per position: set of positions */
    std::vector<int> assertion;       /* per position: 0 = a character position, else the A_* bit of a zero-width
                                       * pseudo-position (eliminated when the NFA is wired) */
    struct Sets {
        bool nullable;
        StateSet first, last;
    };
    static const u32 MAX_POSITIONS = MAX_NFA_STATES - 2; /* the two start states come first */

    Sets build(const NodeP &n) {
        switch (n->kind) {
        case Node::EMPTY:
            return {true, StateSet(), StateSet()};
        case Node::CLASS: {
            if (cls.size() >= MAX_POSITIONS) {
                throw RegexError{"Pattern is too large: more than 510 character positions."};
            }
            const u32 p = (u32)cls.size();
            cls.push_back(n->cls);
            follow.push_back(StateSet());
            assertion.push_back(0);
            return {false, stateBit(p), stateBit(p)};
        }
        case Node::ASSERT: {
            if (cls.size() >= MAX_POSITIONS) {
                throw RegexError{"Pattern is too large: more than 510 character positions."};
            }
            const u32 p = (u32)cls.size();
            cls.push_back(CharSet());
            follow.push_back(StateSet());
            assertion.push_back(n->assertKind);
            return {false, stateBit(p), stateBit(p)};
        }
        case Node::CAT: {
            Sets acc = {true, StateSet(), StateSet()};
            for (const NodeP &k : n->kids) {
                const Sets s = build(k);
                link(acc.last, s.first);
                const StateSet first = acc.nullable ? (acc.first | s.first) : acc.first;
                const StateSet last = s.nullable ? (acc.last | s.last) : s.last;
                acc = {acc.nullable && s.nullable, first, last};
            }
            return acc;
        }
        case Node::ALT: {
            Sets acc = {false, StateSet(), StateSet()};
            for (const NodeP &k : n->kids) {
                const Sets s = build(k);
                acc = {acc.nullable || s.nullable, acc.first | s.first, acc.last | s.last};
            }
            return acc;
        }
        case Node::STAR:
        case Node::PLUS: {
            const Sets s = build(n->kids[0]);
            link(s.last, s.first);
            return {n->kind == Node::STAR || s.nullable, s.first, s.last};
        }
        case Node::OPT: {
            const Sets s = build(n->kids[0]);
            return {true, s.first, s.last};
        }
        }
        return {true, StateSet(), StateSet()};
    }

    void link(const StateSet &from, const StateSet &to) {
        for (u32 p = 0; p < follow.size(); p++) {
            if (from.test(p)) {
                follow[p] |= to;
            }
        }
    }

    /* ---- zero-width assertions --------------------------------------------------------------
     * A path between two character positions p -> q may cross \b / \B pseudo-positions; what they
     * assert is about the two characters on either side: (p is a word character) != / == (q is).
     * need: bit 0 = some \b crossed, bit 1 = some \B crossed. */
    static bool holds(u32 need, bool leftWord, bool rightWord) {
        return !((need & 1) && leftWord == rightWord) && !((need & 2) && leftWord != rightWord);
    }
    bool isWord(u32 p) const { /* positions of an expression with assertions are split: all word or none */
        static const CharSet W = wordSet();
        return (cls[p] & W).any();
    }
    static CharSet wordSet() {
        CharSet w;
        for (int c = '0'; c <= '9'; c++) w[(size_t)c] = true;
        for (int c = 'a'; c <= 'z'; c++) w[(size_t)c] = w[(size_t)(c - 32)] = true;
        w['_'] = true;
        return w;
    }
    /* character positions reachable from the position set `from` through assertion pseudo-positions only,
     * each with the assertions crossed: out[(q, need)] */
    void reachThroughAssertions(const StateSet &from, u32 need, std::vector<std::pair<u32, u32>> *out,
                                std::vector<u8> *seen /* [position][need] */) const {
        for (u32 x = 0; x < cls.size(); x++) {
            if (!from.test(x)) {
                continue;
            }
            if (!assertion[x]) {
                out->push_back({x, need});
                continue;
            }
            const u32 n2 = need | (u32)assertion[x];
            u8 &mark = (*seen)[x * (A_ALL + 1) + n2];
            if (mark) {
                continue;
            }
            mark = 1;
            reachThroughAssertions(follow[x], n2, out, seen);
        }
    }
    /* the assertion sets under which a path from p (exclusive) through assertions only ends in `last` */
    void exitsThroughAssertions(const StateSet &from, u32 need, const StateSet &last, std::vector<u32> *needs, std::vector<u8> *seen) const {
        for (u32 x = 0; x < cls.size(); x++) {
            if (!from.test(x) || !assertion[x]) {
                continue;
            }
            const u32 n2 = need | (u32)assertion[x];
            u8 &mark = (*seen)[x * (A_ALL + 1) + n2];
            if (mark) {
                continue;
            }
            mark = 1;
            if (last.test(x)) {
                needs->push_back(n2);
            }
            exitsThroughAssertions(follow[x], n2, last, needs, seen);
        }
    }
    /* the assertion sets of the ways from `first` to `last` that cross assertions only (no character) */
    void emptyPaths(const StateSet &from, u32 need, const StateSet &last, std::vector<u32> *needs, std::vector<u8> *seen) const {
        for (u32 x = 0; x < cls.size(); x++) {
            if (!from.test(x) || !assertion[x]) {
                continue;
            }
            const u32 n2 = need | (u32)assertion[x];
            u8 &mark = (*seen)[x * (A_ALL + 1) + n2];
            if (mark) {
                continue;
            }
            mark = 1;
            if (last.test(x)) {
                needs->push_back(n2);
            }
            emptyPaths(follow[x], n2, last, needs, seen);
        }
    }
    bool anyAssertion() const {
        for (int a : assertion) {
            if (a) return true;
        }
        return false;
    }
};

bool hasAssertion(const NodeP &n, int kinds) {
    if (n->kind == Node::ASSERT && (n->assertKind & kinds)) {
        return true;
    }
    for (const NodeP &k : n->kids) {
        if (hasAssertion(k, kinds)) return true;
    }
    return false;
}

/* an expression with \b / \B: every class that mixes word and non-word characters becomes an
 * alternation of its two halves, so that each character position is one or the other */
void splitByWordness(NodeP &n) {
    if (n->kind == Node::CLASS) {
        const CharSet W = Glushkov::wordSet();
        const CharSet w = n->cls & W, o = n->cls & ~W;
        if (w.any() && o.any()) {
            NodeP a = mk(Node::ALT);
            NodeP l = mk(Node::CLASS), r = mk(Node::CLASS);
            l->cls = w;
            r->cls = o;
            a->kids = {l, r};
            n = a;
        }
        return;
    }
    for (NodeP &k : n->kids) {
        splitByWordness(k);
    }
}

u32 minLenOf(const NodeP &n) {
    switch (n->kind) {
    case Node::EMPTY: return 0;
    case Node::CLASS: return 1;
    case Node::CAT: {
        u32 s = 0;
        for (const NodeP &k : n->kids) s += minLenOf(k);
        return s;
    }
    case Node::ALT: {
        u32 m = ~0u;
        for (const NodeP &k : n->kids) m = std::min(m, minLenOf(k));
        return m;
    }
    case Node::PLUS: return minLenOf(n->kids[0]);
    case Node::STAR:
    case Node::OPT: return 0;
    }
    return 0;
}

u64 maxLenOf(const NodeP &n) { /* > 0xfffffffe = unbounded */
    const u64 INF = 1ull << 40;
    switch (n->kind) {
    case Node::EMPTY: return 0;
    case Node::CLASS: return 1;
    case Node::CAT: {
        u64 s = 0;
        for (const NodeP &k : n->kids) s = std::min(INF, s + maxLenOf(k));
        return s;
    }
    case Node::ALT: {
        u64 m = 0;
        for (const NodeP &k : n->kids) m = std::max(m, maxLenOf(k));
        return m;
    }
    case Node::PLUS:
    case Node::STAR: return maxLenOf(n->kids[0]) ? INF : 0;
    case Node::OPT: return maxLenOf(n->kids[0]);
    }
    return 0;
}

/* top-level alternatives of the expression, each with its anchored flag */
std::vector<NodeP> topArms(const NodeP &root) {
    NodeP r = root; /* "(a|b)" as a whole expression is the alternation a|b */
    while (r->kind == Node::CAT && r->kids.size() == 1) {
        r = r->kids[0];
    }
    if (r->kind == Node::ALT && !r->unit) {
        return r->kids;
    }
    return {root};
}

void addTree(RawNfa *nfa, const NodeP &root, u32 report, u32 reportBeforeNewline, u64 minLength);

/* The expression's tree, and the min_length its automaton keeps.  Under HS_FLAG_PREFILTER an expression whose own
 * automaton would be too large is reduced to a superset that fits (the role of src/nfagraph/ng_prefilter.cpp):
 * bounded repeats x{m,n} become x{m',}, the largest contribution first, each with the largest m' <= m that fits;
 * if that is not enough, min_length goes and the repeats are reduced again.  An expression that fits without a
 * reduction keeps its tree, so its database is the one it has without the flag. */
struct Parsed {
    NodeP root;
    u64 minLength;
};

/* what the reduction chose for one expression: the widened repeats and the min_length kept, or its error */
struct Reduction {
    std::vector<long> widen;
    u64 minLength;
    std::string error;
};

Reduction reduce(const char *re, unsigned flags, u64 minLength) {
    std::vector<long> widen;
    std::vector<Repeat> repeats;
    std::string tooLarge;
    /* does its own automaton fit?  Syntax and other errors are thrown as they are */
    auto fits = [&](u64 ml) -> bool {
        Parser p(re, flags, &widen);
        NodeP r = p.parse();
        repeats = p.repeats;
        if (p.overflow) {
            tooLarge = tooLarge.empty() ? "Pattern is too large." : tooLarge;
            return false;
        }
        try {
            RawNfa own;
            regexNfaInit(&own);
            addTree(&own, r, 1, 2, ml);
        } catch (const RegexError &e) {
            if (e.msg.find("too large") == std::string::npos) {
                return true; /* (not a size error: the real build reports it) */
            }
            tooLarge = tooLarge.empty() ? e.msg : tooLarge;
            return false;
        }
        return true;
    };
    for (const u64 ml : {minLength, (u64)0}) {
        widen.clear();
        if (fits(ml)) {
            return {widen, ml, ""};
        }
        const std::vector<Repeat> all = repeats;
        std::vector<size_t> order(all.size());
        for (size_t i = 0; i < order.size(); i++) order[i] = i;
        std::stable_sort(order.begin(), order.end(),
                         [&](size_t a, size_t b) { return all[a].positions > all[b].positions; });
        widen.assign(all.size(), -1);
        for (const size_t i : order) {
            const long least = std::min<long>(all[i].lo, 1); /* x{1,} is x+, as small as x* and not nullable */
            widen[i] = least;
            if (!fits(ml)) {
                continue; /* too large even so: this one stays at its least, and the next one widens too */
            }
            long good = least, tooBig = (long)all[i].lo + 1;
            while (tooBig - good > 1) {
                const long mid = (good + tooBig) / 2;
                widen[i] = mid;
                (fits(ml) ? good : tooBig) = mid;
            }
            widen[i] = good;
            return {widen, ml, ""};
        }
        if (!minLength) {
            break;
        }
    }
    return {{}, 0, tooLarge};
}

Parsed parseExpr(const char *re, unsigned flags, u64 minLength) {
    if (!(flags & HS_FLAG_PREFILTER)) {
        return {Parser(re, flags).parse(), minLength};
    }
    /* one compile asks for the same expression several times (widths, the "can never match" check, the build):
     * the reduction's search runs once per expression and thread */
    thread_local std::map<std::tuple<std::string, unsigned, u64>, Reduction> cache;
    const auto key = std::make_tuple(std::string(re), flags, minLength);
    auto it = cache.find(key);
    if (it == cache.end()) {
        if (cache.size() >= 4096) {
            cache.clear();
        }
        it = cache.emplace(key, reduce(re, flags, minLength)).first;
    }
    const Reduction &red = it->second;
    if (!red.error.empty()) {
        throw RegexError{red.error};
    }
    return {Parser(re, flags, &red.widen).parse(), red.minLength};
}

} // namespace

RegexInfo regexInfo(const char *re, unsigned flags, bool forInfo, u64 minLength) {
    const Parsed parsed = parseExpr(re, flags, minLength);
    const NodeP &root = parsed.root;
    RegexInfo info;
    info.minLengthDropped = parsed.minLength != minLength;
    info.minLen = ~0u;
    bool someOtherExit = false, someFloatingEntry = false;
    /* one way out of the expression: the assertions crossed after the last character, and whether that character
     * is a word character (-1: there is none, the byte before the match is whatever it is) */
    auto exitVia = [&](u32 need, int leftWord) {
        info.unordered |= (need & (A_BOUNDARY | A_END_LF | A_END_LINE)) != 0;
        bool canEod = false;
        if (need & (A_ENDS | A_BOUNDARY)) {
            for (int lw = 0; lw < 2; lw++) {
                if (leftWord >= 0 && lw != leftWord) {
                    continue;
                }
                if ((need & A_STARTS) && lw) {
                    continue; /* the start of the data / a newline before: not a word character */
                }
                canEod |= Glushkov::holds(need, lw != 0, false);
            }
        }
        info.atEod |= canEod;
        if (!(need & (A_END | A_END_LF))) {
            someOtherExit = true;
        }
    };
    for (NodeP arm : topArms(root)) {
        const bool asserts = hasAssertion(arm, A_BOUNDARY);
        if (asserts) {
            splitByWordness(arm);
        }
        /* an assertion at the end may look one byte ahead */
        info.needsAdjust |= hasAssertion(arm, A_BOUNDARY | A_END_LF | A_END_LINE);
        Glushkov g;
        const Glushkov::Sets s = g.build(arm);
        if (!forInfo && (s.nullable || minLenOf(arm) == 0)) {
            throw RegexError{"Pattern matches empty buffer; use HS_FLAG_ALLOWEMPTY to enable support."};
        }
        info.minLen = std::min(info.minLen, minLenOf(arm));
        const u64 mx = maxLenOf(arm);
        info.maxLen = std::max<u32>(info.maxLen, mx > 0xfffffffeull ? 0xffffffffu : (u32)mx);
        info.armWidths.push_back({minLenOf(arm), mx > 0xfffffffeull ? 0xffffffffu : (u32)mx});
        info.positions += (u32)g.cls.size();
        const u32 np = (u32)g.cls.size();
        for (u32 p = 0; p < np; p++) {
            if (g.assertion[p]) {
                continue;
            }
            const int lw = asserts ? (int)g.isWord(p) : -1;
            if (s.last.test(p)) {
                exitVia(0, lw);
            }
            std::vector<u32> needs;
            std::vector<u8> seen(np * (A_ALL + 1), 0);
            g.exitsThroughAssertions(g.follow[p], 0, s.last, &needs, &seen);
            for (u32 need : needs) {
                exitVia(need, lw);
            }
        }
        {
            std::vector<std::pair<u32, u32>> entries;
            std::vector<u8> seenE(np * (A_ALL + 1), 0);
            g.reachThroughAssertions(s.first, 0, &entries, &seenE);
            for (const auto &e : entries) {
                someFloatingEntry |= !(e.second & A_BEGIN);
            }
        }
        if (s.nullable) {
            exitVia(0, -1);
            someFloatingEntry = true;
        }
        std::vector<u32> needs;
        std::vector<u8> seen(np * (A_ALL + 1), 0);
        g.emptyPaths(s.first, 0, s.last, &needs, &seen);
        for (u32 need : needs) {
            exitVia(need, -1);
        }
    }
    info.onlyAtEod = info.atEod && !someOtherExit;
    info.anchored = !someFloatingEntry;
    return info;
}

void regexNfaInit(RawNfa *nfa) {
    *nfa = RawNfa();
    nfa->nstates = 2; /* 0 = floating start (.* loop), 1 = anchored start (offset 0 only) */
    nfa->succ.assign(2, StateSet());
    nfa->succ[0] = stateBit(0);
    nfa->squashMask.assign(2, allStates());
    nfa->squashKind.assign(2, LIMEX_SQUASH_NONE);
    nfa->reports.resize(2);
    nfa->reportsEod.resize(2);
    for (u32 b = 0; b < 256; b++) {
        nfa->reach[b] = stateBit(0); /* the floating start survives every byte; nothing re-enters state 1 */
    }
    nfa->init = nfa->initDS = stateSetOf(3);
}

void regexNfaAdd(RawNfa *nfa, const char *re, unsigned flags, u32 report, u32 reportBeforeNewline, u64 minLength) {
    const Parsed p = parseExpr(re, flags, minLength);
    addTree(nfa, p.root, report, reportBeforeNewline, p.minLength);
}

namespace {

void addTree(RawNfa *nfa, const NodeP &root, u32 report, u32 reportBeforeNewline, u64 minLength) {
    const CharSet W = Glushkov::wordSet();
    auto newState = [&]() -> u32 {
        if (nfa->nstates >= MAX_NFA_STATES) {
            throw RegexError{"Pattern set is too large: its character positions exceed the 512-state NFA model."};
        }
        nfa->nstates++;
        nfa->succ.push_back(StateSet());
        nfa->squashMask.push_back(allStates());
        nfa->squashKind.push_back(LIMEX_SQUASH_NONE);
        nfa->reports.emplace_back();
        nfa->reportsEod.emplace_back();
        return nfa->nstates - 1;
    };
    auto reachClass = [&](u32 st, const CharSet &c) {
        for (u32 b = 0; b < 256; b++) {
            if (c[b]) {
                nfa->reach[b].set(st);
            }
        }
    };
    for (NodeP arm : topArms(root)) {
        const bool asserts = hasAssertion(arm, A_BOUNDARY);
        if (asserts) {
            splitByWordness(arm);
        }
        Glushkov g;
        const Glushkov::Sets s = g.build(arm);
        if (s.nullable || minLenOf(arm) == 0) {
            throw RegexError{"Pattern matches empty buffer; use HS_FLAG_ALLOWEMPTY to enable support."};
        }
        const u32 np = (u32)g.cls.size();
        /* hs_expr_ext.min_length: only matches of at least that many bytes count.  The automaton then carries the
         * number of bytes consumed since the match began, saturating at the minimum: K copies ("levels") of every
         * position, a transition goes one level up, and only the top level accepts.  (No minimum, or every match
         * is long enough anyway: one level.) */
        if (minLength > MAX_NFA_STATES) {
            throw RegexError{"Pattern is too large: min_length beyond the 512-state NFA model."};
        }
        const u32 K = minLength > minLenOf(arm) ? (u32)minLength : 1;
        /* NFA states of every character position, one per level (assertion pseudo-positions get none) */
        std::vector<std::vector<u32>> lv(np, std::vector<u32>(K, 0));
        for (u32 p = 0; p < np; p++) {
            if (!g.assertion[p]) {
                for (u32 c = 0; c < K; c++) {
                    lv[p][c] = newState();
                    reachClass(lv[p][c], g.cls[p]);
                }
            }
        }
        /* the accepting copy of a position */
        std::vector<u32> st(np, 0);
        for (u32 p = 0; p < np; p++) {
            st[p] = lv[p][K - 1];
        }

        /* --- transitions between character positions --- */
        for (u32 p = 0; p < np; p++) {
            if (g.assertion[p]) {
                continue;
            }
            std::vector<std::pair<u32, u32>> to;
            std::vector<u8> seen(np * (A_ALL + 1), 0);
            g.reachThroughAssertions(g.follow[p], 0, &to, &seen);
            for (const auto &e : to) {
                if (e.second & (A_STARTS | A_ENDS)) {
                    continue; /* an anchor between two characters (the parser lets none through) */
                }
                if (Glushkov::holds(e.second, g.isWord(p), g.isWord(e.first))) {
                    for (u32 c = 0; c < K; c++) {
                        nfa->succ[lv[p][c]].set(lv[e.first][std::min(c + 1, K - 1)]);
                    }
                }
            }
        }

        /* --- entries --- */
        std::vector<std::pair<u32, u32>> entries;
        {
            std::vector<u8> seen(np * (A_ALL + 1), 0);
            g.reachThroughAssertions(s.first, 0, &entries, &seen);
        }
        for (const auto &e : entries) {
            const u32 entry = lv[e.first][0]; /* one byte consumed */
            const bool qw = asserts && g.isWord(e.first);
            if (e.second & A_ENDS) {
                continue; /* a character after the end of the data */
            }
            if (e.second & A_STARTS) {
                /* what precedes is the start of the data or a newline: not a word character */
                if (!Glushkov::holds(e.second, false, qw)) {
                    continue;
                }
                nfa->succ[1].set(entry);
                if (!(e.second & A_BEGIN)) {
                    /* "^" under (?m): entered at offset 0 (anchored start) or right after any newline --
                     * one state shared by all such entries, on after every '\n' */
                    if (!nfa->mlStartState) {
                        nfa->mlStartState = newState();
                        nfa->reach[(u8)'\n'].set(nfa->mlStartState);
                        nfa->succ[0].set(nfa->mlStartState);
                    }
                    nfa->succ[nfa->mlStartState].set(entry);
                }
            } else if (e.second == 0) {
                nfa->succ[0].set(entry);
            } else {
                /* a leading \b / \B of a floating entry: the byte before the match decides.  Two
                 * shared context states hang off the floating start: "previous byte is a word character"
                 * and "previous byte is none, or not a word character" (the latter also on at offset 0) */
                if (!nfa->ctxWord) {
                    nfa->ctxWord = newState();
                    nfa->ctxNonWord = newState();
                    reachClass(nfa->ctxWord, W);
                    reachClass(nfa->ctxNonWord, ~W);
                    nfa->succ[0].set(nfa->ctxWord).set(nfa->ctxNonWord);
                    nfa->init.set(nfa->ctxNonWord);
                    nfa->initDS.set(nfa->ctxNonWord);
                }
                if (Glushkov::holds(e.second, true, qw)) {
                    nfa->succ[nfa->ctxWord].set(entry);
                }
                if (Glushkov::holds(e.second, false, qw)) {
                    nfa->succ[nfa->ctxNonWord].set(entry);
                }
            }
        }

        /* --- accepts --- */
        auto adjusted = [&]() -> u32 {
            if (!reportBeforeNewline) {
                throw RegexError{"internal: no adjusted report program"};
            }
            return reportBeforeNewline;
        };
        auto addOnce = [](std::vector<u32> &v, u32 r) {
            if (std::find(v.begin(), v.end(), r) == v.end()) {
                v.push_back(r);
            }
        };
        /* one byte of look-ahead, reported one byte back (offset_adjust -1, as the reference compiles "$"):
         * a word character, a non-word character (trailing \b / \B), any newline ("$" under (?m)), a newline
         * that ends the data ("$", \Z) */
        u32 aheadWord = 0, aheadNonWord = 0, aheadNewline = 0, aheadLastNewline = 0;
        for (u32 p = 0; p < np; p++) {
            if (g.assertion[p]) {
                continue;
            }
            if (s.last.test(p)) {
                addOnce(nfa->reports[st[p]], report);
            }
            std::vector<u32> needs;
            std::vector<u8> seen(np * (A_ALL + 1), 0);
            g.exitsThroughAssertions(g.follow[p], 0, s.last, &needs, &seen);
            const bool pw = asserts && g.isWord(p);
            for (u32 need : needs) {
                if (need & A_STARTS) {
                    continue; /* a start anchor after a character (the parser lets none through) */
                }
                if (Glushkov::holds(need, pw, false)) { /* the end of the data counts as a non-word character */
                    addOnce(nfa->reportsEod[st[p]], report);
                }
                if (need & A_ENDS) {
                    if ((need & A_END) || !Glushkov::holds(need, pw, false)) {
                        continue; /* \z: nothing but the end of the data will do; a newline is not a word character */
                    }
                    if (need & A_END_LF) {
                        if (!aheadLastNewline) {
                            aheadLastNewline = newState();
                            nfa->reach[(u8)'\n'].set(aheadLastNewline);
                            nfa->reportsEod[aheadLastNewline].push_back(adjusted());
                        }
                        nfa->succ[st[p]].set(aheadLastNewline);
                    } else {
                        if (!aheadNewline) {
                            aheadNewline = newState();
                            nfa->reach[(u8)'\n'].set(aheadNewline);
                            nfa->reports[aheadNewline].push_back(adjusted());
                        }
                        nfa->succ[st[p]].set(aheadNewline);
                    }
                    continue;
                }
                if (Glushkov::holds(need, pw, true)) {
                    if (!aheadWord) {
                        aheadWord = newState();
                        reachClass(aheadWord, W);
                        nfa->reports[aheadWord].push_back(adjusted());
                    }
                    nfa->succ[st[p]].set(aheadWord);
                }
                if (Glushkov::holds(need, pw, false)) {
                    if (!aheadNonWord) {
                        aheadNonWord = newState();
                        reachClass(aheadNonWord, ~W);
                        nfa->reports[aheadNonWord].push_back(adjusted());
                    }
                    nfa->succ[st[p]].set(aheadNonWord);
                }
            }
        }
    }
}

} // namespace

} // namespace hsb
