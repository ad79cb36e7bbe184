/*
 * regex_nfa.h -- regular expressions to a LimEx NFA (32- to 512-state model): the position (Glushkov)
 * automaton the reference builds for its NFA engines (src/nfagraph/ng_builder.cpp,
 * src/parser/buildstate.cpp: one state per character position, epsilon free), for
 * expression sets whose positions fit the 512-state model together with the start states.
 *
 * Syntax (PCRE as the reference's parser accepts it, src/parser/Parser.rl): literal
 * characters and escapes (\n \t \r \f \a \e \xHH \x{hh} \0oo \cX, escaped punctuation, \Q...\E),
 * the class escapes \d \D \w \W \s \S \h \H \v \V \N, "." (any byte but \n; any byte under
 * HS_FLAG_DOTALL), character classes with ranges, negation, class escapes and POSIX classes,
 * groups "(...)" / "(?:...)" (Hyperscan does not capture), option groups "(?ims-ims)" and
 * "(?ims-ims:...)" scoped to the enclosing group, alternation, the quantifiers ? * + {n} {n,}
 * {n,m} (a lazy "?" suffix changes nothing when every match end is reported), \b and \B, and the
 * anchors "^" \A (offset 0; "^" under HS_FLAG_MULTILINE also after any newline), "$" \Z (end of
 * data or before a final newline; "$" under HS_FLAG_MULTILINE before any newline or at the end),
 * \z (end of data) -- anywhere the reference takes them: where nothing can have been consumed
 * before a start anchor / can be consumed after an end anchor (ComponentBoundary.cpp:162-185),
 * groups and alternations included.  HS_FLAG_CASELESS folds letters.
 *
 * HS_FLAG_UTF8 (src/parser/Utf8ComponentClass.cpp): the expression must be valid UTF-8; a character
 * is a code point (literal, \x{h..h}, \o{o..o} up to 0x10FFFF) and matches its encoding; ".",
 * negated classes, classes with non-ASCII members and \W \D \S \H \V \N match whole encoded
 * characters -- each is a small byte automaton (the encodings of its code-point set as a tree of
 * byte ranges) whose positions join the Glushkov construction.  \w \d \s, POSIX classes and
 * \b \B keep their ASCII meaning; \C is one byte.  Case folding is ASCII only (plus KELVIN SIGN
 * and LONG S, which fold to "k" and "s"); a caseless non-ASCII character, \p \P \X and
 * HS_FLAG_UCP are refused.
 *
 * Named groups (?<n>...) (?'n'...) (?P<n>...) are capturing groups in every mode.
 *
 * HS_FLAG_PREFILTER (src/parser/prefilter.cpp): the expression is rewritten into one whose matches are
 * a superset of its own -- a back-reference (\1..\99, \g, \k, (?P=n)) becomes a copy of its group when
 * that group is one character position (folded where the reference is caseless), else any byte
 * sequence; look-around becomes nothing, an atomic group a plain group, a possessive quantifier the
 * greedy one, a conditional group the alternation of its branches, \X ".+" -- and an expression whose automaton would be too large is widened until it fits
 * (bounded repeats x{m,n} become x{m',}; then min_length goes).
 *
 * Everything else -- look-around and the rest without HS_FLAG_PREFILTER, UCP, SOM, expressions
 * that match the empty string -- is refused with a compile error: those need parts of the
 * reference's compiler and runtime this build does not have.
 */
#ifndef HSB200_REGEX_NFA_H
#define HSB200_REGEX_NFA_H

#include <string>
#include <vector>

#include "limex_build.h"

namespace hsb {

struct RegexError {
    std::string msg;
};

struct RegexInfo {
    u32 minLen = 0;      /* length of the shortest match */
    u32 maxLen = 0;      /* of the longest; 0xffffffff = unbounded (hs_expr_info_t.max_width convention) */
    u32 positions = 0;   /* character positions of the expression */
    bool needsAdjust = false; /* an alternative ends in "$" / \Z: see regexNfaAdd */
    /* hs_expr_info_t (src/hs_compile.h:169-216): some match is raised one byte late and delivered back in time
     * (a trailing "$" / \Z / \b); some match can be raised at the end of the data only because it is the end
     * ("$" \z \Z, a trailing \b); every match is of that kind */
    bool unordered = false, atEod = false, onlyAtEod = false;
    std::vector<std::pair<u32, u32>> armWidths; /* (shortest, longest) match of every top-level alternative */
    bool anchored = false; /* every way into the expression crosses \A / a non-multiline "^" */
    bool minLengthDropped = false; /* HS_FLAG_PREFILTER: the automaton fits only without the min_length */
};

/* Valid UTF-8 (src/parser/utf8_validate.cpp): no overlong form, surrogate, code point above 0x10FFFF or
 * truncated character. */
bool validUtf8(const char *s, size_t len);

/* Number of positions / shortest match of one expression (throws RegexError).  forInfo: hs_expression_info also
 * describes expressions that match the empty buffer (hs_compile refuses those without HS_FLAG_ALLOWEMPTY).
 * minLength: as for regexNfaAdd, so that a prefiltered expression is described as the same reduction. */
RegexInfo regexInfo(const char *re, unsigned flags, bool forInfo = false, u64 minLength = 0);

/* Add the expression's position automaton to `nfa`: its accepting positions raise `report`.
 * State 0 of `nfa` is the floating start (always on), state 1 the anchored start (on at
 * offset 0 only); call regexNfaInit first.  Throws RegexError, also when the 64 states
 * are exceeded. */
void regexNfaInit(RawNfa *nfa);
void regexNfaAdd(RawNfa *nfa, const char *re, unsigned flags, u32 report, u32 reportBeforeNewline = 0,
                 u64 minLength = 0); /* minLength: hs_expr_ext.min_length, 0 = none */
/* reportBeforeNewline: the same report delivered one byte back (a report program with offset_adjust -1) --
 * needed when RegexInfo.needsAdjust: "$" / \Z match before a final newline, "$" under (?m) before any */

} // namespace hsb
#endif
