/*
 * api_host.cpp -- host-only half of the C ABI: compile entry points, the
 * hs_database container (create / serialize / deserialize / info) and the
 * allocator hooks.  Names, argument checks and error codes follow the
 * reference so that its own API tests read the same here:
 *   compile   src/hs.cpp:168-330 (arg checks), src/compiler/compiler.cpp:391-440
 *   database  src/database.c:62-468, src/database.h:102-127
 *   alloc     src/alloc.c:38-135
 */
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <cctype>
#include <new>
#include <set>
#include <string>
#include <vector>

#include "../../../include/hs_b200.h"
#include "api_internal.h"
#include "rose_build.h"
#include "dfa_build.h"
#include "limex_build.h"
#include "regex_nfa.h"

using namespace hsb;

/* ------------------------------------------------------------ allocators */

namespace hsb {
hs_alloc_t g_db_alloc = malloc, g_misc_alloc = malloc, g_scratch_alloc = malloc,
           g_stream_alloc = malloc;
hs_free_t g_db_free = free, g_misc_free = free, g_scratch_free = free,
          g_stream_free = free;

hs_error_t checkAlloc(const void *p) { /* src/alloc.c:111-119 */
    if (!p) {
        return HS_NOMEM;
    }
    if ((uintptr_t)p % alignof(unsigned long long)) {
        return HS_BAD_ALLOC;
    }
    return HS_SUCCESS;
}
} // namespace hsb

extern "C" {

hs_error_t hs_set_database_allocator(hs_alloc_t a, hs_free_t f) {
    g_db_alloc = a ? a : malloc;
    g_db_free = f ? f : free;
    return HS_SUCCESS;
}
hs_error_t hs_set_misc_allocator(hs_alloc_t a, hs_free_t f) {
    g_misc_alloc = a ? a : malloc;
    g_misc_free = f ? f : free;
    return HS_SUCCESS;
}
hs_error_t hs_set_scratch_allocator(hs_alloc_t a, hs_free_t f) {
    g_scratch_alloc = a ? a : malloc;
    g_scratch_free = f ? f : free;
    return HS_SUCCESS;
}
hs_error_t hs_set_stream_allocator(hs_alloc_t a, hs_free_t f) {
    g_stream_alloc = a ? a : malloc;
    g_stream_free = f ? f : free;
    return HS_SUCCESS;
}
hs_error_t hs_set_allocator(hs_alloc_t a, hs_free_t f) {
    hs_set_database_allocator(a, f);
    hs_set_misc_allocator(a, f);
    hs_set_stream_allocator(a, f);
    hs_set_scratch_allocator(a, f);
    return HS_SUCCESS;
}

const char *hs_version(void) { return "5.4.2 b200"; }

/* ------------------------------------------------------ compile errors */

static hs_compile_error_t g_enomem = {(char *)"Unable to allocate memory.", -1};

static hs_compile_error_t *makeError(const std::string &msg, int idx) {
    hs_compile_error_t *e = (hs_compile_error_t *)g_misc_alloc(sizeof(*e));
    if (!e) {
        return &g_enomem;
    }
    e->message = (char *)g_misc_alloc(msg.size() + 1);
    if (!e->message) {
        g_misc_free(e);
        return &g_enomem;
    }
    memcpy(e->message, msg.c_str(), msg.size() + 1);
    e->expression = idx;
    return e;
}

hs_error_t hs_free_compile_error(hs_compile_error_t *error) {
    if (!error || error == &g_enomem) {
        return HS_SUCCESS;
    }
    g_misc_free(error->message);
    g_misc_free(error);
    return HS_SUCCESS;
}

hs_error_t hs_populate_platform(hs_platform_info_t *platform) {
    if (!platform) {
        return HS_INVALID;
    }
    /* The scan engines run on the GPU; the database we emit uses only the
     * baseline (non-AVX2) table variants, which every reference build also
     * accepts (src/database.c:115-124). */
    memset(platform, 0, sizeof(*platform));
    return HS_SUCCESS;
}

/* --------------------------------------------------------- db container */

static hs_database_t *dbCreate(const std::vector<u8> &bc, u64 platform,
                               hs_error_t *err) {
    const size_t len = sizeof(DbHeader) + bc.size();
    DbHeader *db = (DbHeader *)g_db_alloc(len);
    *err = checkAlloc(db);
    if (*err != HS_SUCCESS) {
        g_db_free(db);
        return nullptr;
    }
    memset(db, 0, len);
    const size_t shift = ((uintptr_t)db + sizeof(DbHeader)) & 0x3f;
    db->bytecode = (u32)(sizeof(DbHeader) - shift);
    db->magic = DB_MAGIC;
    db->version = DB_VERSION;
    db->length = (u32)bc.size();
    db->platform = platform;
    u8 *dst = (u8 *)db + db->bytecode;
    memcpy(dst, bc.data(), bc.size());
    db->crc32 = crc32c(0, dst, bc.size());
    return (hs_database_t *)db;
}

hs_error_t hs_free_database(hs_database_t *db) {
    if (db && ((DbHeader *)db)->magic != DB_MAGIC) {
        return HS_INVALID;
    }
    g_db_free(db);
    return HS_SUCCESS;
}

static bool dbAligned(const void *db) { return (uintptr_t)db % 8 == 0; }

static hs_error_t validDb(const hs_database_t *db) {
    const DbHeader *h = (const DbHeader *)db;
    if (!h || h->magic != DB_MAGIC) {
        return HS_INVALID;
    }
    if (h->version != DB_VERSION) {
        return HS_DB_VERSION_ERROR;
    }
    return HS_SUCCESS;
}

hs_error_t hs_serialize_database(const hs_database_t *db, char **bytes,
                                 size_t *length) {
    if (!db || !bytes || !length) {
        return HS_INVALID;
    }
    if (!dbAligned(db)) {
        return HS_BAD_ALIGN;
    }
    hs_error_t ret = validDb(db);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    const DbHeader *h = (const DbHeader *)db;
    const size_t len = sizeof(DbHeader) + h->length;
    char *out = (char *)g_misc_alloc(len);
    ret = checkAlloc(out);
    if (ret != HS_SUCCESS) {
        g_misc_free(out);
        return ret;
    }
    memset(out, 0, len);
    u32 *w = (u32 *)out;
    w[0] = h->magic;
    w[1] = h->version;
    w[2] = h->length;
    memcpy(w + 3, &h->platform, 8);
    w[5] = h->crc32;
    w[6] = h->reserved0;
    w[7] = h->reserved1;
    memcpy(w + 8, (const char *)h + h->bytecode, h->length);
    *bytes = out;
    *length = len;
    return HS_SUCCESS;
}

/* Any combination of the three NO* feature bits is a database some reference
 * build could have produced; the H100 engines consume every table variant, so
 * (unlike src/database.c:115-124) none of them is a platform mismatch. */
static hs_error_t checkPlatform(u64 p) {
    const u64 known = PLATFORM_NOAVX2 | PLATFORM_NOAVX512 | PLATFORM_NOAVX512VBMI;
    return (p & ~known) ? HS_DB_PLATFORM_ERROR : HS_SUCCESS;
}

static hs_error_t decodeHeader(const char **bytes, size_t length, DbHeader *h) {
    if (!*bytes) {
        return HS_INVALID;
    }
    if (length < sizeof(DbHeader)) {
        return HS_INVALID;
    }
    u32 w[8];
    memcpy(w, *bytes, sizeof(w));
    memset(h, 0, sizeof(*h));
    h->magic = w[0];
    if (h->magic != DB_MAGIC) {
        return HS_INVALID;
    }
    h->version = w[1];
    if (h->version != DB_VERSION) {
        return HS_DB_VERSION_ERROR;
    }
    h->length = w[2];
    if (length != sizeof(DbHeader) + h->length) {
        return HS_INVALID;
    }
    memcpy(&h->platform, &w[3], 8);
    h->crc32 = w[5];
    h->reserved0 = w[6];
    h->reserved1 = w[7];
    *bytes += 32;
    return HS_SUCCESS;
}

static void placeBytecode(const char *ser, DbHeader *db) {
    const size_t shift = ((uintptr_t)db + sizeof(DbHeader)) & 0x3f;
    db->bytecode = (u32)(sizeof(DbHeader) - shift);
    memcpy((char *)db + db->bytecode, ser, db->length);
}

static hs_error_t checkCrc(const DbHeader *db) {
    u32 c = crc32c(0, (const char *)db + db->bytecode, db->length);
    return c == db->crc32 ? HS_SUCCESS : HS_INVALID;
}

hs_error_t hs_deserialize_database_at(const char *bytes, const size_t length,
                                      hs_database_t *db) {
    if (!bytes || !db) {
        return HS_INVALID;
    }
    if (!dbAligned(db)) {
        return HS_BAD_ALIGN;
    }
    DbHeader h;
    hs_error_t ret = decodeHeader(&bytes, length, &h);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    ret = checkPlatform(h.platform);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    memset(db, 0, sizeof(DbHeader) + h.length);
    memcpy(db, &h, sizeof(h));
    placeBytecode(bytes, (DbHeader *)db);
    return checkCrc((DbHeader *)db);
}

hs_error_t hs_deserialize_database(const char *bytes, const size_t length,
                                   hs_database_t **db) {
    if (!bytes || !db) {
        return HS_INVALID;
    }
    *db = nullptr;
    DbHeader h;
    hs_error_t ret = decodeHeader(&bytes, length, &h);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    ret = checkPlatform(h.platform);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    const size_t len = sizeof(DbHeader) + h.length;
    DbHeader *out = (DbHeader *)g_db_alloc(len);
    ret = checkAlloc(out);
    if (ret != HS_SUCCESS) {
        g_db_free(out);
        return ret;
    }
    memset(out, 0, len);
    memcpy(out, &h, sizeof(h));
    placeBytecode(bytes, out);
    if (checkCrc(out) != HS_SUCCESS) {
        g_db_free(out);
        return HS_INVALID;
    }
    *db = (hs_database_t *)out;
    return HS_SUCCESS;
}

hs_error_t hs_database_size(const hs_database_t *db, size_t *size) {
    if (!size) {
        return HS_INVALID;
    }
    hs_error_t ret = validDb(db);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    *size = sizeof(DbHeader) + ((const DbHeader *)db)->length;
    return HS_SUCCESS;
}

hs_error_t hs_serialized_database_size(const char *bytes, const size_t length,
                                       size_t *size) {
    DbHeader h;
    hs_error_t ret = decodeHeader(&bytes, length, &h);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    if (!size) {
        return HS_INVALID;
    }
    *size = sizeof(DbHeader) + h.length;
    return HS_SUCCESS;
}

hs_error_t hs_stream_size(const hs_database_t *db, size_t *stream_size) {
    if (!stream_size) {
        return HS_INVALID;
    }
    hs_error_t ret = validDb(db);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    const RoseEngine *r = dbRose(db);
    if (r->mode != MODE_STREAM) { /* src/runtime.c:1058-1080 */
        return HS_DB_MODE_ERROR;
    }
    *stream_size = 16 + r->stateOffsets.end;
    return HS_SUCCESS;
}

static hs_error_t infoString(char **s, u32 version, u64 plat, u32 mode) {
    const char *features =
        (plat & PLATFORM_NOAVX512VBMI)
            ? (plat & PLATFORM_NOAVX512) ? (plat & PLATFORM_NOAVX2) ? "" : "AVX2"
                                         : "AVX512"
            : "AVX512VBMI";
    const char *m = mode == MODE_STREAM ? "STREAM"
                    : mode == MODE_VECTORED ? "VECTORED" : "BLOCK";
    char tmp[256];
    int n = snprintf(tmp, sizeof(tmp), "Version: %u.%u.%u Features: %s Mode: %s",
                     (version >> 24) & 0xff, (version >> 16) & 0xff,
                     (version >> 8) & 0xff, features, m);
    char *buf = (char *)g_misc_alloc((size_t)n + 1);
    hs_error_t ret = checkAlloc(buf);
    if (ret != HS_SUCCESS) {
        g_misc_free(buf);
        return ret;
    }
    memcpy(buf, tmp, (size_t)n + 1);
    *s = buf;
    return HS_SUCCESS;
}

hs_error_t hs_database_info(const hs_database_t *db, char **info) {
    if (!info) {
        return HS_INVALID;
    }
    *info = nullptr;
    const DbHeader *h = (const DbHeader *)db;
    if (!h || !dbAligned(h) || h->magic != DB_MAGIC) {
        return HS_INVALID;
    }
    return infoString(info, h->version, h->platform, dbRose(db)->mode);
}

hs_error_t hs_serialized_database_info(const char *bytes, size_t length,
                                       char **info) {
    if (!info) {
        return HS_INVALID;
    }
    *info = nullptr;
    DbHeader h;
    hs_error_t ret = decodeHeader(&bytes, length, &h);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    u32 mode;
    memcpy(&mode, bytes + offsetof(RoseEngine, mode), 4);
    return infoString(info, h.version, h.platform, mode);
}

hs_error_t hs_b200_db_info(const hs_database_t *db, hs_b200_db_info_t *out) {
    if (!out) {
        return HS_INVALID;
    }
    hs_error_t ret = validDb(db);
    if (ret != HS_SUCCESS) {
        return ret;
    }
    memset(out, 0, sizeof(*out));
    const RoseEngine *r = dbRose(db);
    out->runtime_impl = r->runtimeImpl;
    out->bytecode_len = ((const DbHeader *)db)->length;
    out->min_width = r->minWidth;
    out->num_literals = r->totalNumLiterals;
    if (r->fmatcherOffset) {
        const HWLM *h = (const HWLM *)((const u8 *)r + r->fmatcherOffset);
        out->hwlm_type = h->type;
        if (h->type == HWLM_ENGINE_FDR) {
            const FDR *f = (const FDR *)((const u8 *)h + HWLM_ENGINE_OFFSET);
            out->engine_id = f->engineID;
            out->num_literals = f->numStrings;
            if (f->engineID == 0) {
                out->fdr_domain = f->domain;
                out->fdr_stride = f->stride;
            }
        }
    } else if (r->runtimeImpl == RUNTIME_SINGLE_OUTFIX && r->nfaInfoOffset) {
        const NfaInfo *ni = (const NfaInfo *)((const u8 *)r + r->nfaInfoOffset);
        const NFA *n = (const NFA *)((const u8 *)r + ni->nfaOffset);
        out->engine_id = n->type;        /* enum NFAEngineType: LimEx 0..5, McClellan 6 / 7, Sheng 17 */
        out->num_literals = n->nPositions; /* states of the engine */
    }
    return HS_SUCCESS;
}

/* -------------------------------------------------------------- compile */

static bool checkMode(unsigned mode, std::string *why) {
    const unsigned known = HS_MODE_BLOCK | HS_MODE_STREAM | HS_MODE_VECTORED |
                           HS_MODE_SOM_HORIZON_LARGE | HS_MODE_SOM_HORIZON_MEDIUM |
                           HS_MODE_SOM_HORIZON_SMALL;
    if (mode & ~known) {
        *why = "Invalid parameter: unrecognised mode flags.";
        return false;
    }
    unsigned m = mode & (HS_MODE_STREAM | HS_MODE_BLOCK | HS_MODE_VECTORED);
    if (__builtin_popcount(m) != 1) {
        *why = "Invalid parameter: mode must have one (and only one) of "
               "HS_MODE_BLOCK, HS_MODE_STREAM or HS_MODE_VECTORED set.";
        return false;
    }
    unsigned som = mode & (HS_MODE_SOM_HORIZON_LARGE | HS_MODE_SOM_HORIZON_MEDIUM |
                           HS_MODE_SOM_HORIZON_SMALL);
    if (som) {
        if (!(mode & HS_MODE_STREAM)) {
            *why = "Invalid parameter: the HS_MODE_SOM_HORIZON_ mode flags may "
                   "only be set in streaming mode.";
            return false;
        }
        if (som & (som - 1)) {
            *why = "Invalid parameter: only one HS_MODE_SOM_HORIZON_ mode flag "
                   "can be set.";
            return false;
        }
    }
    return true;
}

static bool checkPlatformInfo(const hs_platform_info_t *p, std::string *why) {
    if (!p) {
        return true;
    }
    const unsigned long long all =
        HS_CPU_FEATURES_AVX2 | HS_CPU_FEATURES_AVX512 | HS_CPU_FEATURES_AVX512VBMI;
    if (p->cpu_features & ~all) {
        *why = "Invalid cpu features specified in the platform information.";
        return false;
    }
    if (p->tune > HS_TUNE_FAMILY_ICX) {
        *why = "Invalid tuning value specified in the platform information.";
        return false;
    }
    return true;
}

/* Turn a regex that denotes a FINITE set of strings into that set: literal
 * characters and PCRE escapes as the reference parser accepts them
 * (src/parser/Parser.rl), groups "(...)" / "(?:...)" (Hyperscan does not
 * capture), alternation, character classes without negation, and the bounded
 * repeats "?", "{n}", "{n,m}".  Every string of the set becomes one literal of
 * the pure-literal matcher under the expression's id (the report rules dedupe
 * equal (id, to)), so such an expression needs none of the regex engines.
 * Throws a CompileError for every construct that does. */
class FiniteRegex {
public:
    FiniteRegex(const char *re_in, unsigned flags_in, int idx_in)
        : re(re_in), n(strlen(re_in)), flags(flags_in), idx(idx_in) {}

    std::vector<std::string> expand() {
        std::set<std::string> out = alt();
        if (pos != n) {
            fail("Unmatched parentheses.");
        }
        return std::vector<std::string>(out.begin(), out.end());
    }

private:
    static const size_t MAX_STRINGS = 4096;   /* literals one expression may expand to */
    static const size_t MAX_CLASS = 64;

    const char *re;
    size_t n, pos = 0;
    unsigned flags;
    int idx;

    [[noreturn]] void fail(const std::string &m) const { throw CompileError{m, idx}; }
    [[noreturn]] void needsRegex(const std::string &what) const {
        fail(what + " needs the regex back end; this build compiles expressions that denote a "
                    "finite set of literals only.");
    }
    bool at(char c) const { return pos < n && re[pos] == c; }

    static void cap(const std::set<std::string> &s, const FiniteRegex *self) {
        if (s.size() > MAX_STRINGS) {
            self->fail("Expression expands to more than 4096 literals; it needs the regex back end.");
        }
    }

    std::set<std::string> product(const std::set<std::string> &a, const std::set<std::string> &b) const {
        std::set<std::string> r;
        for (const std::string &x : a) {
            for (const std::string &y : b) {
                if (x.size() + y.size() > LIMIT_PATTERN_LENGTH) {
                    fail("Pattern length exceeds limit.");
                }
                r.insert(x + y);
            }
            cap(r, this);
        }
        return r;
    }

    std::set<std::string> alt() {
        std::set<std::string> r = seq();
        while (at('|')) {
            pos++;
            std::set<std::string> t = seq();
            r.insert(t.begin(), t.end());
            cap(r, this);
        }
        return r;
    }

    std::set<std::string> seq() {
        std::set<std::string> cur = {std::string()};
        while (pos < n && re[pos] != '|' && re[pos] != ')') {
            const std::set<std::string> a = atom();
            unsigned lo = 1, hi = 1;
            quantifier(&lo, &hi);
            std::set<std::string> opts, power = {std::string()};
            for (unsigned k = 0; k <= hi; k++) {
                if (k >= lo) {
                    opts.insert(power.begin(), power.end());
                    cap(opts, this);
                }
                if (k < hi) {
                    power = product(power, a);
                }
            }
            cur = product(cur, opts);
        }
        return cur;
    }

    void quantifier(unsigned *lo, unsigned *hi) {
        if (pos >= n) {
            return;
        }
        const char c = re[pos];
        if (c == '*' || c == '+') {
            needsRegex(std::string("Unbounded repeat '") + c + "'");
        }
        if (c == '?') {
            pos++;
            *lo = 0;
            *hi = 1;
        } else if (c == '{') {
            size_t q = pos + 1;
            unsigned long a = 0, b = 0;
            bool haveA = false, haveB = false, comma = false;
            while (q < n && isdigit((unsigned char)re[q])) {
                a = std::min(a * 10 + (re[q++] - '0'), 100000ul);
                haveA = true;
            }
            if (q < n && re[q] == ',') {
                comma = true;
                q++;
                while (q < n && isdigit((unsigned char)re[q])) {
                    b = std::min(b * 10 + (re[q++] - '0'), 100000ul);
                    haveB = true;
                }
            }
            if (!haveA || q >= n || re[q] != '}') {
                needsRegex("A '{' that does not start a repeat"); /* PCRE: literal brace */
            }
            if (comma && !haveB) {
                needsRegex("Unbounded repeat '{n,}'");
            }
            if (!comma) {
                b = a;
            }
            if (b < a) {
                fail("Bounded repeat is invalid: min > max.");
            }
            if (b > LIMIT_PATTERN_LENGTH) {
                fail("Bounded repeat is too large.");
            }
            pos = q + 1;
            *lo = (unsigned)a;
            *hi = (unsigned)b;
        } else {
            return;
        }
        if (pos < n && (re[pos] == '?' || re[pos] == '+')) {
            needsRegex("Lazy / possessive quantifier");
        }
    }

    static int hexval(char c) {
        if (c >= '0' && c <= '9') return c - '0';
        if (c >= 'a' && c <= 'f') return c - 'a' + 10;
        if (c >= 'A' && c <= 'F') return c - 'A' + 10;
        return -1;
    }

    /* one escaped character; pos is at the backslash */
    unsigned char escape(bool inClass) {
        if (++pos >= n) {
            fail("Unterminated escape at end of pattern.");
        }
        const unsigned char e = (unsigned char)re[pos++];
        switch (e) {
        case 'n': return '\n';
        case 't': return '\t';
        case 'r': return '\r';
        case 'f': return '\f';
        case 'a': return '\a';
        case 'e': return 0x1b;
        case 'x': {
            const int h1 = pos < n ? hexval(re[pos]) : -1;
            const int h2 = pos + 1 < n ? hexval(re[pos + 1]) : -1;
            if (h1 < 0 || h2 < 0) {
                needsRegex("A hex escape other than \\xHH");
            }
            pos += 2;
            return (unsigned char)(h1 * 16 + h2);
        }
        default:
            if (inClass && e == 'b') {
                return 0x08; /* backspace inside a class */
            }
            if (isalnum(e)) {
                needsRegex(std::string("Escape sequence \\") + (char)e);
            }
            return e; /* escaped punctuation */
        }
    }

    unsigned char plain(unsigned char c) const {
        if (c >= 0x80 && (flags & (HS_FLAG_UTF8 | HS_FLAG_UCP))) {
            fail("Non-ASCII characters under HS_FLAG_UTF8/UCP are not supported by the literal "
                 "compiler.");
        }
        return c;
    }

    /* "[...]": PCRE rules -- "]" first is literal, "-" is literal first, last or
     * right after a range */
    std::set<std::string> charClass() {
        pos++; /* [ */
        if (at('^')) {
            needsRegex("Negated character class");
        }
        bool present[256] = {false};
        bool first = true;
        int prev = -1; /* last single character that may start a range */
        for (;; first = false) {
            if (pos >= n) {
                fail("Unterminated character class.");
            }
            unsigned char c = (unsigned char)re[pos];
            if (c == ']' && !first) {
                pos++;
                break;
            }
            if (c == '[' && pos + 1 < n && (re[pos + 1] == ':' || re[pos + 1] == '.' || re[pos + 1] == '=')) {
                needsRegex("POSIX character class");
            }
            int lo;
            if (c == '-' && prev >= 0 && pos + 1 < n && re[pos + 1] != ']') {
                /* range prev-hi */
                pos++;
                unsigned char hi;
                if (re[pos] == '[' && pos + 1 < n && strchr(":.=", re[pos + 1])) {
                    fail("Invalid range in character class.");
                }
                if (re[pos] == '\\') {
                    hi = escape(true);
                } else {
                    hi = plain((unsigned char)re[pos++]);
                }
                if (hi < prev) {
                    fail("Invalid range in character class.");
                }
                for (int v = prev; v <= hi; v++) {
                    present[v] = true;
                }
                prev = -1; /* a "-" right after a range is literal */
                continue;
            }
            if (c == '\\') {
                lo = escape(true);
            } else {
                lo = plain(c);
                pos++;
            }
            present[lo] = true;
            prev = lo;
        }
        std::set<std::string> r;
        for (int v = 0; v < 256; v++) {
            if (present[v]) {
                r.insert(std::string(1, (char)v));
            }
        }
        if (r.size() > MAX_CLASS) {
            needsRegex("A character class of more than 64 characters");
        }
        return r;
    }

    std::set<std::string> atom() {
        const unsigned char c = (unsigned char)re[pos];
        if (c == '(') {
            pos++;
            if (at('?')) {
                if (pos + 1 < n && re[pos + 1] == ':') {
                    pos += 2;
                } else {
                    needsRegex("Group option / assertion \"(?\"");
                }
            }
            std::set<std::string> r = alt();
            if (!at(')')) {
                fail("Missing close parenthesis.");
            }
            pos++;
            return r;
        }
        if (c == '[') {
            /* "[:name:]", "[.x.]", "[=x=]" where a class should start (PCRE's check_posix_syntax) */
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
            return charClass();
        }
        if (c == '\\') {
            return {std::string(1, (char)escape(false))};
        }
        if (strchr(".^$", c)) {
            needsRegex(std::string("Metacharacter '") + (char)c + "'");
        }
        if (strchr("*+?{", c)) {
            fail("Invalid repeat: nothing to repeat.");
        }
        pos++;
        return {std::string(1, (char)plain(c))};
    }
};

static std::vector<std::string> regexToLiterals(const char *re, unsigned flags, int idx) {
    return FiniteRegex(re, flags, idx).expand();
}

static hs_error_t compileCommon(const char *const *expressions,
                                const unsigned *flags, const unsigned *ids,
                                const hs_expr_ext_t *const *ext,
                                const size_t *lens, unsigned elements,
                                unsigned mode, const hs_platform_info_t *platform,
                                hs_database_t **db, hs_compile_error_t **error,
                                bool litApi) {
    if (!error) {
        if (db) {
            *db = nullptr;
        }
        return HS_COMPILER_ERROR;
    }
    if (!db) {
        *error = makeError("Invalid parameter: db is NULL", -1);
        return HS_COMPILER_ERROR;
    }
    *db = nullptr;
    if (!expressions) {
        *error = makeError("Invalid parameter: expressions is NULL", -1);
        return HS_COMPILER_ERROR;
    }
    if (litApi && !lens) {
        *error = makeError("Invalid parameter: len is NULL", -1);
        return HS_COMPILER_ERROR;
    }
    if (elements == 0) {
        *error = makeError("Invalid parameter: elements is zero", -1);
        return HS_COMPILER_ERROR;
    }
    std::string why;
    if (!checkMode(mode, &why) || !checkPlatformInfo(platform, &why)) {
        *error = makeError(why, -1);
        return HS_COMPILER_ERROR;
    }
    try {
        std::vector<LitPattern> pats;
        pats.reserve(elements);
        std::vector<RegexPattern> rpats; /* every expression, for the NFA route */
        bool needNfa = false;
        for (unsigned i = 0; i < elements; i++) {
            const unsigned f = flags ? flags[i] : 0;
            if (!expressions[i]) {
                throw CompileError{"Invalid parameter: expression is NULL", (int)i};
            }
            const hs_expr_ext_t *xp = ext && ext[i] && ext[i]->flags != 0 ? ext[i] : nullptr;
            if (xp) {
                /* validation as src/compiler/compiler.cpp:80-110 */
                if (litApi) {
                    throw CompileError{"Extended parameters are not supported for pure literal matching API.", (int)i};
                }
                const unsigned long long known = HS_EXT_FLAG_MIN_OFFSET | HS_EXT_FLAG_MAX_OFFSET | HS_EXT_FLAG_MIN_LENGTH |
                                                 HS_EXT_FLAG_EDIT_DISTANCE | HS_EXT_FLAG_HAMMING_DISTANCE;
                if (xp->flags & ~known) {
                    throw CompileError{"Invalid hs_expr_ext flag set.", (int)i};
                }
                if ((xp->flags & HS_EXT_FLAG_MIN_OFFSET) && (xp->flags & HS_EXT_FLAG_MAX_OFFSET) &&
                    xp->min_offset > xp->max_offset) {
                    throw CompileError{"In hs_expr_ext, min_offset must be less than or equal to max_offset.", (int)i};
                }
                if ((xp->flags & HS_EXT_FLAG_MIN_LENGTH) && (xp->flags & HS_EXT_FLAG_MAX_OFFSET) &&
                    xp->min_length > xp->max_offset) {
                    throw CompileError{"In hs_expr_ext, min_length must be less than or equal to max_offset.", (int)i};
                }
                if (xp->flags & (HS_EXT_FLAG_EDIT_DISTANCE | HS_EXT_FLAG_HAMMING_DISTANCE)) {
                    throw CompileError{"Approximate matching (edit / Hamming distance) needs the reference's graph "
                                       "transformations; not supported.", (int)i};
                }
            }
            if (f & ~0x7ffu) {
                throw CompileError{"Unrecognised flag.", (int)i};
            }
            if ((f & HS_FLAG_SINGLEMATCH) && (f & HS_FLAG_SOM_LEFTMOST)) {
                throw CompileError{"HS_FLAG_SINGLEMATCH is not supported in "
                                   "combination with HS_FLAG_SOM_LEFTMOST.", (int)i};
            }
            LitPattern p;
            p.index = i;
            p.report = ids ? ids[i] : 0;
            p.caseless = f & HS_FLAG_CASELESS;
            p.singlematch = f & HS_FLAG_SINGLEMATCH;
            if (litApi) {
                const unsigned bad = HS_FLAG_DOTALL | HS_FLAG_ALLOWEMPTY | HS_FLAG_UTF8 |
                                     HS_FLAG_UCP | HS_FLAG_PREFILTER | HS_FLAG_COMBINATION |
                                     HS_FLAG_QUIET | HS_FLAG_MULTILINE;
                if (f & bad) {
                    throw CompileError{"Only HS_FLAG_CASELESS, HS_FLAG_SINGLEMATCH and "
                                       "HS_FLAG_SOM_LEFTMOST are supported in literal API.",
                                       (int)i};
                }
                if (lens[i] == 0 || expressions[i][0] == '\0') {
                    throw CompileError{"Pure literal API doesn't support empty string.", (int)i};
                }
                p.s.assign(expressions[i], lens[i]);
            } else {
                if (f & (HS_FLAG_COMBINATION | HS_FLAG_QUIET)) {
                    throw CompileError{"HS_FLAG_COMBINATION / HS_FLAG_QUIET need the regex "
                                       "back end; this build compiles literal patterns only.",
                                       (int)i};
                }
                if (f & HS_FLAG_SOM_LEFTMOST) {
                    throw CompileError{"HS_FLAG_SOM_LEFTMOST is not supported by the H100 "
                                       "literal compiler yet.", (int)i};
                }
                {
                    RegexPattern rp;
                    rp.re = expressions[i];
                    rp.flags = f;
                    rp.report = p.report;
                    rp.index = i;
                    if (xp) {
                        /* bounds on the match end and a minimum match length: the NFA route has them
                         * (CHECK_BOUNDS in the report programs; a length counter in the automaton) */
                        rp.minOffset = (xp->flags & HS_EXT_FLAG_MIN_OFFSET) ? xp->min_offset : 0;
                        rp.maxOffset = (xp->flags & HS_EXT_FLAG_MAX_OFFSET) ? xp->max_offset : ~0ull;
                        rp.minLength = (xp->flags & HS_EXT_FLAG_MIN_LENGTH) ? xp->min_length : 0;
                        needNfa = true;
                    }
                    rpats.push_back(rp);
                }
                if (xp) {
                    continue; /* (no literal expansion: the literal programs carry no bounds) */
                }
                /* one literal per string of the expression's (finite) language,
                 * all under the expression's id */
                std::vector<std::string> lang;
                try {
                    lang = regexToLiterals(expressions[i], f, (int)i);
                } catch (const CompileError &ce) {
                    if (ce.msg.find("regex back end") == std::string::npos) {
                        throw;
                    }
                    needNfa = true; /* not a finite set of literals: the whole set goes to one LimEx-32 NFA */
                    continue;
                }
                for (const std::string &str : lang) {
                    if (str.empty()) {
                        throw CompileError{(f & HS_FLAG_ALLOWEMPTY)
                                               ? "Empty patterns need the regex back end "
                                                 "(boundary reports)."
                                               : "Pattern matches empty buffer; use "
                                                 "HS_FLAG_ALLOWEMPTY to enable support.",
                                           (int)i};
                    }
                    p.s = str;
                    pats.push_back(p);
                }
                continue;
            }
            if (f & HS_FLAG_SOM_LEFTMOST) {
                throw CompileError{"HS_FLAG_SOM_LEFTMOST is not supported by the H100 "
                                   "literal compiler yet.", (int)i};
            }
            pats.push_back(p);
        }
        CompileOpts opts;
        opts.pureLiteralApi = litApi;
        opts.streaming = (mode & (HS_MODE_STREAM | HS_MODE_VECTORED)) != 0; /* isStreaming || isVectored: src/hs.cpp, util/compile_context.h:47-48 */
        opts.vectored = (mode & HS_MODE_VECTORED) != 0;
        if (platform && (platform->cpu_features & HS_CPU_FEATURES_AVX2)) {
            /* the caller targets AVX2+ reference runtimes: 16-bucket Teddy is
             * allowed and the database is stamped accordingly
             * (src/compiler/compiler.cpp:455-470 target_to_platform) */
            opts.hwlm.allowFatTeddy = true;
            opts.platform &= ~PLATFORM_NOAVX2;
            if (platform->cpu_features & HS_CPU_FEATURES_AVX512) {
                opts.platform &= ~PLATFORM_NOAVX512;
            }
            if (platform->cpu_features & HS_CPU_FEATURES_AVX512VBMI) {
                opts.platform &= ~PLATFORM_NOAVX512VBMI;
            }
        }
        applyBuildOptions(&opts.hwlm);
        opts.outfixKind = outfixEngineOption();
        opts.regexDfa = regexDfaOption() != 0;
        if (opts.hwlm.allowFatTeddy) {
            opts.platform &= ~PLATFORM_NOAVX2; /* 16-bucket Teddy needs AVX2 on CPUs */
        }
        std::vector<u8> bc = needNfa ? buildRegexRose(rpats, opts) : buildLiteralRose(pats, opts, nullptr);
        hs_error_t aerr;
        hs_database_t *out = dbCreate(bc, opts.platform, &aerr);
        if (!out) {
            *error = makeError("Could not allocate memory for bytecode.", -1);
            return HS_COMPILER_ERROR;
        }
        *db = out;
        *error = nullptr;
        return HS_SUCCESS;
    } catch (const CompileError &e) {
        *error = makeError(e.msg, e.index);
        return HS_COMPILER_ERROR;
    } catch (const std::bad_alloc &) {
        *error = &g_enomem;
        return HS_COMPILER_ERROR;
    } catch (const std::exception &e) {
        *error = makeError(std::string("Internal error: ") + e.what(), -1);
        return HS_COMPILER_ERROR;
    }
}

hs_error_t hs_compile_multi(const char *const *expressions, const unsigned *flags,
                            const unsigned *ids, unsigned elements, unsigned mode,
                            const hs_platform_info_t *platform, hs_database_t **db,
                            hs_compile_error_t **error) {
    return compileCommon(expressions, flags, ids, nullptr, nullptr, elements, mode,
                         platform, db, error, false);
}

hs_error_t hs_compile_ext_multi(const char *const *expressions,
                                const unsigned *flags, const unsigned *ids,
                                const hs_expr_ext_t *const *ext, unsigned elements,
                                unsigned mode, const hs_platform_info_t *platform,
                                hs_database_t **db, hs_compile_error_t **error) {
    return compileCommon(expressions, flags, ids, ext, nullptr, elements, mode,
                         platform, db, error, false);
}

hs_error_t hs_compile(const char *expression, unsigned flags, unsigned mode,
                      const hs_platform_info_t *platform, hs_database_t **db,
                      hs_compile_error_t **error) {
    if (expression == nullptr) {
        if (db) {
            *db = nullptr;
        }
        if (error) {
            *error = makeError("Invalid parameter: expression is NULL", -1);
        }
        return HS_COMPILER_ERROR;
    }
    unsigned id = 0;
    return compileCommon(&expression, &flags, &id, nullptr, nullptr, 1, mode,
                         platform, db, error, false);
}

hs_error_t hs_compile_lit_multi(const char *const *expressions,
                                const unsigned *flags, const unsigned *ids,
                                const size_t *lens, unsigned elements,
                                unsigned mode, const hs_platform_info_t *platform,
                                hs_database_t **db, hs_compile_error_t **error) {
    return compileCommon(expressions, flags, ids, nullptr, lens, elements, mode,
                         platform, db, error, true);
}

hs_error_t hs_compile_lit(const char *expression, unsigned flags, const size_t len,
                          unsigned mode, const hs_platform_info_t *platform,
                          hs_database_t **db, hs_compile_error_t **error) {
    if (expression == nullptr) {
        if (db) {
            *db = nullptr;
        }
        if (error) {
            *error = makeError("Invalid parameter: expression is NULL", -1);
        }
        return HS_COMPILER_ERROR;
    }
    unsigned id = 0;
    return compileCommon(&expression, &flags, &id, nullptr, &len, 1, mode, platform,
                         db, error, true);
}

/* hs_expression_info / hs_expression_ext_info (src/hs.cpp:337-432): widths of
 * a literal pattern are its byte length; a literal has no out-of-order or
 * end-of-data matches. */
static hs_error_t exprInfo(const char *expression, unsigned flags, const hs_expr_ext_t *ext,
                           hs_expr_info_t **info, hs_compile_error_t **error) {
    if (!error) {
        return HS_COMPILER_ERROR;
    }
    if (!info) {
        *error = makeError("Invalid parameter: info is NULL", -1);
        return HS_COMPILER_ERROR;
    }
    *info = nullptr;
    if (!expression) {
        *error = makeError("Invalid parameter: expression is NULL", -1);
        return HS_COMPILER_ERROR;
    }
    try {
        if (flags & ~0x7ffu) {
            throw CompileError{"Unrecognised flag.", 0};
        }
        if (ext && ext->flags != 0) {
            if (ext->flags & ~(HS_EXT_FLAG_MIN_OFFSET | HS_EXT_FLAG_MAX_OFFSET | HS_EXT_FLAG_MIN_LENGTH |
                               HS_EXT_FLAG_EDIT_DISTANCE | HS_EXT_FLAG_HAMMING_DISTANCE)) {
                throw CompileError{"Invalid hs_expr_ext flag set.", 0};
            }
            if ((ext->flags & HS_EXT_FLAG_MIN_OFFSET) && (ext->flags & HS_EXT_FLAG_MAX_OFFSET) &&
                ext->min_offset > ext->max_offset) {
                throw CompileError{"In hs_expr_ext, min_offset must be less than or equal to max_offset.", 0};
            }
            if ((ext->flags & HS_EXT_FLAG_MIN_LENGTH) && (ext->flags & HS_EXT_FLAG_MAX_OFFSET) &&
                ext->min_length > ext->max_offset) {
                throw CompileError{"In hs_expr_ext, min_length must be less than or equal to max_offset.", 0};
            }
            if (ext->flags & (HS_EXT_FLAG_EDIT_DISTANCE | HS_EXT_FLAG_HAMMING_DISTANCE)) {
                throw CompileError{"Approximate matching (edit / Hamming distance) needs the reference's graph "
                                   "transformations; not supported.", 0};
            }
        }
        size_t minW = 0, maxW = 0;
        RegexInfo ri;
        try {
            const std::vector<std::string> lang = regexToLiterals(expression, flags, 0);
            minW = lang.empty() ? 0 : lang[0].size();
            for (const std::string &str : lang) {
                minW = std::min(minW, str.size());
                maxW = std::max(maxW, str.size());
            }
        } catch (const CompileError &ce) {
            if (ce.msg.find("regex back end") == std::string::npos) {
                throw;
            }
            try { /* not a finite set of literals: the NFA route's parser knows the widths */
                ri = regexInfo(expression, flags, true);
                minW = ri.minLen;
                maxW = ri.maxLen; /* 0xffffffff = unbounded, as in the reference (src/hs.cpp:398-403) */
            } catch (const RegexError &re) {
                throw CompileError{re.msg, 0};
            }
        }
        hs_expr_info_t *out = (hs_expr_info_t *)g_misc_alloc(sizeof(*out));
        if (!out) {
            *error = &g_enomem;
            return HS_COMPILER_ERROR;
        }
        memset(out, 0, sizeof(*out));
        if (ext && (ext->flags & HS_EXT_FLAG_MIN_LENGTH) && ext->min_length <= 0xfffffffeull) {
            /* a min_length is a lower bound for the match width (checkVertex, src/nfagraph/ng_expr_info.cpp:104-109) */
            minW = std::max<size_t>(minW, (size_t)ext->min_length);
            maxW = std::max<size_t>(maxW, (size_t)ext->min_length);
        }
        if (ext && (ext->flags & HS_EXT_FLAG_MAX_OFFSET) && ext->max_offset && ext->max_offset <= 0xfffffffeull) {
            /* ... and a max_offset an upper bound (:111-116) */
            minW = std::min<size_t>(minW, (size_t)ext->max_offset);
            maxW = std::min<size_t>(maxW, (size_t)ext->max_offset);
        }
        out->min_width = (unsigned)minW;
        out->max_width = (unsigned)maxW;
        out->unordered_matches = ri.unordered;
        out->matches_at_eod = ri.atEod;
        out->matches_only_at_eod = ri.onlyAtEod;
        *info = out;
        *error = nullptr;
        return HS_SUCCESS;
    } catch (const CompileError &e) {
        *error = makeError(e.msg, e.index);
        return HS_COMPILER_ERROR;
    }
}

hs_error_t hs_expression_info(const char *expression, unsigned int flags, hs_expr_info_t **info,
                              hs_compile_error_t **error) {
    return exprInfo(expression, flags, nullptr, info, error);
}

hs_error_t hs_expression_ext_info(const char *expression, unsigned int flags,
                                  const hs_expr_ext_t *ext, hs_expr_info_t **info,
                                  hs_compile_error_t **error) {
    return exprInfo(expression, flags, ext, info, error);
}

} /* extern "C" */

/* Build tunables (test / tuning hooks): select table variants the way the
 * reference's unit tests force engines through hints
 * (unit/internal/fdr.cpp:114-137, src/fdr/fdr_compile.cpp:862-866) and its
 * tools override Grey values with -G.  Keys: "force_engine" (-1 auto, 0 FDR,
 * 3..18 Teddy id), "fdr_domain", "fdr_stride", "max_domain", "allow_teddy",
 * "allow_fat_teddy", "allow_flood", "allow_noodle"; "outfix_engine" (0 = literal
 * matchers as usual; 1 DFA chosen by size, 2 McClellan-8, 3 McClellan-16, 4 Sheng,
 * 5 LimEx-32: block-mode literal sets are compiled to a database whose only matcher is
 * that engine run as an outfix, ROSE_RUNTIME_SINGLE_OUTFIX); "regex_dfa" (1: regular expressions whose
 * determinised automaton stays small run as a McClellan DFA, 0: always as a LimEx NFA). */
namespace hsb {
static HwlmBuildOpts g_tunables;
static bool g_tun_set[8];
static int g_outfixEngine = 0; /* "outfix_engine": see enum OutfixKind (rose_build.h) */
static int g_regexDfa = 1;     /* "regex_dfa": 0 = expressions always become a LimEx NFA */
int outfixEngineOption() { return g_outfixEngine; }
int regexDfaOption() { return g_regexDfa; }
void applyBuildOptions(HwlmBuildOpts *o) {
    if (g_tun_set[0]) o->forceEngine = g_tunables.forceEngine;
    if (g_tun_set[1]) o->forceDomain = g_tunables.forceDomain;
    if (g_tun_set[2]) o->forceStride = g_tunables.forceStride;
    if (g_tun_set[3]) o->maxDomain = g_tunables.maxDomain;
    if (g_tun_set[4]) o->allowTeddy = g_tunables.allowTeddy;
    if (g_tun_set[5]) o->allowFatTeddy = g_tunables.allowFatTeddy;
    if (g_tun_set[6]) o->allowFlood = g_tunables.allowFlood;
    if (g_tun_set[7]) o->allowNoodle = g_tunables.allowNoodle;
}
} // namespace hsb

extern "C" hs_error_t hs_b200_set_build_option(const char *key, int value) {
    if (!key) {
        return HS_INVALID;
    }
    std::string k(key);
    if (k == "reset") {
        memset(g_tun_set, 0, sizeof(g_tun_set));
        g_tunables = HwlmBuildOpts();
        hsb::g_outfixEngine = 0;
        hsb::g_regexDfa = 1;
        return HS_SUCCESS;
    }
    if (k == "regex_dfa") {
        hsb::g_regexDfa = value != 0;
        return HS_SUCCESS;
    }
    if (k == "outfix_engine") {
        if (value < 0 || value > 5) {
            return HS_INVALID;
        }
        hsb::g_outfixEngine = value;
        return HS_SUCCESS;
    }
    struct { const char *n; int i; } keys[] = {
        {"force_engine", 0}, {"fdr_domain", 1}, {"fdr_stride", 2}, {"max_domain", 3},
        {"allow_teddy", 4}, {"allow_fat_teddy", 5}, {"allow_flood", 6}, {"allow_noodle", 7}};
    for (auto &e : keys) {
        if (k == e.n) {
            switch (e.i) {
            case 0: g_tunables.forceEngine = value; break;
            case 1: g_tunables.forceDomain = value; break;
            case 2: g_tunables.forceStride = value; break;
            case 3: g_tunables.maxDomain = value; break;
            case 4: g_tunables.allowTeddy = value != 0; break;
            case 5: g_tunables.allowFatTeddy = value != 0; break;
            case 6: g_tunables.allowFlood = value != 0; break;
            case 7: g_tunables.allowNoodle = value != 0; break;
            }
            g_tun_set[e.i] = true;
            return HS_SUCCESS;
        }
    }
    return HS_INVALID;
}

/* Table-builder entry point at the boundary the reference's unit tests use
 * (hwlmBuild(), unit/internal/fdr.cpp:140-165): builds a raw HWLM table for
 * literals given as (bytes, nocase, noruns, id).  engine: -1 auto, 0 FDR,
 * 3..18 Teddy id.  Returns the table size, or -1 if it cannot be built / does
 * not fit `cap`. */
extern "C" long hs_b200_test_build_hwlm(const char *const *lits, const size_t *lens,
                                        const unsigned *nocase, const unsigned *noruns,
                                        const unsigned *ids, unsigned n, int engine, void *out,
                                        size_t cap) {
    try {
        std::vector<HwlmLit> v;
        for (unsigned i = 0; i < n; i++) {
            HwlmLit l;
            l.s.assign(lits[i], lens[i]);
            l.nocase = nocase[i] != 0;
            if (l.nocase) {
                for (char &c : l.s) {
                    c = (char)asciiUpper((u8)c);
                }
            }
            l.noruns = noruns[i] != 0;
            l.id = ids[i];
            l.groups = 1;
            v.push_back(l);
        }
        HwlmBuildOpts o;
        o.forceEngine = engine;
        if (engine == 0) {
            o.forceDomain = 9; /* the unit-test hint: src/fdr/fdr_compile.cpp:862-866 */
            o.forceStride = 1;
        }
        if (engine >= 3 && engine <= 10) {
            o.allowFatTeddy = true;
        }
        std::vector<u8> t = buildHwlm(v, o, nullptr);
        if (t.size() > cap) {
            return -1;
        }
        memcpy(out, t.data(), t.size());
        return (long)t.size();
    } catch (const std::exception &) {
        return -1;
    }
}

/* Test hook: a pure-literal block database whose literal programs are raw
 * instruction bytes supplied by the caller (tests/test_programs.py assembles them
 * from the layouts in src/rose/rose_program.h), so that every opcode of
 * roseRunProgram_l can be reached on the device and by the reference runtime
 * from the same bytes.  `area` lands at hs_b200_test_program_base() in the
 * bytecode; prog_off[i] is literal i's program inside it. */
extern "C" unsigned hs_b200_test_program_base(void) { return programAreaBase(); }

extern "C" hs_error_t hs_b200_test_compile_programs(const char *const *lits, const size_t *lens,
                                                    const unsigned *nocase, const unsigned *prog_off,
                                                    unsigned n, const void *area, size_t area_len,
                                                    unsigned ekey_count, const unsigned *inv_dkey,
                                                    unsigned dkey_count, hs_database_t **db) {
    if (!lits || !lens || !nocase || !prog_off || !area || !db || !n) {
        return HS_INVALID;
    }
    try {
        std::vector<HwlmLit> v;
        for (unsigned i = 0; i < n; i++) {
            HwlmLit l;
            l.s.assign(lits[i], lens[i]);
            l.nocase = nocase[i] != 0;
            if (l.nocase) {
                for (char &c : l.s) {
                    c = (char)asciiUpper((u8)c);
                }
            }
            l.id = prog_off[i];
            l.groups = 1;
            v.push_back(l);
        }
        CompileOpts opts;
        opts.pureLiteralApi = true;
        applyBuildOptions(&opts.hwlm);
        if (opts.hwlm.allowFatTeddy) {
            opts.platform &= ~PLATFORM_NOAVX2;
        }
        std::vector<u8> a((const u8 *)area, (const u8 *)area + area_len);
        std::vector<u32> inv(inv_dkey ? inv_dkey : nullptr, inv_dkey ? inv_dkey + dkey_count : nullptr);
        std::vector<u8> bc = buildRawProgramRose(v, a, ekey_count, inv, opts, nullptr);
        hs_error_t aerr;
        hs_database_t *out = dbCreate(bc, opts.platform, &aerr);
        if (!out) {
            return aerr;
        }
        *db = out;
        return HS_SUCCESS;
    } catch (const CompileError &) {
        return HS_COMPILER_ERROR;
    } catch (const std::exception &) {
        return HS_COMPILER_ERROR;
    }
}

/* ---- DFA engine emitters (host/dfa_build.h) ---------------------------------------
 * Return the engine's size in bytes (struct NFA first, the reference's own layout),
 * or -1 if it cannot be built / does not fit `cap`. */
static long emitInto(const hsb::RawDfa &d, int kind, int sherman, void *out, size_t cap) {
    std::vector<u8> b = hsb::emitDfa(d, (hsb::DfaKind)kind, sherman != 0);
    if (b.size() > cap || !out) {
        return -1;
    }
    memcpy(out, b.data(), b.size());
    return (long)b.size();
}

extern "C" long hs_b200_dfa_from_literals(const char *const *lits, const size_t *lens, const unsigned *caseless,
                                          const unsigned *reports, unsigned n, int anchored, int kind,
                                          int sherman, void *out, size_t cap) {
    if (!lits || !lens || !reports || !n) {
        return -1;
    }
    try {
        std::vector<hsb::DfaLiteral> v(n);
        for (unsigned i = 0; i < n; i++) {
            v[i].s.assign(lits[i], lens[i]);
            v[i].caseless = caseless && caseless[i];
            v[i].report = reports[i];
        }
        return emitInto(hsb::dfaFromLiterals(v, anchored != 0), kind, sherman, out, cap);
    } catch (const std::exception &) {
        return -1;
    }
}

extern "C" long hs_b200_dfa_from_table(unsigned nstates, const unsigned short *next, unsigned start_anchored,
                                       unsigned start_floating, const unsigned *report_off,
                                       const unsigned *reports, const unsigned *eod_off,
                                       const unsigned *eod_reports, int kind, int sherman, void *out,
                                       size_t cap) {
    if (!next || !report_off || !eod_off || nstates < 2) {
        return -1;
    }
    try {
        hsb::RawDfa d;
        d.next.resize(nstates);
        d.reports.resize(nstates);
        d.reportsEod.resize(nstates);
        for (unsigned s = 0; s < nstates; s++) {
            for (unsigned c = 0; c < 256; c++) {
                d.next[s][c] = next[(size_t)s * 256 + c];
            }
            d.reports[s].assign(reports + report_off[s], reports + report_off[s + 1]);
            d.reportsEod[s].assign(eod_reports + eod_off[s], eod_reports + eod_off[s + 1]);
        }
        d.startAnchored = (u16)start_anchored;
        d.startFloating = (u16)start_floating;
        return emitInto(d, kind, sherman, out, cap);
    } catch (const std::exception &) {
        return -1;
    }
}

/* ---- LimEx-32 emitters (include/hs_b200.h) ------------------------------------------- */

static long copyOut(const std::vector<u8> &b, void *out, size_t cap) {
    if (b.size() > cap || !out) {
        return -1;
    }
    memcpy(out, b.data(), b.size());
    return (long)b.size();
}

extern "C" long hs_b200_limex32_from_literals(const char *const *lits, const size_t *lens, const unsigned *caseless,
                                              const unsigned *reports, unsigned n, void *out, size_t cap) {
    if (!lits || !lens || !reports || !n) {
        return -1;
    }
    try {
        std::vector<hsb::DfaLiteral> v(n);
        for (unsigned i = 0; i < n; i++) {
            v[i].s.assign(lits[i], lens[i]);
            v[i].caseless = caseless && caseless[i];
            v[i].report = reports[i];
        }
        return copyOut(hsb::emitLimEx(hsb::nfaFromLiterals(v)), out, cap);
    } catch (const std::exception &) {
        return -1;
    }
}

/* state sets as `words` little-endian 64-bit words each */
static hsb::StateSet setFromWords(const unsigned long long *w, unsigned words) {
    hsb::StateSet s;
    for (unsigned j = 0; j < words; j++) {
        s |= hsb::stateSetOf(w[j]) << (64 * j);
    }
    return s;
}

static long limexFromSpec(unsigned nstates, unsigned words, const unsigned long long *reach256,
                          const unsigned long long *init, const unsigned long long *init_ds,
                          const unsigned long long *succ, const unsigned long long *squash_mask,
                          const unsigned char *squash_kind, const unsigned *report_off, const unsigned *reports,
                          const unsigned *eod_off, const unsigned *eod_reports, void *out, size_t cap) {
    if (!reach256 || !succ || !init || !init_ds || !report_off || !eod_off || nstates == 0 || words == 0 ||
        words > hsb::MAX_NFA_STATES / 64 || nstates > 64 * words) {
        return -1;
    }
    try {
        hsb::RawNfa n;
        n.nstates = nstates;
        for (unsigned b = 0; b < 256; b++) {
            n.reach[b] = setFromWords(reach256 + (size_t)b * words, words);
        }
        n.init = setFromWords(init, words);
        n.initDS = setFromWords(init_ds, words);
        n.succ.resize(nstates);
        n.squashMask.assign(nstates, hsb::allStates());
        n.squashKind.assign(nstates, 0);
        n.reports.resize(nstates);
        n.reportsEod.resize(nstates);
        for (unsigned i = 0; i < nstates; i++) {
            n.succ[i] = setFromWords(succ + (size_t)i * words, words);
            if (squash_mask && squash_kind) {
                n.squashMask[i] = setFromWords(squash_mask + (size_t)i * words, words);
                n.squashKind[i] = squash_kind[i];
            }
            n.reports[i].assign(reports + report_off[i], reports + report_off[i + 1]);
            n.reportsEod[i].assign(eod_reports + eod_off[i], eod_reports + eod_off[i + 1]);
        }
        return copyOut(hsb::emitLimEx(n), out, cap);
    } catch (const std::exception &) {
        return -1;
    }
}

extern "C" long hs_b200_limex_from_spec_wide(unsigned nstates, unsigned words, const unsigned long long *reach256,
                                             const unsigned long long *init, const unsigned long long *init_ds,
                                             const unsigned long long *succ, const unsigned long long *squash_mask,
                                             const unsigned char *squash_kind, const unsigned *report_off,
                                             const unsigned *reports, const unsigned *eod_off,
                                             const unsigned *eod_reports, void *out, size_t cap) {
    return limexFromSpec(nstates, words, reach256, init, init_ds, succ, squash_mask, squash_kind, report_off, reports,
                         eod_off, eod_reports, out, cap);
}

extern "C" long hs_b200_limex_from_spec64(unsigned nstates, const unsigned long long *reach256,
                                          unsigned long long init, unsigned long long init_ds,
                                          const unsigned long long *succ, const unsigned long long *squash_mask,
                                          const unsigned char *squash_kind, const unsigned *report_off,
                                          const unsigned *reports, const unsigned *eod_off,
                                          const unsigned *eod_reports, void *out, size_t cap) {
    if (nstates > 64) {
        return -1;
    }
    return limexFromSpec(nstates, 1, reach256, &init, &init_ds, succ, squash_mask, squash_kind, report_off, reports,
                         eod_off, eod_reports, out, cap);
}

extern "C" long hs_b200_limex32_from_spec(unsigned nstates, const unsigned *reach256, unsigned init, unsigned init_ds,
                                          const unsigned *succ, const unsigned *squash_mask,
                                          const unsigned char *squash_kind, const unsigned *report_off,
                                          const unsigned *reports, const unsigned *eod_off,
                                          const unsigned *eod_reports, void *out, size_t cap) {
    if (!reach256 || !succ || nstates == 0 || nstates > 32) {
        return -1;
    }
    std::vector<unsigned long long> r(reach256, reach256 + 256), sc(succ, succ + nstates), sq;
    if (squash_mask) {
        sq.assign(squash_mask, squash_mask + nstates);
    }
    const unsigned long long i0 = init, i1 = init_ds;
    return limexFromSpec(nstates, 1, r.data(), &i0, &i1, sc.data(), squash_mask ? sq.data() : nullptr, squash_kind,
                         report_off, reports, eod_off, eod_reports, out, cap);
}
