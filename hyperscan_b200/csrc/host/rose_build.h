/*
 * rose_build.h -- host-side assembly of a pure-literal RoseEngine bytecode
 * (programs + floating literal matcher) and the hs_database container.
 * Stands where the reference's RoseBuildImpl::buildFinalEngine + dbCreate stand
 * (src/rose/rose_build_bytecode.cpp:3609-3888, src/compiler/compiler.cpp:476-
 * 536), restricted to databases whose runtimeImpl is ROSE_RUNTIME_PURE_LITERAL,
 * ROSE_RUNTIME_SINGLE_OUTFIX, or ROSE_RUNTIME_FULL_ROSE with only the floating
 * literal matcher and one outfix, or with any number of outfixes and no literal matcher.
 */
#ifndef HSB200_ROSE_BUILD_H
#define HSB200_ROSE_BUILD_H

#include <string>
#include <vector>

#include "hwlm_build.h"

namespace hsb {

struct CompileError {
    std::string msg;
    int index; /* expression index or -1 */
};

} // namespace hsb

#include "logical.h"

namespace hsb {

struct LitPattern {
    std::string s;      /* raw bytes of the literal */
    bool caseless = false;
    bool singlematch = false;
    bool quiet = false; /* HS_FLAG_QUIET: no report, only its part in combinations */
    u32 report = 0;     /* user-visible id */
    u32 index = 0;      /* position in the caller's expression array */
};

struct CompileOpts {
    bool pureLiteralApi = false; /* hs_compile_lit*: sets RoseEngine.pureLiteral */
    bool streaming = false;      /* HS_MODE_STREAM / HS_MODE_VECTORED: history + per-stream state
                                  * (literals <= 8 bytes); src/util/compile_context.h:47-48 */
    bool vectored = false;       /* HS_MODE_VECTORED: a streaming database stamped for hs_scan_vector */
    bool smallWrite = true;      /* block mode: also emit the small-write DFA (src/smallwrite/) for buffers
                                  * shorter than 70 bytes when the literal set's automaton stays small */
    int outfixKind = 0;          /* != 0: no literal matcher, ONE engine over the whole literals run as an
                                  * outfix (ROSE_RUNTIME_SINGLE_OUTFIX): see enum OutfixKind */
    bool regexDfa = true;        /* regex route: determinise the position automaton when the DFA stays small
                                  * (McClellan-8 up to 256 states, McClellan-16 up to 1024), else LimEx */
    u64 platform = PLATFORM_NOAVX2 | PLATFORM_NOAVX512 | PLATFORM_NOAVX512VBMI;
    HwlmBuildOpts hwlm;
};

enum OutfixKind { OUTFIX_NONE = 0, OUTFIX_DFA_AUTO = 1, OUTFIX_MCCLELLAN8 = 2, OUTFIX_MCCLELLAN16 = 3, OUTFIX_SHENG = 4,
                  OUTFIX_LIMEX32 = 5 };

/* grey-box limits mirrored from src/grey.cpp:40-160 */
static const size_t LIMIT_PATTERN_LENGTH = 16000;
static const size_t LIMIT_LITERAL_LENGTH = 1600;
static const size_t LIMIT_LITERAL_COUNT = 8000000;

/** Build the RoseEngine bytecode for a set of literal patterns.  `logic` (may be null): the
 * logical combinations over them; combinations with HS_FLAG_SINGLEMATCH get their ekeys here. */
std::vector<u8> buildLiteralRose(const std::vector<LitPattern> &pats,
                                 const CompileOpts &opts, HwlmBuildInfo *info, LogicalSet *logic = nullptr);

/** Expressions that need an NFA (regex_nfa.h): ONE LimEx-32 engine over all of them, run as the
 * database's single outfix (ROSE_RUNTIME_SINGLE_OUTFIX).  Block mode only.  Throws CompileError. */
struct RegexPattern {
    std::string re;
    unsigned flags = 0;
    u32 report = 0;
    u32 index = 0;
    u64 minOffset = 0, maxOffset = ~0ull; /* hs_expr_ext: bounds on the match end (CHECK_BOUNDS in the report programs) */
    u64 minLength = 0;                    /* hs_expr_ext: shortest match that counts (regex_nfa.cpp) */
};
std::vector<u8> buildRegexRose(const std::vector<RegexPattern> &pats, const CompileOpts &opts,
                               LogicalSet *logic = nullptr);

/** A set of literals AND expressions that need an engine (ROSE_RUNTIME_FULL_ROSE): the floating
 * literal matcher over `lits`, whose programs catch the outfix up before they report, and ONE
 * engine over `regexes` as the outfix on queue 0.  Report ids share their exhaustion and dedupe
 * keys across both halves.  Block mode only; no logical combinations.  Throws CompileError. */
std::vector<u8> buildMixedRose(const std::vector<LitPattern> &lits, const std::vector<RegexPattern> &regexes,
                               const CompileOpts &opts, HwlmBuildInfo *info);

/** Expressions too many for one engine (ROSE_RUNTIME_FULL_ROSE without a literal matcher): the
 * expressions packed greedily, in order, into groups whose automaton fits one engine, and each group's
 * engine (McClellan-8 / 16 or LimEx, as buildRegexRose picks it) as the outfix on its own queue, as many
 * queues as there are groups.  Report ids share their exhaustion and dedupe keys across all engines.  Block
 * mode only; no logical combinations.  Throws CompileError, also when one expression alone does not fit. */
std::vector<u8> buildMultiOutfixRose(const std::vector<RegexPattern> &pats, const CompileOpts &opts);

/** The sparse iterator over `keys` (ascending, each < totalBits) of a multibit of totalBits bits, as
 * mmbBuildSparseIterator lays it out (src/util/multibit_build.cpp:158-206): one record per node of the key
 * tree that holds a key, breadth first; one record while totalBits <= 64. */
std::vector<MmbSparseIter> mmbSparseIterator(const std::vector<u32> &keys, u32 totalBits);

/** The scatter units that clear a multibit of totalBits bits at state offset `at` (mmbBuildClearPlan,
 * src/util/multibit_build.cpp:208-325): the flat form (<= 256 bits) as 64-bit words and a last word of 1-64
 * bits split into u64 / u32 / u16 / u8 units; the tree form (> 256 bits) as its root word. */
struct MmbClearPlan {
    std::vector<ScatterUnitU64> u64s;
    std::vector<ScatterUnitU32> u32s;
    std::vector<ScatterUnitU16> u16s;
    std::vector<ScatterUnitU8> u8s;
};
MmbClearPlan mmbClearPlan(u32 totalBits, u32 at);

/** Test hook: pure-literal block database from raw literal programs (`area`
 * is placed at programAreaBase(); lits[i].id = its program's offset in area). */
u32 programAreaBase();
std::vector<u8> buildRawProgramRose(std::vector<HwlmLit> lits, const std::vector<u8> &area,
                                    u32 ekeyCount, const std::vector<u32> &invDkey,
                                    const CompileOpts &opts, HwlmBuildInfo *info);

} // namespace hsb
#endif
