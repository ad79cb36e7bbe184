/*
 * db_walk.h -- how a database's raw match records become delivered matches: the
 * database's shape, the walk over its report programs (the literal programs held in
 * the hash-confirm structures, src/fdr/fdr_confirm.h:36-94, and the engine's report
 * programs), the reports that carry an exhaustion key (HS_FLAG_SINGLEMATCH;
 * REPORT_EXHAUST, src/rose/rose_program.h:485), and the order-dependent report
 * rules -- logical combinations included -- applied to a list of raw records.
 */
#ifndef HSB200_DB_WALK_H
#define HSB200_DB_WALK_H

#include <set>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../../include/hs_b200.h"
#include "../ref_layout.h"

namespace hsb {

static_assert(sizeof(DevMatch) == sizeof(hs_b200_match_t) && offsetof(DevMatch, id) == offsetof(hs_b200_match_t, id) &&
                  offsetof(DevMatch, block) == offsetof(hs_b200_match_t, block) &&
                  offsetof(DevMatch, to) == offsetof(hs_b200_match_t, to),
              "record layout");

/* Delivery order of records: by block, then end offset, then id. */
struct RecordOrder {
    bool operator()(const DevMatch &a, const DevMatch &b) const {
        if (a.block != b.block) return a.block < b.block;
        if (a.to != b.to) return a.to < b.to;
        return a.id < b.id;
    }
};

struct LitTail {
    u64 v, msk;
    u32 size;
    u32 bucket;
};

/* a report instruction of a program: what it raises, and the bounds on the match end (CHECK_BOUNDS,
 * src/rose/program_runtime.c:2319-2326) under which the program reaches it */
struct ProgReport {
    u32 onmatch;     /* report id, or the lkey of a SET_LOGICAL */
    s32 offset_adjust;
    u64 min_bound, max_bound;
    bool logical = false;
};
/* lkey -> the report id whose report block sets it (a SET_LOGICAL after a report instruction; a quiet
 * sub-expression has none) */
typedef std::unordered_map<u32, u32> LkeyReports;

/* Logical combinations of a database (RoseEngine.ckeyCount != 0): the tables the reference evaluates
 * per block (src/rose/program_runtime.c:2026-2120, src/report.h:190-245), copied from the bytecode. */
struct Combinations {
    u32 lkeyCount = 0;
    u32 minWidth = 0;                 /* blocks shorter than this are not scanned (src/runtime.c:346) */
    std::vector<LogicalOp> tree;
    std::vector<CombInfo> combs;
    std::vector<std::vector<u32>> ckeysOf; /* lkey -> the combinations that name it, ascending */
    LkeyReports lkeyReport;
    bool any() const { return !combs.empty(); }
};

/* The bit of DevMatch.to that marks a logical-key record (id = lkey): written by SET_LOGICAL, consumed by
 * the combination rules.  No match offset reaches 2^63. */
static const u64 LKEY_RECORD = 1ull << 63;
/* The bit of DevMatch.to that marks an engine's record in a database with a literal matcher and an
 * outfix: its id is a report PROGRAM offset, resolved on the host; the literal records carry report ids. */
static const u64 ENGINE_RECORD = 1ull << 62;

/* The database shapes the device runs (DESIGN.md sections 10a, 10d, 10e). */
enum DbShape {
    SHAPE_UNSUPPORTED = 0, /* needs the full rose interpreter (SURVEY.md section 8f rank 1): not in this build */
    SHAPE_PURE_LITERAL,    /* the floating literal matcher alone */
    SHAPE_SOLE_OUTFIX,     /* one engine over the whole block, no literal matcher */
    SHAPE_LITERALS_OUTFIX, /* the floating literal matcher beside one outfix (FULL_ROSE, block mode) */
    SHAPE_OUTFIXES,        /* any number of outfixes and no literal matcher (FULL_ROSE, block mode) */
    SHAPE_MALFORMED,       /* the header of SHAPE_OUTFIXES, but its queue, state or EOD tables do not fit its queue
                            * count or its bytecode: refused with HS_INVALID */
};
DbShape dbShape(const hs_database_t *db);

/* The report rules of one database.  Borrows the database's bytecode, which must outlive it. */
struct ReportRules {
    DbShape shape = SHAPE_UNSUPPORTED;
    bool hasDedupe = false;                /* RoseEngine.dkeyCount != 0 */
    std::unordered_set<u32> exhaustible;   /* report ids under HS_FLAG_SINGLEMATCH (an engine's: found with its
                                            * programs as they are first met) */
    Combinations comb;
    const u8 *bc = nullptr;
    u32 bcLen = 0;
    /* an engine's report program offset -> the report instructions it reaches, filled as programs are met */
    std::unordered_map<u32, std::vector<ProgReport>> progReports;
    /* the report ids the programs walked so far can raise (logical keys excluded) */
    std::set<u32> reportIds;
    /* the smallest offset_adjust of the programs walked so far (at most 0): after loadReportRules (every literal
     * program) and buildDeviceRules (every engine program), no report lies more than -minAdjust bytes before the
     * raw end offset of the match that raised it */
    s32 minAdjust = 0;

    /* Without dedupe keys, exhaustion keys, combinations or engine records, the raw record count is the
     * delivered count. */
    bool rawCountDelivered() const {
        return shape == SHAPE_PURE_LITERAL && exhaustible.empty() && !hasDedupe && !comb.any();
    }

    /* Records of a scan in delivery order, (block, to, id), with the report rules the device skipped
     * applied.  An engine's records carry report PROGRAM offsets (and the padding of the lanes' reserved
     * slots) -- all records of a database without a literal matcher, and those tagged ENGINE_RECORD beside
     * a literal matcher; each is replaced by the reports its program raises -- roseReportAdaptor -> roseRunProgram
     * (src/rose/match.c:611-633) -- with CHECK_BOUNDS and offset_adjust applied, and the literals' records
     * join them as they are.  Then one report per (block, id, to) (dedupe, src/report.h:55-119) and, for
     * HS_FLAG_SINGLEMATCH reports, only the first match per block (exhaustion keys, src/report.h:121-147,
     * program_runtime.c:464-481); with logical combinations, the combination reports are added and the
     * logical-key records removed, which needs the block lengths (lengths[0, nblocks)). */
    hs_error_t deliver(std::vector<DevMatch> *v, const u32 *lengths, size_t nblocks);
};

/* Classify the database and walk the floating matcher's literal programs once: HS_ARCH_ERROR for a shape
 * the device does not run, or for a program that holds an opcode the device does not implement (callers
 * refuse the database instead of failing mid-scan).  tails, if given, receives the LitInfo v/msk/size and
 * bucket of every literal of an FDR or Teddy matcher. */
hs_error_t loadReportRules(const hs_database_t *db, ReportRules *rules, std::vector<LitTail> *tails = nullptr);

/* The report rules as tables, for the device's form of ReportRules::deliver (order_kernels.h). */
struct DeviceRules {
    /* every report program the engine can raise, ascending; program k's report instructions are
     * reps[progStart[k], progStart[k + 1]) */
    std::vector<u32> progOff, progStart;
    std::vector<ProgReport> reps;
    u32 maxFanout = 1;  /* the most records one input record becomes (at least 1: a literal's record) */
    s32 maxAdjust = 0;  /* the largest offset_adjust (at least 0) */
    /* every report id a record can carry, ascending (the dense rank of an id is its index), and whether
     * it is exhaustible (HS_FLAG_SINGLEMATCH) */
    std::vector<u32> ids;
    std::vector<u8> idExhaustible;
};
/* an engine's bytes, struct NFA first */
struct EngineBytes {
    const u8 *nfa;
    u32 len;
};
/* The engines of a database with outfixes (queues [0, queueCount)), in queue order; false when its queue table or
 * an engine does not lie inside its bytecode. */
bool outfixEngines(const hs_database_t *db, std::vector<EngineBytes> *out);
/* Walk every report program of the engines (none for a pure-literal database) as ReportRules::deliver
 * would on meeting it, which completes rules->progReports and rules->exhaustible, and lay the rules out
 * as tables.  HS_INVALID: an engine's report lists run past its end; HS_UNKNOWN_ERROR: a program holds an
 * opcode the device does not implement. */
hs_error_t buildDeviceRules(ReportRules *rules, const std::vector<EngineBytes> &engines, DeviceRules *out);

} // namespace hsb
#endif
