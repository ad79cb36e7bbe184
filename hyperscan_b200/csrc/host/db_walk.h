/*
 * db_walk.h -- host-side walks over a literal database's bytecode: enumerate
 * the literal tails held in the hash-confirm structures
 * (src/fdr/fdr_confirm.h:36-94), find the reports that carry an exhaustion key
 * (HS_FLAG_SINGLEMATCH; REPORT_EXHAUST, src/rose/rose_program.h:485), and apply
 * the order-dependent report rules -- logical combinations included -- to a list of
 * raw match records.
 */
#ifndef HSB200_DB_WALK_H
#define HSB200_DB_WALK_H

#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../../include/hs_b200.h"
#include "../ref_layout.h"

namespace hsb {

struct LitTail {
    u64 v, msk;
    u32 size;
    u32 bucket;
};

struct MatchRec { /* == hs_b200_match_t */
    u32 id;
    u32 block;
    u64 to;
};

/* Both return false if a program holds an opcode the device does not implement
 * (callers refuse the database with HS_ARCH_ERROR instead of failing mid-scan). */
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
/* catchUp: the program belongs to a database with an outfix, where CATCH_UP only orders the outfix's
 * reports before the literal's -- which the host's ordering does -- and is accepted */
bool collectProgramReports(const u8 *bc, u32 bcLen, u32 prog, std::unordered_set<u32> *ex,
                           std::vector<ProgReport> *reports = nullptr, /* every report instruction, in program order */
                           LkeyReports *lkeys = nullptr, bool catchUp = false);

bool walkConfirm(const u8 *bc, u32 bcLen, u32 confOff, u32 nBuckets,
                 std::unordered_set<u32> *ex, std::vector<LitTail> *tails, LkeyReports *lkeys = nullptr,
                 bool catchUp = false);

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
void loadCombinations(const RoseEngine *r, Combinations *cb);

/* The bit of MatchRec.to that marks a logical-key record (id = lkey): written by SET_LOGICAL, consumed by
 * postprocessCombinations.  No match offset reaches 2^63. */
static const u64 LKEY_RECORD = 1ull << 63;
/* The bit of MatchRec.to that marks an engine's record in a database with a literal matcher and an
 * outfix: its id is a report PROGRAM offset, resolved on the host; the literal records carry report ids. */
static const u64 ENGINE_RECORD = 1ull << 62;

/** Reports compiled with HS_FLAG_SINGLEMATCH in a pure-literal database. */
hs_error_t collectExhaustible(const hs_database_t *db, std::unordered_set<u32> *ex, LkeyReports *lkeys = nullptr);

/** Order records for delivery and apply the order-dependent report rules the
 * device skipped: one report per (block, id, to) (dedupe, src/report.h:55-119)
 * and, for HS_FLAG_SINGLEMATCH reports, only the first match per block
 * (exhaustion keys, src/report.h:121-147, program_runtime.c:464-481).
 * Returns the number of records kept (in place, sorted by (block, to, id)). */
size_t postprocessRecords(const std::unordered_set<u32> &exhaustible, MatchRec *m, size_t n);

/* The same for a database with logical combinations, whose records include logical-key records:
 * the records of blocks [0, nblocks) (block i is lengths[i] bytes long) in delivery order -- by
 * (block, to), at one offset the reports by id and then the combinations it completes, by ckey --
 * with the combination reports added and the logical-key records gone. */
void postprocessCombinations(const Combinations &cb, const std::unordered_set<u32> &exhaustible,
                             std::vector<MatchRec> *v, const u32 *lengths, size_t nblocks);

} // namespace hsb
#endif
