/* db_walk.cpp -- see db_walk.h */
#include "db_walk.h"

#include <algorithm>
#include <cstring>

#include "api_internal.h"

namespace hsb {

/* Linear walk over one literal program.  A program is a sequence of blocks, each
 * ending in END or FINAL_REPORT; later blocks are reached through the fail_jump
 * of a check in an earlier one (src/rose/rose_build_program.cpp:525-829), so
 * the walk continues past a terminator while a jump target lies beyond it.
 * Returns false on an opcode the device interpreter (scan_kernels.cu
 * runProgram) does not implement -- the state-carrying ones of
 * roseRunProgram_l: PUSH_DELAYED, CATCH_UP* (CATCH_UP is accepted on request), SOM_*, TRIGGER_SUFFIX, REPORT_CHAIN,
 * REPORT_SOM*, SET_EXHAUST.  SET_LOGICAL is a report of its own here (a logical-key record
 * on the device); FLUSH_COMBINATION and SET_COMBINATION follow from it on the host. */
bool collectProgramReports(const u8 *bc, u32 bcLen, u32 prog, std::unordered_set<u32> *ex,
                           std::vector<ProgReport> *reports, LkeyReports *lkeys, bool catchUp) {
    u32 pc = prog, furthest = prog;
    u32 lastReport = INVALID_EKEY; /* the report of the current report block, for SET_LOGICAL */
    /* CHECK_BOUNDS guards the instructions up to its fail_jump target */
    struct Guard { u32 until; u64 lo, hi; };
    std::vector<Guard> guards;
    auto report = [&](u32 onmatch, s32 adjust) {
        u64 lo = 0, hi = ~0ull;
        for (const Guard &g : guards) {
            if (pc < g.until) {
                lo = std::max(lo, g.lo);
                hi = std::min(hi, g.hi);
            }
        }
        reports->push_back({onmatch, adjust, lo, hi, false});
    };
    auto jump = [&](u32 from, u32 rel) { furthest = std::max(furthest, from + rel); };
#define STEP(T) pc += (u32)HSB_ROUNDUP(sizeof(T), INSTR_ALIGN)
#define STEP_JUMP(T)                                \
    do {                                            \
        T in;                                       \
        memcpy(&in, bc + pc, sizeof(in));           \
        jump(pc, in.fail_jump);                     \
        STEP(T);                                    \
    } while (0)
    for (int guard = 0; guard < 65536; guard++) {
        if (pc + 8 > bcLen) {
            return false;
        }
        const u8 code = bc[pc];
        switch (code) {
        case OP_END:
            if (furthest <= pc) {
                return true;
            }
            STEP(InstrEnd);
            break;
        case OP_FINAL_REPORT: {
            if (reports) {
                InstrFinalReport in;
                memcpy(&in, bc + pc, sizeof(in));
                report(in.onmatch, in.offset_adjust);
            }
            if (furthest <= pc) {
                return true;
            }
            STEP(InstrFinalReport);
            break;
        }
        case OP_CHECK_GROUPS: STEP(InstrCheckGroups); break;
        case OP_CHECK_BOUNDS: {
            InstrCheckBounds in;
            memcpy(&in, bc + pc, sizeof(in));
            guards.push_back({pc + in.fail_jump, in.min_bound, in.max_bound});
            STEP_JUMP(InstrCheckBounds);
            break;
        }
        case OP_CHECK_MASK: STEP_JUMP(InstrCheckMask); break;
        case OP_CHECK_MASK_32: STEP_JUMP(InstrCheckMask32); break;
        case OP_CHECK_MASK_64: STEP_JUMP(InstrCheckMask64); break;
        case OP_CHECK_BYTE: STEP_JUMP(InstrCheckByte); break;
        case OP_CHECK_MED_LIT:
        case OP_CHECK_MED_LIT_NOCASE:
        case OP_CHECK_LONG_LIT:
        case OP_CHECK_LONG_LIT_NOCASE: STEP_JUMP(InstrCheckLit); break;
        case OP_CHECK_EXHAUSTED: STEP_JUMP(InstrCheckExhausted); break;
        case OP_DEDUPE: STEP_JUMP(InstrDedupe); break;
        case OP_REPORT: {
            InstrReport in;
            memcpy(&in, bc + pc, sizeof(in));
            lastReport = in.onmatch;
            if (reports) {
                report(in.onmatch, in.offset_adjust);
            }
            STEP(InstrReport);
            break;
        }
        case OP_REPORT_EXHAUST: {
            InstrReportExhaust in;
            memcpy(&in, bc + pc, sizeof(in));
            ex->insert(in.onmatch);
            lastReport = in.onmatch;
            if (reports) {
                report(in.onmatch, in.offset_adjust);
            }
            STEP(InstrReportExhaust);
            break;
        }
        case OP_DEDUPE_AND_REPORT: {
            InstrDedupeAndReport in;
            memcpy(&in, bc + pc, sizeof(in));
            lastReport = in.onmatch;
            if (reports) {
                report(in.onmatch, in.offset_adjust);
            }
            STEP_JUMP(InstrDedupeAndReport);
            break;
        }
        case OP_FLUSH_COMBINATION: /* starts a report block of a database with combinations */
            lastReport = INVALID_EKEY;
            STEP(InstrFlushCombination);
            break;
        case OP_SET_COMBINATION: STEP(InstrSetCombination); break;
        case OP_SET_LOGICAL: {
            InstrSetLogical in;
            memcpy(&in, bc + pc, sizeof(in));
            if (lkeys && lastReport != INVALID_EKEY) {
                (*lkeys)[in.lkey] = lastReport;
            }
            if (reports) {
                report(in.lkey, in.offset_adjust);
                reports->back().logical = true;
            }
            STEP(InstrSetLogical);
            break;
        }
        case OP_SQUASH_GROUPS: STEP(InstrSquashGroups); break;
        case OP_CLEAR_WORK_DONE: pc += INSTR_ALIGN; break;
        case OP_INCLUDED_JUMP: STEP(InstrIncludedJump); break;
        case OP_CATCH_UP:
            if (!catchUp) {
                return false;
            }
            STEP(InstrCatchUp);
            break;
        default:
            return false;
        }
    }
#undef STEP
#undef STEP_JUMP
    return false;
}

/* Walk the hash-confirm structures to enumerate literal programs
 * (src/fdr/fdr_confirm.h:36-94). */
bool walkConfirm(const u8 *bc, u32 bcLen, u32 confOff, u32 nBuckets,
                 std::unordered_set<u32> *ex, std::vector<LitTail> *tails, LkeyReports *lkeys, bool catchUp) {
    bool ok = true;
    const u8 *confBase = bc + confOff;
    for (u32 b = 0; b < nBuckets; b++) {
        u32 cf;
        memcpy(&cf, confBase + 4 * b, 4);
        if (!cf) {
            continue;
        }
        const u8 *fc = confBase + cf;
        FDRConfirm h;
        memcpy(&h, fc, sizeof(h));
        const u32 n = 1u << h.nBits;
        for (u32 c = 0; c < n; c++) {
            u32 start;
            memcpy(&start, fc + sizeof(FDRConfirm) + 4 * c, 4);
            if (!start) {
                continue;
            }
            const u8 *li = fc + start;
            for (;;) {
                LitInfo x;
                memcpy(&x, li, sizeof(x));
                ok &= collectProgramReports(bc, bcLen, x.id, ex, nullptr, lkeys, catchUp);
                tails->push_back({x.v, x.msk, x.size, b});
                if (!x.next) {
                    break;
                }
                li += sizeof(LitInfo);
            }
        }
    }
    return ok;
}

hs_error_t collectExhaustible(const hs_database_t *db, std::unordered_set<u32> *ex, LkeyReports *lkeys) {
    const DbHeader *h = (const DbHeader *)db;
    if (!h || h->magic != DB_MAGIC) {
        return HS_INVALID;
    }
    const RoseEngine *r = dbRose(db);
    const u8 *bc = (const u8 *)r;
    if (r->runtimeImpl != RUNTIME_PURE_LITERAL || !r->fmatcherOffset) {
        return HS_ARCH_ERROR;
    }
    const HWLM *hw = (const HWLM *)(bc + r->fmatcherOffset);
    const u32 engOff = r->fmatcherOffset + HWLM_ENGINE_OFFSET;
    if (hw->type == HWLM_ENGINE_NOOD) {
        NoodTable n;
        memcpy(&n, bc + engOff, sizeof(n));
        return collectProgramReports(bc, h->length, n.id, ex, nullptr, lkeys) ? HS_SUCCESS : HS_ARCH_ERROR;
    }
    FDR f;
    memcpy(&f, bc + engOff, sizeof(f));
    const u32 nb = f.engineID == 0 ? 8 : teddyNumBuckets(f.engineID);
    std::vector<LitTail> tails;
    return walkConfirm(bc, h->length, engOff + f.confOffset, nb, ex, &tails, lkeys) ? HS_SUCCESS : HS_ARCH_ERROR;
}

size_t postprocessRecords(const std::unordered_set<u32> &exhaustible, MatchRec *m, size_t n) {
    std::sort(m, m + n, [](const MatchRec &a, const MatchRec &b) {
        if (a.block != b.block) return a.block < b.block;
        if (a.to != b.to) return a.to < b.to;
        return a.id < b.id;
    });
    size_t w = 0;
    std::unordered_set<u32> seen;
    u32 curBlock = 0xffffffffu;
    const bool anyEx = !exhaustible.empty();
    for (size_t i = 0; i < n; i++) {
        if (w && m[w - 1].block == m[i].block && m[w - 1].to == m[i].to && m[w - 1].id == m[i].id) {
            continue;
        }
        if (anyEx) {
            if (m[i].block != curBlock) {
                curBlock = m[i].block;
                seen.clear();
            }
            if (exhaustible.count(m[i].id) && !seen.insert(m[i].id).second) {
                continue;
            }
        }
        m[w++] = m[i];
    }
    return w;
}

void loadCombinations(const RoseEngine *r, Combinations *cb) {
    const u8 *bc = (const u8 *)r;
    cb->lkeyCount = r->lkeyCount;
    cb->minWidth = r->minWidth;
    cb->tree.resize(r->lopCount);
    cb->combs.resize(r->ckeyCount);
    if (r->lopCount) {
        memcpy(cb->tree.data(), bc + r->logicalTreeOffset, r->lopCount * sizeof(LogicalOp));
    }
    if (r->ckeyCount) {
        memcpy(cb->combs.data(), bc + r->combInfoMapOffset, r->ckeyCount * sizeof(CombInfo));
    }
    cb->ckeysOf.assign(r->lkeyCount, {});
    for (u32 ck = 0; ck < r->ckeyCount; ck++) {
        const CombInfo &ci = cb->combs[ck];
        for (u32 i = ci.start; i <= ci.result && i - r->lkeyCount < r->lopCount; i++) {
            const LogicalOp &o = cb->tree[i - r->lkeyCount];
            for (u32 k : {o.lo, o.ro}) {
                if ((o.op != LOGICAL_OP_NOT || k == o.ro) && k < r->lkeyCount &&
                    (cb->ckeysOf[k].empty() || cb->ckeysOf[k].back() != ck)) {
                    cb->ckeysOf[k].push_back(ck);
                }
            }
        }
    }
}

namespace {

/* the per-block state of src/rose/program_runtime.c:2026-2120: logical values of lkeys and operations,
 * the combinations touched since the last flush */
struct CombState {
    const Combinations &cb;
    std::vector<u8> lvec;
    std::vector<u8> active;
    bool anyActive = false;
    explicit CombState(const Combinations &c)
        : cb(c), lvec(c.lkeyCount + c.tree.size()), active(c.combs.size()) {}

    bool inBounds(const CombInfo &ci, u64 end) const {
        return !(ci.min_offset != 0 && end < ci.min_offset) && !(ci.max_offset != MAX_OFFSET && end > ci.max_offset);
    }
    /* isLogicalCombination (src/report.h:190-223) */
    bool evaluate(const CombInfo &ci) {
        for (u32 i = ci.start; i <= ci.result; i++) {
            const LogicalOp &o = cb.tree[i - cb.lkeyCount];
            lvec[o.id] = o.op == LOGICAL_OP_NOT ? !lvec[o.ro]
                         : o.op == LOGICAL_OP_AND ? (lvec[o.lo] & lvec[o.ro])
                                                  : (lvec[o.lo] | lvec[o.ro]);
        }
        return lvec[ci.result];
    }
    /* isPurelyNegativeMatch (src/report.h:225-268): true with every sub-expression unmatched */
    bool purelyNegative(const CombInfo &ci) {
        for (u32 i = ci.start; i <= ci.result; i++) {
            const LogicalOp &o = cb.tree[i - cb.lkeyCount];
            if ((o.ro < cb.lkeyCount && lvec[o.ro]) || (o.op != LOGICAL_OP_NOT && o.lo < cb.lkeyCount && lvec[o.lo])) {
                return false;
            }
        }
        return evaluate(ci);
    }
};

} // namespace

void postprocessCombinations(const Combinations &cb, const std::unordered_set<u32> &exhaustible,
                             std::vector<MatchRec> *v, const u32 *lengths, size_t nblocks) {
    std::vector<MatchRec> &m = *v;
    std::sort(m.begin(), m.end(), [](const MatchRec &a, const MatchRec &b) {
        if (a.block != b.block) return a.block < b.block;
        const u64 ta = a.to & ~LKEY_RECORD, tb = b.to & ~LKEY_RECORD;
        if (ta != tb) return ta < tb;
        if ((a.to & LKEY_RECORD) != (b.to & LKEY_RECORD)) return (a.to & LKEY_RECORD) < (b.to & LKEY_RECORD);
        return a.id < b.id;
    });
    std::vector<MatchRec> out;
    out.reserve(m.size());
    CombState st(cb);
    std::unordered_map<u32, u64> firstAt; /* exhaustible id -> offset of its one delivered report */
    size_t i = 0;
    for (size_t blk = 0; blk < nblocks || i < m.size(); blk++) {
        const size_t b0 = i;
        while (i < m.size() && m[i].block == blk) {
            i++;
        }
        if (blk >= nblocks || lengths[blk] < cb.minWidth) {
            continue; /* not scanned (or no length given): no records to order, no end-of-data flush */
        }
        std::fill(st.lvec.begin(), st.lvec.end(), 0);
        firstAt.clear();
        u64 last = 0; /* lastCombMatchOffset */
        auto flush = [&](u64 end) {
            if (!st.anyActive) {
                return;
            }
            for (u32 ck = 0; ck < cb.combs.size(); ck++) {
                if (!st.active[ck]) {
                    continue;
                }
                const CombInfo &ci = cb.combs[ck];
                if (!st.inBounds(ci, end) || (ci.ekey != INVALID_EKEY && firstAt.count(ci.id))) {
                    continue;
                }
                if (st.evaluate(ci)) {
                    out.push_back({ci.id, (u32)blk, end});
                    if (ci.ekey != INVALID_EKEY) {
                        firstAt[ci.id] = end;
                    }
                }
            }
            std::fill(st.active.begin(), st.active.end(), 0);
            st.anyActive = false;
        };
        for (size_t k = b0; k < i; k++) {
            const MatchRec &r = m[k];
            const u64 to = r.to & ~LKEY_RECORD;
            if (to > last) {
                flush(last); /* FLUSH_COMBINATION at the first report past the last one that set an lkey */
            }
            if (!(r.to & LKEY_RECORD)) {
                if (k > b0 && m[k - 1].to == r.to && m[k - 1].id == r.id) {
                    continue; /* dedupe */
                }
                if (exhaustible.count(r.id)) {
                    if (firstAt.count(r.id)) {
                        continue;
                    }
                    firstAt[r.id] = to;
                }
                out.push_back(r);
                continue;
            }
            if (r.id >= cb.lkeyCount) {
                continue;
            }
            auto rep = cb.lkeyReport.find(r.id);
            if (rep != cb.lkeyReport.end() && exhaustible.count(rep->second)) {
                /* CHECK_EXHAUSTED skips the SET_LOGICAL of a single-match report after its first match */
                auto f = firstAt.find(rep->second);
                if (f == firstAt.end() || f->second != to) {
                    continue;
                }
            }
            st.lvec[r.id] = 1;
            for (u32 ck : cb.ckeysOf[r.id]) {
                st.active[ck] = 1;
                st.anyActive = true;
            }
            last = to;
        }
        /* LAST_FLUSH_COMBINATION at the end of the block: the active combinations, then the purely
         * negative ones at the block's end */
        flush(last);
        const u64 end = lengths[blk];
        for (u32 ck = 0; ck < cb.combs.size(); ck++) {
            const CombInfo &ci = cb.combs[ck];
            if (!st.inBounds(ci, end) || (ci.ekey != INVALID_EKEY && firstAt.count(ci.id))) {
                continue;
            }
            if (st.purelyNegative(ci)) {
                out.push_back({ci.id, (u32)blk, end});
                if (ci.ekey != INVALID_EKEY) {
                    firstAt[ci.id] = end;
                }
            }
        }
    }
    v->swap(out);
}

} // namespace hsb

extern "C" hs_error_t hs_b200_postprocess_matches(const hs_database_t *db, hs_b200_match_t *recs,
                                                  size_t n, unsigned long long *nout) {
    if (!db || (n && !recs) || !nout) {
        return HS_INVALID;
    }
    if (hsb::dbRose(db)->ckeyCount) {
        return HS_INVALID; /* combination reports need the block lengths: hs_b200_postprocess_blocks */
    }
    std::unordered_set<hsb::u32> ex;
    hs_error_t r = hsb::collectExhaustible(db, &ex);
    if (r != HS_SUCCESS) {
        return r;
    }
    static_assert(sizeof(hsb::MatchRec) == sizeof(hs_b200_match_t), "record layout");
    *nout = hsb::postprocessRecords(ex, (hsb::MatchRec *)recs, n);
    return HS_SUCCESS;
}

extern "C" hs_error_t hs_b200_postprocess_blocks(const hs_database_t *db, const hs_b200_match_t *recs, size_t n,
                                                 const unsigned int *lengths, size_t nblocks,
                                                 hs_b200_match_t *out, size_t cap, unsigned long long *nout) {
    if (!db || (n && !recs) || (nblocks && !lengths) || (cap && !out) || !nout) {
        return HS_INVALID;
    }
    const hsb::DbHeader *h = (const hsb::DbHeader *)db;
    if (h->magic != hsb::DB_MAGIC) {
        return HS_INVALID;
    }
    std::unordered_set<hsb::u32> ex;
    hsb::Combinations cb;
    hs_error_t r = hsb::collectExhaustible(db, &ex, &cb.lkeyReport);
    if (r != HS_SUCCESS) {
        return r;
    }
    std::vector<hsb::MatchRec> v((const hsb::MatchRec *)recs, (const hsb::MatchRec *)recs + n);
    if (hsb::dbRose(db)->ckeyCount) {
        hsb::loadCombinations(hsb::dbRose(db), &cb);
        hsb::postprocessCombinations(cb, ex, &v, lengths, nblocks);
    } else {
        v.resize(hsb::postprocessRecords(ex, v.data(), v.size()));
    }
    *nout = v.size();
    if (v.size() > cap) {
        return HS_INSUFFICIENT_SPACE;
    }
    if (!v.empty()) {
        memcpy(out, v.data(), v.size() * sizeof(hsb::MatchRec));
    }
    return HS_SUCCESS;
}
