/* db_walk.cpp -- see db_walk.h */
#include "db_walk.h"

#include <algorithm>
#include <cstring>

#include "api_internal.h"
#include "rose_build.h"

namespace hsb {

namespace {

/* Linear walk over one program of rr's bytecode.  A program is a sequence of blocks, each
 * ending in END or FINAL_REPORT; later blocks are reached through the fail_jump
 * of a check in an earlier one (src/rose/rose_build_program.cpp:525-829), so
 * the walk continues past a terminator while a jump target lies beyond it.
 * Returns false on an opcode the device interpreter (scan_kernels.cu
 * runProgram) does not implement -- the state-carrying ones of
 * roseRunProgram_l: PUSH_DELAYED, CATCH_UP* (CATCH_UP is accepted beside an outfix), SOM_*, TRIGGER_SUFFIX, REPORT_CHAIN,
 * REPORT_SOM*, SET_EXHAUST.  SET_LOGICAL is a report of its own here (a logical-key record
 * on the device); FLUSH_COMBINATION and SET_COMBINATION follow from it on the host.
 * Collects the exhaustible reports and the lkeys' reports into rr; reports, if given, receives
 * every report instruction, in program order. */
bool collectProgramReports(ReportRules *rr, u32 prog, std::vector<ProgReport> *reports) {
    const u8 *bc = rr->bc;
    const u32 bcLen = rr->bcLen;
    u32 pc = prog, furthest = prog;
    u32 lastReport = INVALID_EKEY; /* the report of the current report block, for SET_LOGICAL */
    /* CHECK_BOUNDS guards the instructions up to its fail_jump target */
    struct Guard { u32 until; u64 lo, hi; };
    std::vector<Guard> guards;
    auto report = [&](u32 onmatch, s32 adjust, bool logical = false) {
        if (!logical) {
            rr->reportIds.insert(onmatch);
        }
        rr->minAdjust = std::min(rr->minAdjust, adjust);
        if (!reports) {
            return;
        }
        u64 lo = 0, hi = ~0ull;
        for (const Guard &g : guards) {
            if (pc < g.until) {
                lo = std::max(lo, g.lo);
                hi = std::min(hi, g.hi);
            }
        }
        reports->push_back({onmatch, adjust, lo, hi, logical});
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
            InstrFinalReport in;
            memcpy(&in, bc + pc, sizeof(in));
            report(in.onmatch, in.offset_adjust);
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
            report(in.onmatch, in.offset_adjust);
            STEP(InstrReport);
            break;
        }
        case OP_REPORT_EXHAUST: {
            InstrReportExhaust in;
            memcpy(&in, bc + pc, sizeof(in));
            rr->exhaustible.insert(in.onmatch);
            lastReport = in.onmatch;
            report(in.onmatch, in.offset_adjust);
            STEP(InstrReportExhaust);
            break;
        }
        case OP_DEDUPE_AND_REPORT: {
            InstrDedupeAndReport in;
            memcpy(&in, bc + pc, sizeof(in));
            lastReport = in.onmatch;
            report(in.onmatch, in.offset_adjust);
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
            if (lastReport != INVALID_EKEY) {
                rr->comb.lkeyReport[in.lkey] = lastReport;
            }
            report(in.lkey, in.offset_adjust, true);
            STEP(InstrSetLogical);
            break;
        }
        case OP_SQUASH_GROUPS: STEP(InstrSquashGroups); break;
        case OP_CLEAR_WORK_DONE: pc += INSTR_ALIGN; break;
        case OP_INCLUDED_JUMP: STEP(InstrIncludedJump); break;
        case OP_CATCH_UP:
            /* beside an outfix, CATCH_UP only orders the outfix's reports before the literal's -- which the
             * host's ordering does */
            if (rr->shape != SHAPE_LITERALS_OUTFIX) {
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
bool walkConfirm(ReportRules *rr, u32 confOff, u32 nBuckets, std::vector<LitTail> *tails) {
    bool ok = true;
    const u8 *confBase = rr->bc + confOff;
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
                ok &= collectProgramReports(rr, x.id, nullptr);
                if (tails) {
                    tails->push_back({x.v, x.msk, x.size, b});
                }
                if (!x.next) {
                    break;
                }
                li += sizeof(LitInfo);
            }
        }
    }
    return ok;
}

/* Order records for delivery and apply dedupe and exhaustion (ReportRules::deliver).  Returns the number
 * of records kept (in place, sorted by (block, to, id)). */
size_t postprocessRecords(const std::unordered_set<u32> &exhaustible, DevMatch *m, size_t n) {
    std::sort(m, m + n, RecordOrder());
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

/* The rules for a database with logical combinations, whose records include logical-key records: the
 * records of blocks [0, nblocks) (block i is lengths[i] bytes long) in delivery order -- by (block, to),
 * at one offset the reports by id and then the combinations it completes, by ckey -- with the
 * combination reports added and the logical-key records gone. */
void postprocessCombinations(const Combinations &cb, const std::unordered_set<u32> &exhaustible,
                             std::vector<DevMatch> *v, const u32 *lengths, size_t nblocks) {
    std::vector<DevMatch> &m = *v;
    std::sort(m.begin(), m.end(), [](const DevMatch &a, const DevMatch &b) {
        if (a.block != b.block) return a.block < b.block;
        const u64 ta = a.to & ~LKEY_RECORD, tb = b.to & ~LKEY_RECORD;
        if (ta != tb) return ta < tb;
        if ((a.to & LKEY_RECORD) != (b.to & LKEY_RECORD)) return (a.to & LKEY_RECORD) < (b.to & LKEY_RECORD);
        return a.id < b.id;
    });
    std::vector<DevMatch> out;
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
            const DevMatch &r = m[k];
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

} // namespace

namespace {

/* units[i] at bytes [off, off + count * sizeof(Unit)) of the bytecode, field by field */
template <class Unit>
bool unitsAre(const u8 *bc, u32 len, u32 off, u32 count, const std::vector<Unit> &units) {
    if (count != units.size()) {
        return false;
    }
    if (!count) {
        return true;
    }
    if (off % alignof(Unit) || (u64)off + (u64)count * sizeof(Unit) > len) {
        return false;
    }
    for (u32 i = 0; i < count; i++) {
        Unit u;
        memcpy(&u, bc + off + (size_t)i * sizeof(Unit), sizeof(u));
        if (u.offset != units[i].offset || u.val != units[i].val) {
            return false;
        }
    }
    return true;
}

/* The tables that run a set of K = queueCount outfixes, checked against K and the bytecode length `len`: the
 * NfaInfo table and every engine lie inside the bytecode, the engines' states tile the state and scratch areas in
 * queue order up to their sizes, the active leaf array has K bits and the state scatter
 * plan is its clear plan, and the EOD program is there exactly when some engine accepts at end of data, its
 * sparse iterator over exactly those queues.  (The runtime walks these with no bound of its own.) */
bool outfixTablesFit(const RoseEngine *r, u32 len) {
    const u8 *bc = (const u8 *)r;
    const u32 k = r->queueCount;
    if (r->nfaInfoOffset % 4 || (u64)r->nfaInfoOffset + (u64)k * sizeof(NfaInfo) > len) {
        return false;
    }
    const StateOffsets &so = r->stateOffsets;
    std::vector<u32> eod;
    u64 state = so.nfaStateBegin, full = 0; /* each queue's stream and scratch state follow the one before */
    for (u32 q = 0; q < k; q++) {
        NfaInfo ni;
        memcpy(&ni, bc + r->nfaInfoOffset + (size_t)q * sizeof(NfaInfo), sizeof(ni));
        if (ni.nfaOffset % 64 || (u64)ni.nfaOffset + sizeof(NFA) > len) {
            return false;
        }
        NFA nh;
        memcpy(&nh, bc + ni.nfaOffset, sizeof(nh));
        if ((u64)ni.nfaOffset + nh.length > len || ni.stateOffset != state || ni.fullStateOffset != full) {
            return false;
        }
        if (nh.flags & NFA_ACCEPTS_EOD) {
            eod.push_back(q);
        }
        state += nh.streamStateSize;
        full = HSB_ROUNDUP(full + nh.scratchStateSize, 64);
    }
    if (state != r->stateSize || full != r->scratchStateSize) {
        return false;
    }
    if (so.activeLeafArray_size != mmbitSize(k) || (u64)so.activeLeafArray + so.activeLeafArray_size > r->stateSize) {
        return false;
    }
    const MmbClearPlan p = mmbClearPlan(k, so.activeLeafArray);
    const ScatterPlan &sp = r->state_init;
    if (!unitsAre(bc, len, sp.s_u64a_offset, sp.s_u64a_count, p.u64s) ||
        !unitsAre(bc, len, sp.s_u32_offset, sp.s_u32_count, p.u32s) ||
        !unitsAre(bc, len, sp.s_u16_offset, sp.s_u16_count, p.u16s) ||
        !unitsAre(bc, len, sp.s_u8_offset, sp.s_u8_count, p.u8s)) {
        return false;
    }
    if (!r->eodProgramOffset || eod.empty()) {
        return !r->eodProgramOffset && eod.empty();
    }
    InstrEnginesEod ee; /* (inside the bytecode: dbShape) */
    memcpy(&ee, bc + r->eodProgramOffset, sizeof(ee));
    const std::vector<MmbSparseIter> want = mmbSparseIterator(eod, k);
    if (ee.iter_offset % alignof(MmbSparseIter) || (u64)ee.iter_offset + want.size() * sizeof(MmbSparseIter) > len) {
        return false;
    }
    for (size_t i = 0; i < want.size(); i++) {
        MmbSparseIter it;
        memcpy(&it, bc + ee.iter_offset + i * sizeof(MmbSparseIter), sizeof(it));
        if (it.mask != want[i].mask || it.val != want[i].val) {
            return false;
        }
    }
    return true;
}

} // namespace

DbShape dbShape(const hs_database_t *db) {
    const DbHeader *h = (const DbHeader *)db;
    const RoseEngine *r = dbRose(db);
    const u8 *bc = (const u8 *)r;
    if (r->runtimeImpl == RUNTIME_PURE_LITERAL && r->fmatcherOffset) {
        return SHAPE_PURE_LITERAL;
    }
    if (r->runtimeImpl == RUNTIME_SINGLE_OUTFIX && r->mode == MODE_BLOCK && r->queueCount == 1 &&
        r->outfixBeginQueue == 0 && r->outfixEndQueue == 1 && r->nfaInfoOffset && !r->amatcherOffset &&
        !r->ematcherOffset && !r->fmatcherOffset && !r->hasSom) {
        return SHAPE_SOLE_OUTFIX;
    }
    /* the FULL_ROSE shapes run here: outfixes on queues [0, K) only, beside the floating literal matcher,
     * whose role-less programs report directly (one outfix, DESIGN.md section 10d), or alone (any K, section
     * 10e) -- no anchored, EOD or small-block matcher, no roles, leftfixes, suffixes, delayed literals, MPV, SOM
     * or long-literal table, and an EOD program that at most checks the engines' EOD accepts */
    const u32 k = r->queueCount;
    if (r->runtimeImpl == RUNTIME_FULL_ROSE && r->mode == MODE_BLOCK && (!r->fmatcherOffset || k == 1) &&
        !r->amatcherOffset && !r->ematcherOffset && !r->sbmatcherOffset && !r->drmatcherOffset && k >= 1 &&
        r->activeArrayCount == k && r->outfixBeginQueue == 0 && r->outfixEndQueue == k &&
        r->leftfixBeginQueue == k && r->nfaInfoOffset && !r->activeLeftCount && !r->rosePrefixCount &&
        !r->rolesWithStateCount && !r->delay_count && !r->anchored_count && r->initMpvNfa == MO_INVALID_IDX &&
        !r->hasSom && !r->longLitTableOffset && !r->ckeyCount && !r->eagerIterOffset && !r->delayProgramOffset &&
        !r->anchoredProgramOffset && !r->boundary.reportEodOffset && !r->boundary.reportZeroOffset &&
        !r->boundary.reportZeroEodOffset && !r->lastByteHistoryIterOffset &&
        (!r->eodProgramOffset ||
         ((size_t)r->eodProgramOffset + 16 <= h->length && r->eodProgramOffset % INSTR_ALIGN == 0 &&
          bc[r->eodProgramOffset] == OP_ENGINES_EOD &&
          bc[r->eodProgramOffset + HSB_ROUNDUP(sizeof(InstrEnginesEod), INSTR_ALIGN)] == OP_END))) {
        if (r->fmatcherOffset) {
            return SHAPE_LITERALS_OUTFIX;
        }
        return outfixTablesFit(r, h->length) ? SHAPE_OUTFIXES : SHAPE_MALFORMED;
    }
    return SHAPE_UNSUPPORTED;
}

hs_error_t loadReportRules(const hs_database_t *db, ReportRules *rules, std::vector<LitTail> *tails) {
    const RoseEngine *r = dbRose(db);
    rules->shape = dbShape(db);
    if (rules->shape == SHAPE_UNSUPPORTED || rules->shape == SHAPE_MALFORMED) {
        return rules->shape == SHAPE_MALFORMED ? HS_INVALID : HS_ARCH_ERROR;
    }
    rules->bc = (const u8 *)r;
    rules->bcLen = ((const DbHeader *)db)->length;
    rules->hasDedupe = r->dkeyCount != 0;
    if (r->ckeyCount) {
        loadCombinations(r, &rules->comb);
    }
    if (rules->shape == SHAPE_SOLE_OUTFIX || rules->shape == SHAPE_OUTFIXES) {
        return HS_SUCCESS; /* no literal programs: the engines' are walked as their records are delivered */
    }
    const HWLM *hw = (const HWLM *)(rules->bc + r->fmatcherOffset);
    const u32 engOff = r->fmatcherOffset + HWLM_ENGINE_OFFSET;
    bool ok;
    if (hw->type == HWLM_ENGINE_NOOD) {
        NoodTable n;
        memcpy(&n, rules->bc + engOff, sizeof(n));
        ok = collectProgramReports(rules, n.id, nullptr);
    } else if (hw->type == HWLM_ENGINE_FDR) {
        FDR f;
        memcpy(&f, rules->bc + engOff, sizeof(f));
        if (f.engineID != 0 && !teddyIdValid(f.engineID)) {
            return HS_INVALID;
        }
        ok = walkConfirm(rules, engOff + f.confOffset, f.engineID == 0 ? 8 : teddyNumBuckets(f.engineID), tails);
    } else {
        return HS_INVALID;
    }
    return ok ? HS_SUCCESS : HS_ARCH_ERROR;
}

namespace {

/* The report program offsets an engine can raise (its reports were remapped to programs at build time):
 * McClellan / Sheng -- the single report, or the accept and EOD-accept report lists of every state's aux
 * record (struct report_list {count; reports[]}); LimEx -- the accept and EOD-accept tables (NFAAccept) and
 * the exceptions' report lists (MO_INVALID_IDX-terminated).  Offsets are relative to struct NFA (DFAs) or
 * to the LimEx structure that follows it.  False on a table that runs past the engine. */
struct EngineWalk {
    const u8 *nfa;
    u32 len;
    std::vector<u32> *out;
    bool ok = true;
    u32 at(u64 off) {
        u32 v = 0;
        if (off + 4 > len) {
            ok = false;
        } else {
            memcpy(&v, nfa + off, 4);
        }
        return v;
    }
    void countedList(u32 off) { /* struct report_list */
        const u32 n = at(off);
        for (u32 i = 0; i < n && ok; i++) {
            out->push_back(at((u64)off + 4 + 4 * (u64)i));
        }
    }
    void terminatedList(u64 off) {
        for (u32 i = 0; ok; i++) {
            const u32 id = at(off + 4 * (u64)i);
            if (id == MO_INVALID_IDX) {
                break;
            }
            out->push_back(id);
        }
    }
    void dfaAux(u32 auxOff, u32 auxSize, u32 states) {
        for (u32 s = 0; s < states && ok; s++) {
            const u64 a = (u64)auxOff + (u64)s * auxSize;
            for (u32 list : {at(a), at(a + 4)}) { /* accept, accept_eod */
                if (list) {
                    countedList(list);
                }
            }
        }
    }
    template <class Nfa, class Exc> void limex() {
        const u64 base = sizeof(NFA);
        if (base + sizeof(Nfa) > len) {
            ok = false;
            return;
        }
        Nfa lx;
        memcpy(&lx, nfa + base, sizeof(lx));
        for (auto t : {std::make_pair(lx.acceptOffset, lx.acceptCount), std::make_pair(lx.acceptEodOffset, lx.acceptEodCount)}) {
            for (u32 i = 0; i < t.second && ok; i++) {
                const u64 a = base + t.first + (u64)i * sizeof(NFAAccept);
                if (a + sizeof(NFAAccept) > len) {
                    ok = false;
                    break;
                }
                NFAAccept acc;
                memcpy(&acc, nfa + a, sizeof(acc));
                if (acc.single_report) {
                    out->push_back(acc.reports);
                } else {
                    terminatedList(base + acc.reports);
                }
            }
        }
        for (u32 i = 0; i < lx.exceptionCount && ok; i++) {
            const u64 x = base + lx.exceptionOffset + (u64)i * sizeof(Exc);
            if (x + sizeof(Exc) > len) {
                ok = false;
                break;
            }
            Exc e;
            memcpy(&e, nfa + x, sizeof(e));
            if (e.reports != MO_INVALID_IDX) {
                terminatedList(base + e.reports);
            }
        }
    }
};

bool enginePrograms(const u8 *nfa, u32 len, std::vector<u32> *out) {
    EngineWalk w{nfa, len, out};
    if (len < sizeof(NFA)) {
        return false;
    }
    NFA h;
    memcpy(&h, nfa, sizeof(h));
    switch (h.type) {
    case NFA_MCCLELLAN_8:
    case NFA_MCCLELLAN_16: {
        if (sizeof(NFA) + sizeof(McClellan) > len) {
            return false;
        }
        McClellan m;
        memcpy(&m, nfa + sizeof(NFA), sizeof(m));
        if (m.flags & MCCLELLAN_FLAG_SINGLE) {
            out->push_back(m.arb_report);
        } else {
            w.dfaAux(m.aux_offset, sizeof(MStateAux), m.state_count);
        }
        break;
    }
    case NFA_SHENG: {
        if (sizeof(NFA) + sizeof(Sheng) > len) {
            return false;
        }
        Sheng s;
        memcpy(&s, nfa + sizeof(NFA), sizeof(s));
        if (s.flags & SHENG_FLAG_SINGLE_REPORT) {
            out->push_back(s.report);
        } else {
            w.dfaAux(s.aux_offset, sizeof(SstateAux), s.n_states);
        }
        break;
    }
    case NFA_LIMEX_32: w.limex<LimExNFA32, NFAException32>(); break;
    case NFA_LIMEX_64: w.limex<LimExNFA64, NFAException64>(); break;
    case NFA_LIMEX_128: w.limex<LimExNFA128, NFAException128>(); break;
    case NFA_LIMEX_256: w.limex<LimExNFA256, NFAException256>(); break;
    case NFA_LIMEX_512: w.limex<LimExNFA512, NFAException512>(); break;
    default: return false;
    }
    return w.ok;
}

} // namespace

bool outfixEngines(const hs_database_t *db, std::vector<EngineBytes> *out) {
    const DbHeader *h = (const DbHeader *)db;
    const RoseEngine *r = dbRose(db);
    const u8 *bc = (const u8 *)r;
    const u32 k = r->queueCount;
    out->clear();
    if ((size_t)r->nfaInfoOffset + (size_t)k * sizeof(NfaInfo) > h->length) {
        return false;
    }
    for (u32 q = 0; q < k; q++) {
        NfaInfo ni;
        memcpy(&ni, bc + r->nfaInfoOffset + q * sizeof(NfaInfo), sizeof(ni));
        if (ni.nfaOffset % 64 || (size_t)ni.nfaOffset + sizeof(NFA) > h->length) {
            return false;
        }
        NFA nh;
        memcpy(&nh, bc + ni.nfaOffset, sizeof(nh));
        if ((size_t)ni.nfaOffset + nh.length > h->length) {
            return false;
        }
        out->push_back({bc + ni.nfaOffset, nh.length});
    }
    return true;
}

hs_error_t buildDeviceRules(ReportRules *rules, const std::vector<EngineBytes> &engines, DeviceRules *out) {
    *out = DeviceRules();
    if (!engines.empty()) {
        std::vector<u32> progs; /* (the engines' reports are offsets into one bytecode: one table serves all) */
        for (const EngineBytes &e : engines) {
            if (!enginePrograms(e.nfa, e.len, &progs)) {
                return HS_INVALID;
            }
        }
        std::sort(progs.begin(), progs.end());
        progs.erase(std::unique(progs.begin(), progs.end()), progs.end());
        out->progStart.push_back(0);
        for (u32 prog : progs) {
            auto it = rules->progReports.find(prog);
            if (it == rules->progReports.end()) {
                std::vector<ProgReport> reps;
                if (prog % INSTR_ALIGN || prog < sizeof(RoseEngine) || prog >= rules->bcLen ||
                    !collectProgramReports(rules, prog, &reps)) {
                    return HS_UNKNOWN_ERROR; /* as ReportRules::deliver would answer a record of it */
                }
                it = rules->progReports.emplace(prog, std::move(reps)).first;
            }
            out->progOff.push_back(prog);
            out->reps.insert(out->reps.end(), it->second.begin(), it->second.end());
            out->progStart.push_back((u32)out->reps.size());
            out->maxFanout = std::max<u32>(out->maxFanout, (u32)it->second.size());
            for (const ProgReport &rp : it->second) {
                out->maxAdjust = std::max<s32>(out->maxAdjust, rp.offset_adjust);
            }
        }
    }
    out->ids.assign(rules->reportIds.begin(), rules->reportIds.end());
    for (u32 id : out->ids) {
        out->idExhaustible.push_back(rules->exhaustible.count(id) ? 1 : 0);
    }
    return HS_SUCCESS;
}

hs_error_t ReportRules::deliver(std::vector<DevMatch> *v, const u32 *lengths, size_t nblocks) {
    if (comb.any() && !lengths && nblocks) {
        return HS_INVALID;
    }
    if (shape != SHAPE_PURE_LITERAL) {
        std::vector<DevMatch> out;
        out.reserve(v->size());
        for (DevMatch m : *v) {
            if (shape == SHAPE_LITERALS_OUTFIX) {
                if (!(m.to & ENGINE_RECORD)) {
                    out.push_back(m); /* a literal's record */
                    continue;
                }
                m.to &= ~ENGINE_RECORD;
            }
            if (m.id == 0xffffffffu) {
                continue; /* a slot some lane reserved and did not fill */
            }
            auto it = progReports.find(m.id);
            if (it == progReports.end()) {
                std::vector<ProgReport> reps;
                if (m.id % INSTR_ALIGN || m.id < sizeof(RoseEngine) || m.id >= bcLen ||
                    !collectProgramReports(this, m.id, &reps)) {
                    return HS_UNKNOWN_ERROR; /* a program with a state-carrying opcode (or a corrupt record) */
                }
                it = progReports.emplace(m.id, std::move(reps)).first;
            }
            for (const ProgReport &rp : it->second) {
                if (m.to < rp.min_bound || m.to > rp.max_bound) {
                    continue; /* CHECK_BOUNDS (hs_expr_ext min_offset / max_offset) */
                }
                DevMatch o = m;
                o.id = rp.onmatch;
                o.to = (u64)((long long)m.to + rp.offset_adjust) | (rp.logical ? LKEY_RECORD : 0);
                out.push_back(o);
            }
        }
        v->swap(out);
    }
    if (comb.any()) {
        postprocessCombinations(comb, exhaustible, v, lengths, nblocks);
    } else {
        v->resize(postprocessRecords(exhaustible, v->data(), v->size()));
    }
    return HS_SUCCESS;
}

} // namespace hsb

extern "C" hs_error_t hs_b200_report_ids(const hs_database_t *db, unsigned int *ids, size_t cap, size_t *count) {
    if (!db || !count || (cap && !ids)) {
        return HS_INVALID;
    }
    const hsb::DbHeader *h = (const hsb::DbHeader *)db;
    if (h->magic != hsb::DB_MAGIC) {
        return HS_INVALID;
    }
    hsb::ReportRules rules;
    hs_error_t r = hsb::loadReportRules(db, &rules);
    if (r != HS_SUCCESS) {
        return r;
    }
    std::vector<hsb::EngineBytes> engines;
    if (rules.shape != hsb::SHAPE_PURE_LITERAL && !hsb::outfixEngines(db, &engines)) {
        return HS_INVALID;
    }
    hsb::DeviceRules dr;
    r = hsb::buildDeviceRules(&rules, engines, &dr);
    if (r != HS_SUCCESS) {
        return r;
    }
    /* the combinations' own reports, which the host adds when it orders the records */
    std::set<unsigned int> all(dr.ids.begin(), dr.ids.end());
    for (const hsb::CombInfo &ci : rules.comb.combs) {
        all.insert(ci.id);
    }
    *count = all.size();
    if (!ids) {
        return HS_SUCCESS;
    }
    if (cap < all.size()) {
        return HS_INSUFFICIENT_SPACE;
    }
    std::copy(all.begin(), all.end(), ids);
    return HS_SUCCESS;
}

extern "C" hs_error_t hs_b200_postprocess_matches(const hs_database_t *db, hs_b200_match_t *recs,
                                                  size_t n, unsigned long long *nout) {
    if (!db || (n && !recs) || !nout) {
        return HS_INVALID;
    }
    if (hsb::dbRose(db)->ckeyCount) {
        return HS_INVALID; /* combination reports need the block lengths: hs_b200_postprocess_blocks */
    }
    /* without combinations no record is added: the result fits where the records were */
    return hs_b200_postprocess_blocks(db, recs, n, nullptr, 0, recs, n, nout);
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
    hsb::ReportRules rules;
    hs_error_t r = hsb::loadReportRules(db, &rules);
    if (r != HS_SUCCESS) {
        return r;
    }
    if (rules.shape != hsb::SHAPE_PURE_LITERAL) {
        return HS_ARCH_ERROR; /* engine records are resolved by the scan entry points only */
    }
    std::vector<hsb::DevMatch> v((const hsb::DevMatch *)recs, (const hsb::DevMatch *)recs + n);
    r = rules.deliver(&v, lengths, nblocks);
    if (r != HS_SUCCESS) {
        return r;
    }
    *nout = v.size();
    if (v.size() > cap) {
        return HS_INSUFFICIENT_SPACE;
    }
    if (!v.empty()) {
        memcpy(out, v.data(), v.size() * sizeof(hsb::DevMatch));
    }
    return HS_SUCCESS;
}
