/*
 * rose_build.cpp -- assembles the RoseEngine bytecode of a pure-literal
 * database: one role program per literal fragment, the dedupe-key table and
 * the floating HWLM table, behind a RoseEngine header whose fields are set the
 * way the reference's back end sets them for ROSE_RUNTIME_PURE_LITERAL
 * databases (src/rose/rose_build_bytecode.cpp:259-305 isPureFloating,
 * :382-465 fillStateOffsets, :3609-3888 buildFinalEngine).
 *
 * Program shapes follow src/rose/rose_build_program.cpp:525-710 (makeReport)
 * and :780-829 (makeCheckLiteralInstruction):
 *
 *   per pattern P of the fragment            (fail_jump -> next pattern / END)
 *     |P| > 8            CHECK_MED_LIT[_NOCASE]  lit bytes live in the blob
 *     SINGLEMATCH        CHECK_EXHAUSTED, [DEDUPE,] REPORT_EXHAUST
 *     shared report id   DEDUPE_AND_REPORT
 *     otherwise          REPORT
 *   END
 * (beside an outfix, CATCH_UP before each report block: buildMixedRose)
 *
 * Literals longer than 8 bytes reach the literal matcher as their 8-byte
 * suffix (src/rose/rose_build_matchers.cpp:717-720); patterns with equal
 * suffix/case share one HWLM literal ("fragment") whose id is the byte offset
 * of its program in the bytecode (src/rose/match.c:238).
 */
#include "rose_build.h"
#include "dfa_build.h"
#include "limex_build.h"
#include "regex_nfa.h"
#include "../../../include/hs_b200.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <tuple>
#include <set>
#include <type_traits>
#include <stdexcept>

namespace hsb {

/* mmbit_keyshift (src/util/multibit.h:182-186): the shift of the root level's keys, the least multiple of 6 with
 * 64 << ks >= totalBits */
static u32 mmbKeyShift(u32 totalBits) {
    u32 ks = 0;
    while ((64ull << ks) < totalBits) {
        ks += 6;
    }
    return ks;
}

std::vector<MmbSparseIter> mmbSparseIterator(const std::vector<u32> &keys, u32 totalBits) {
    /* level by level from the root, the records of the nodes that hold a key in key order (the breadth-first
     * layout); a node at shift s is key >> (s + 6), its bit (key >> s) & 63 */
    std::vector<std::vector<MmbSparseIter>> levels;
    for (s32 s = (s32)mmbKeyShift(totalBits); s >= 0; s -= 6) {
        std::vector<MmbSparseIter> lv;
        u64 node = 0;
        for (u32 key : keys) {
            if (lv.empty() || (u64)key >> (s + 6) != node) {
                node = (u64)key >> (s + 6);
                MmbSparseIter rec;
                memset(&rec, 0, sizeof(rec));
                lv.push_back(rec);
            }
            lv.back().mask |= 1ull << ((key >> s) & 63);
        }
        levels.push_back(lv);
    }
    /* val: above the last level, where the record's children start (the next level's start plus the keys of the
     * records before it on its level); on the last level, the keys of the records before it there */
    std::vector<MmbSparseIter> out;
    u32 next = 0;
    for (size_t l = 0; l < levels.size(); l++) {
        next += (u32)levels[l].size();
        u32 before = l + 1 < levels.size() ? next : 0;
        for (MmbSparseIter &rec : levels[l]) {
            rec.val = before;
            before += (u32)__builtin_popcountll(rec.mask);
            out.push_back(rec);
        }
    }
    return out;
}

MmbClearPlan mmbClearPlan(u32 totalBits, u32 at) {
    MmbClearPlan p;
    auto unit = [](auto *v, u32 offset) {
        typename std::remove_reference<decltype(*v)>::type::value_type u;
        memset(&u, 0, sizeof(u));
        u.offset = offset;
        v->push_back(u);
    };
    if (totalBits > 256) {
        unit(&p.u64s, at); /* the tree: clearing its root clears it */
        return p;
    }
    u32 bits = totalBits;
    for (; bits > 64; bits -= 64, at += 8) {
        unit(&p.u64s, at);
    }
    /* the last word of 1-64 bits */
    if (bits > 56) {
        unit(&p.u64s, at);
        return p;
    }
    if (bits > 24) {
        unit(&p.u32s, at);
    }
    if ((bits > 8 && bits <= 24) || bits > 40) {
        unit(&p.u16s, bits > 24 ? at + 4 : at);
    }
    if (bits <= 8 || (bits > 16 && bits <= 24) || (bits > 32 && bits <= 40) || bits > 48) {
        unit(&p.u8s, bits <= 8 ? at : bits <= 24 ? at + 2 : bits <= 40 ? at + 4 : at + 6);
    }
    return p;
}

namespace {

struct Blob {
    std::vector<u8> bytes; /* starts at RoseEngine offset `base` */
    u32 base;
    explicit Blob(u32 b) : base(b) {}
    u32 reserve(size_t len, size_t align) {
        size_t pos = HSB_ROUNDUP(base + bytes.size(), align);
        bytes.resize(pos - base + len, 0);
        return (u32)pos;
    }
    u32 add(const void *p, size_t len, size_t align) {
        u32 off = reserve(len, align);
        memcpy(bytes.data() + (off - base), p, len);
        return off;
    }
    u8 *at(u32 off) { return bytes.data() + (off - base); }
};

template <class T> u32 instrSize() { return (u32)HSB_ROUNDUP(sizeof(T), INSTR_ALIGN); }

struct PatInfo {
    const LitPattern *p;
    std::string folded; /* upper-cased if caseless */
    bool anyAlpha;
    u32 ekey, dkey;
};

/* Combination bookkeeping of a report block (makeReport, src/rose/rose_build_program.cpp:568-626): when
 * the database has combinations, FLUSH_COMBINATION before the report; when the report's id is a
 * sub-expression of one, SET_LOGICAL and one SET_COMBINATION per combination that names it after it. */
u32 flushSize(const LogicalSet *ls) { return ls && !ls->empty() ? instrSize<InstrFlushCombination>() : 0; }

u32 logicalSize(const LogicalSet *ls, u32 report) {
    const u32 lk = ls ? ls->lkey(report) : INVALID_LKEY;
    if (lk == INVALID_LKEY) {
        return 0;
    }
    return instrSize<InstrSetLogical>() + (u32)ls->ckeysOfLkey.at(lk).size() * instrSize<InstrSetCombination>();
}

u32 writeFlush(Blob &blob, u32 pc, const LogicalSet *ls) {
    if (flushSize(ls)) {
        InstrFlushCombination f;
        f.code = OP_FLUSH_COMBINATION;
        memcpy(blob.at(pc), &f, sizeof(f));
        pc += instrSize<InstrFlushCombination>();
    }
    return pc;
}

u32 writeLogical(Blob &blob, u32 pc, const LogicalSet *ls, u32 report, s32 adjust) {
    const u32 lk = ls ? ls->lkey(report) : INVALID_LKEY;
    if (lk == INVALID_LKEY) {
        return pc;
    }
    InstrSetLogical sl;
    memset(&sl, 0, sizeof(sl));
    sl.code = OP_SET_LOGICAL;
    sl.lkey = lk;
    sl.offset_adjust = adjust;
    memcpy(blob.at(pc), &sl, sizeof(sl));
    pc += instrSize<InstrSetLogical>();
    for (u32 ck : ls->ckeysOfLkey.at(lk)) {
        InstrSetCombination sc;
        memset(&sc, 0, sizeof(sc));
        sc.code = OP_SET_COMBINATION;
        sc.ckey = ck;
        memcpy(blob.at(pc), &sc, sizeof(sc));
        pc += instrSize<InstrSetCombination>();
    }
    return pc;
}

/* the report block of one pattern, without its literal check */
u32 reportSize(const PatInfo &pi, const LogicalSet *ls) {
    u32 sz = flushSize(ls) + logicalSize(ls, pi.p->report);
    if (pi.ekey != INVALID_EKEY) {
        sz += instrSize<InstrCheckExhausted>();
        if (pi.dkey != INVALID_DKEY) {
            sz += instrSize<InstrDedupe>();
        }
        sz += instrSize<InstrReportExhaust>();
    } else if (pi.dkey != INVALID_DKEY) {
        sz += pi.p->quiet ? instrSize<InstrDedupe>() : instrSize<InstrDedupeAndReport>();
    } else if (!pi.p->quiet) {
        sz += instrSize<InstrReport>();
    }
    return sz;
}

u32 blockSize(const PatInfo &pi, const LogicalSet *ls) {
    return (pi.p->s.size() > 8 ? instrSize<InstrCheckLit>() : 0) + reportSize(pi, ls);
}

/* Write the report block of pattern pi at pc; a failed check jumps to `failTo`. */
void writeReport(Blob &blob, u32 pc, const PatInfo &pi, u32 failTo, const LogicalSet *ls) {
    const u32 report = pi.p->report;
    if (pi.ekey != INVALID_EKEY) {
        InstrCheckExhausted ce;
        memset(&ce, 0, sizeof(ce));
        ce.code = OP_CHECK_EXHAUSTED;
        ce.ekey = pi.ekey;
        ce.fail_jump = failTo - pc;
        memcpy(blob.at(pc), &ce, sizeof(ce));
        pc += instrSize<InstrCheckExhausted>();
        pc = writeFlush(blob, pc, ls);
        if (pi.dkey != INVALID_DKEY) {
            InstrDedupe d;
            memset(&d, 0, sizeof(d));
            d.code = OP_DEDUPE;
            d.dkey = pi.dkey;
            d.fail_jump = failTo - pc;
            memcpy(blob.at(pc), &d, sizeof(d));
            pc += instrSize<InstrDedupe>();
        }
        InstrReportExhaust re;
        memset(&re, 0, sizeof(re));
        re.code = OP_REPORT_EXHAUST;
        re.onmatch = report;
        re.ekey = pi.ekey;
        memcpy(blob.at(pc), &re, sizeof(re));
        pc += instrSize<InstrReportExhaust>();
    } else if (pi.dkey != INVALID_DKEY) {
        pc = writeFlush(blob, pc, ls);
        if (pi.p->quiet) {
            InstrDedupe d;
            memset(&d, 0, sizeof(d));
            d.code = OP_DEDUPE;
            d.dkey = pi.dkey;
            d.fail_jump = failTo - pc;
            memcpy(blob.at(pc), &d, sizeof(d));
            pc += instrSize<InstrDedupe>();
        } else {
            InstrDedupeAndReport dr;
            memset(&dr, 0, sizeof(dr));
            dr.code = OP_DEDUPE_AND_REPORT;
            dr.dkey = pi.dkey;
            dr.onmatch = report;
            dr.fail_jump = failTo - pc;
            memcpy(blob.at(pc), &dr, sizeof(dr));
            pc += instrSize<InstrDedupeAndReport>();
        }
    } else {
        pc = writeFlush(blob, pc, ls);
        if (!pi.p->quiet) {
            InstrReport r;
            memset(&r, 0, sizeof(r));
            r.code = OP_REPORT;
            r.onmatch = report;
            memcpy(blob.at(pc), &r, sizeof(r));
            pc += instrSize<InstrReport>();
        }
    }
    writeLogical(blob, pc, ls, report, 0);
}

/* The combination tables (src/rose/rose_build_bytecode.cpp:2497-2506 writeLogicalInfo) and the
 * LAST_FLUSH_COMBINATION program run at the end of a block (:3362-3369), added to the blob. */
void writeLogicalInfo(Blob &blob, const LogicalSet *ls, RoseEngine *r) {
    if (!ls || ls->empty()) {
        return;
    }
    if (!ls->tree.empty()) {
        r->logicalTreeOffset = blob.add(ls->tree.data(), ls->tree.size() * sizeof(LogicalOp), alignof(LogicalOp));
    }
    r->combInfoMapOffset = blob.add(ls->combs.data(), ls->combs.size() * sizeof(CombInfo), alignof(CombInfo));
    r->lkeyCount = (u32)ls->lkeyOf.size();
    r->lopCount = (u32)ls->tree.size();
    r->ckeyCount = (u32)ls->combs.size();
    const u32 prog = blob.reserve(instrSize<InstrLastFlushCombination>() + instrSize<InstrEnd>(), INSTR_ALIGN);
    *blob.at(prog) = OP_LAST_FLUSH_COMBINATION;
    *blob.at(prog + instrSize<InstrLastFlushCombination>()) = OP_END;
    r->lastFlushCombProgramOffset = prog;
}

/* A combination with HS_FLAG_SINGLEMATCH takes the exhaustion key of its id (compiler.cpp:297-299
 * getExhaustibleKey), after those of the expressions. */
void assignCombinationEkeys(LogicalSet *ls, std::map<u32, u32> *ekeys) {
    if (!ls) {
        return;
    }
    for (CombInfo &ci : ls->combs) {
        if (ci.ekey != INVALID_EKEY) {
            ci.ekey = ekeys->emplace(ci.id, (u32)ekeys->size()).first->second;
        }
    }
}

/* the logical and combination multibits in the state, after the exhaustion vector (fillStateOffsets,
 * src/rose/rose_build_bytecode.cpp:429-438); returns the offset after them */
u32 layoutLogicalState(const RoseEngine &r, StateOffsets *so, u32 cur) {
    so->logicalVec = cur;
    if (r.ckeyCount) {
        so->logicalVec_size = mmbitSize(r.lkeyCount + r.lopCount);
        cur += so->logicalVec_size;
    }
    so->combVec = cur;
    if (r.ckeyCount) {
        so->combVec_size = mmbitSize(r.ckeyCount);
        cur += so->combVec_size;
    }
    return cur;
}

/* What the header needs to know about the literal set. */
struct RoseTail {
    u32 minLen, maxLen, ekeyCount, dkeyCount, invDkeyOffset;
    bool canExhaust;
    u32 smallWriteOffset = 0;
    const LogicalSet *logic = nullptr;
};

/* Header fields that every route sets alike: report keys, widths, and the sizes of the
 * runtime's (empty) delay / anchored / SOM / handled-key structures. */
void commonHeader(RoseEngine *r, const RoseTail &t) {
    r->canExhaust = t.canExhaust ? 1 : 0;
    r->ekeyCount = t.ekeyCount;
    r->dkeyCount = t.dkeyCount;
    r->dkeyLogSize = fatbitSize(r->dkeyCount);
    r->invDkeyOffset = t.invDkeyOffset;
    r->somLocationFatbitSize = fatbitSize(0);
    r->handledKeyFatbitSize = fatbitSize(0);
    r->minWidth = t.minLen;
    r->minWidthExcludingBoundaries = t.minLen;
    r->maxBiAnchoredWidth = ROSE_BOUND_INF;
    r->floatingDistance = ROSE_BOUND_INF;
    r->delay_fatbit_size = fatbitSize(0);
    r->anchored_fatbit_size = fatbitSize(0);
    r->initMpvNfa = 0xffffffffu; /* MO_INVALID_IDX: no MPV outfix */
}

/* The state layout (fillStateOffsets, src/rose/rose_build_bytecode.cpp:382-465): the status byte
 * (no roles), the active leaf array of `leafCount` engines, `groupsSize` bytes of literal groups,
 * `history` bytes, then the exhaustion, logical and combination vectors.  Returns nfaStateBegin,
 * where the engines' stream state goes. */
u32 layoutState(RoseEngine *r, u32 leafCount, u32 groupsSize, u32 history) {
    StateOffsets &so = r->stateOffsets;
    u32 cur = 1;
    so.activeLeafArray = cur;
    so.activeLeafArray_size = leafCount ? mmbitSize(leafCount) : 0;
    cur += so.activeLeafArray_size;
    so.activeLeftArray = so.longLitState = so.leftfixLagTable = so.anchorState = cur;
    so.groups = cur;
    so.groups_size = groupsSize;
    cur += groupsSize;
    so.history = cur;
    cur += history;
    so.exhausted = cur;
    so.exhausted_size = mmbitSize(r->ekeyCount);
    cur += so.exhausted_size;
    cur = layoutLogicalState(*r, &so, cur);
    so.nfaStateBegin = so.end = cur;
    return cur;
}

/* The floating literal matcher (HWLM over `hl`), added to the blob; the header fields that
 * describe it.  minLen: the shortest literal. */
void addFloatingMatcher(Blob &blob, RoseEngine *r, const std::vector<HwlmLit> &hl, u32 minLen,
                        const CompileOpts &opts, HwlmBuildInfo *info) {
    std::vector<u8> hwlm;
    try {
        hwlm = buildHwlm(hl, opts.hwlm, info);
    } catch (const std::runtime_error &e) {
        throw CompileError{std::string("Unable to build literal matcher: ") + e.what(), -1};
    }
    r->fmatcherOffset = blob.add(hwlm.data(), hwlm.size(), 64);
    r->fmatcherMinWidth = minLen;
    r->floatingMinLiteralMatchOffset = minLen;
    r->initialGroups = 1;
    r->floating_group_mask = 1;
    r->totalNumLiterals = (u32)hl.size();
}

/* Queues [0, K) hold the K engines added to the blob (`engines`: offset and header of each) as the
 * database's outfixes: one NfaInfo per queue, the queue counts, each queue's full state in scratch
 * (64-byte aligned) and its stream state from `cur` (nfaStateBegin) on, in queue order
 * (allocateStateSpace, src/rose/rose_build_bytecode.cpp:2077-2099). */
void addOutfixQueues(Blob &blob, RoseEngine *r, const std::vector<std::pair<u32, NFA>> &engines, u32 cur) {
    const u32 k = (u32)engines.size();
    r->activeArrayCount = k;
    r->queueCount = k;
    r->activeQueueArraySize = fatbitSize(k);
    r->outfixBeginQueue = 0;
    r->outfixEndQueue = k;
    r->leftfixBeginQueue = k;
    std::vector<NfaInfo> infos(k);
    memset(infos.data(), 0, k * sizeof(NfaInfo));
    u32 full = 0;
    for (u32 q = 0; q < k; q++) {
        infos[q].nfaOffset = engines[q].first;
        infos[q].stateOffset = cur;
        infos[q].fullStateOffset = full;
        cur += engines[q].second.streamStateSize;
        full = (u32)HSB_ROUNDUP(full + engines[q].second.scratchStateSize, 64);
    }
    r->scratchStateSize = full;
    r->stateOffsets.end = cur;
    r->stateSize = cur;
    r->nfaInfoOffset = blob.add(infos.data(), k * sizeof(NfaInfo), 4);
}

/* each engine's bytes added to the blob, 64-byte aligned: its offset and header */
std::vector<std::pair<u32, NFA>> addEngines(Blob &blob, const std::vector<std::vector<u8>> &nfas) {
    std::vector<std::pair<u32, NFA>> out;
    for (const std::vector<u8> &nfa : nfas) {
        NFA hdr;
        memcpy(&hdr, nfa.data(), sizeof(hdr));
        out.emplace_back(blob.add(nfa.data(), nfa.size(), 64), hdr);
    }
    return out;
}

/* makeEodProgram (rose_build_bytecode.cpp:3334-3350) with only addEnginesEodProgram: when some engine accepts
 * at end of data, ENGINES_EOD over a sparse iterator of those queues (buildEodNfaIterator, :2276-2294) and END;
 * requiresEodCheck (hasEodAnchors, :2446-2475). */
void addEnginesEodProgram(Blob &blob, RoseEngine *r, const std::vector<std::pair<u32, NFA>> &engines) {
    std::vector<u32> eodQueues;
    for (u32 q = 0; q < engines.size(); q++) {
        if (engines[q].second.flags & NFA_ACCEPTS_EOD) {
            eodQueues.push_back(q);
        }
    }
    if (eodQueues.empty()) {
        return;
    }
    const std::vector<MmbSparseIter> it = mmbSparseIterator(eodQueues, (u32)engines.size());
    const u32 iter = blob.add(it.data(), it.size() * sizeof(MmbSparseIter), alignof(MmbSparseIter));
    const u32 prog = blob.reserve(instrSize<InstrEnginesEod>() + instrSize<InstrEnd>(), INSTR_ALIGN);
    InstrEnginesEod ee;
    memset(&ee, 0, sizeof(ee));
    ee.code = OP_ENGINES_EOD;
    ee.iter_offset = iter;
    memcpy(blob.at(prog), &ee, sizeof(ee));
    *blob.at(prog + instrSize<InstrEnginesEod>()) = OP_END;
    r->eodProgramOffset = prog;
    r->requiresEodCheck = 1;
}

/* The state scatter plan of a block-mode database without roles or leftfixes (buildStateScatterPlan,
 * rose_build_scatter.cpp:66-97): the clear plan of the active leaf array of `leaves` bits, its units laid out
 * as write_out lays them out (u64, u32, u16, u8). */
void addStateScatterPlan(Blob &blob, RoseEngine *r, u32 leaves) {
    const MmbClearPlan p = mmbClearPlan(leaves, r->stateOffsets.activeLeafArray);
    ScatterPlan &sp = r->state_init;
    auto add = [&](const auto &units, u32 *offset, u32 *count) {
        if (!units.empty()) {
            typedef typename std::remove_reference<decltype(units)>::type::value_type Unit;
            *offset = blob.add(units.data(), units.size() * sizeof(Unit), alignof(Unit));
            *count = (u32)units.size();
        }
    };
    add(p.u64s, &sp.s_u64a_offset, &sp.s_u64a_count);
    add(p.u32s, &sp.s_u32_offset, &sp.s_u32_count);
    add(p.u16s, &sp.s_u16_offset, &sp.s_u16_count);
    add(p.u8s, &sp.s_u8_offset, &sp.s_u8_count);
}

/* header + blob, the header's size field set */
std::vector<u8> emitRose(const Blob &blob, RoseEngine *r) {
    const u32 total = (u32)HSB_ROUNDUP(blob.base + blob.bytes.size(), 64);
    r->size = total;
    std::vector<u8> out(total, 0);
    memcpy(out.data(), r, sizeof(*r));
    memcpy(out.data() + blob.base, blob.bytes.data(), blob.bytes.size());
    return out;
}

/* A database whose only matcher is ONE engine run as an outfix over the whole block
 * (ROSE_RUNTIME_SINGLE_OUTFIX: hs_scan -> soleOutfixBlockExec, src/runtime.c:245-280): queue 0,
 * no literal matchers.  What the reference's compiler emits for a pattern set that is all
 * engine and no literal (rose_build_bytecode.cpp:3672-3690 pickRuntimeImpl); here it is built
 * for literal sets on request, so that the DFA / NFA engines run inside a real database. */
std::vector<u8> finishOutfixRose(Blob &blob, const std::vector<u8> &nfa, const RoseTail &t) {
    const std::vector<std::pair<u32, NFA>> engines = addEngines(blob, {nfa});
    RoseEngine r;
    memset(&r, 0, sizeof(r));
    writeLogicalInfo(blob, t.logic, &r);
    commonHeader(&r, t);
    r.runtimeImpl = RUNTIME_SINGLE_OUTFIX;
    r.mode = MODE_BLOCK;
    addOutfixQueues(blob, &r, engines, layoutState(&r, 1, 0, 0));
    return emitRose(blob, &r);
}

/* Floating literal matcher + RoseEngine header around a finished program blob. */
std::vector<u8> finishRose(Blob &blob, const std::vector<HwlmLit> &hl, const RoseTail &t,
                           const CompileOpts &opts, HwlmBuildInfo *info) {
    RoseEngine r;
    memset(&r, 0, sizeof(r));
    addFloatingMatcher(blob, &r, hl, t.minLen, opts, info);
    writeLogicalInfo(blob, t.logic, &r);
    commonHeader(&r, t);
    r.pureLiteral = opts.pureLiteralApi ? 1 : 0;
    r.runtimeImpl = RUNTIME_PURE_LITERAL;
    /* src/rose/rose_build_bytecode.cpp:3615-3622 */
    r.mode = !opts.streaming ? MODE_BLOCK : opts.vectored ? MODE_VECTORED : MODE_STREAM;
    /* matches may start in earlier writes: keep the last maxLen-1 bytes
     * (calcHistoryRequired, src/rose/rose_build_misc.cpp; updated by HWLM) */
    r.historyRequired = opts.streaming && t.maxLen > 1 ? t.maxLen - 1 : 0;
    r.smallWriteOffset = t.smallWriteOffset;
    r.activeQueueArraySize = fatbitSize(0);
    layoutState(&r, 0, 1, r.historyRequired);
    return emitRose(blob, &r);
}

/* A FULL_ROSE database (hs_scan -> roseBlockExec, src/rose/block.c:345-422) whose engines (`nfas`) run as
 * the outfixes on queues [0, K), beside the floating literal matcher over `hl` or, with `hl` empty, alone:
 * init_for_block clears the active leaf array through the state scatter plan, blockInitSufPQ starts every
 * outfix, the literal programs' CATCH_UP and roseCatchUpTo(length) run them and merge their reports in
 * offset order, and for the outfixes that accept at end of data the EOD program's ENGINES_EOD checks their
 * final states (roseBlockEodExec).  litMinLen: the shortest literal; t.minLen: the shortest match of all. */
std::vector<u8> finishFullRose(Blob &blob, const std::vector<HwlmLit> &hl, u32 litMinLen,
                               const std::vector<std::vector<u8>> &nfas, const RoseTail &t, const CompileOpts &opts,
                               HwlmBuildInfo *info) {
    RoseEngine r;
    memset(&r, 0, sizeof(r));
    if (!hl.empty()) {
        addFloatingMatcher(blob, &r, hl, litMinLen, opts, info);
    }
    const std::vector<std::pair<u32, NFA>> engines = addEngines(blob, nfas);
    commonHeader(&r, t);
    r.runtimeImpl = RUNTIME_FULL_ROSE;
    r.mode = MODE_BLOCK;
    /* no bi-anchored patterns (findMaxBAWidth): roseBlockFloating scans blocks of any length */
    r.amatcherMaxBiAnchoredWidth = ROSE_BOUND_INF;
    r.fmatcherMaxBiAnchoredWidth = ROSE_BOUND_INF;
    const u32 cur = layoutState(&r, (u32)engines.size(), hl.empty() ? 0 : 1, 0);
    addEnginesEodProgram(blob, &r, engines);
    addStateScatterPlan(blob, &r, (u32)engines.size());
    addOutfixQueues(blob, &r, engines, cur);
    return emitRose(blob, &r);
}

/* report id -> (HS_FLAG_SINGLEMATCH, index of the first expression with it) */
typedef std::map<u32, std::pair<bool, u32>> HighlanderMap;

/* Every expression with one report id must agree on HS_FLAG_SINGLEMATCH (src/compiler/compiler.cpp). */
void checkHighlander(HighlanderMap *seen, u32 report, bool single, u32 index) {
    auto it = seen->find(report);
    if (it == seen->end()) {
        (*seen)[report] = {single, index};
    } else if (it->second.first != single) {
        std::string m = "Expression (index " + std::to_string(index) + ") with match ID " + std::to_string(report) + " ";
        m += single ? "specified " : "did not specify ";
        m += "HS_FLAG_SINGLEMATCH whereas previous expression (index " + std::to_string(it->second.second) +
             ") with the same match ID did";
        m += single ? " not." : ".";
        throw CompileError{m, (int)index};
    }
}

/* The literal set validated, case-folded and without exact duplicates; keys not yet assigned. */
std::vector<PatInfo> prepareLiterals(const std::vector<LitPattern> &patsIn, const CompileOpts &opts,
                                     HighlanderMap *idHighlander) {
    if (patsIn.empty()) {
        throw CompileError{"Invalid parameter: elements is zero", -1};
    }
    if (patsIn.size() > LIMIT_LITERAL_COUNT) {
        throw CompileError{"Number of patterns too large", -1};
    }
    std::vector<PatInfo> pats;
    std::set<std::tuple<std::string, bool, u32>> seen;
    for (const LitPattern &p : patsIn) {
        if (p.s.empty()) {
            throw CompileError{"Pure literal API doesn't support empty string.", (int)p.index};
        }
        if (p.s.size() > LIMIT_PATTERN_LENGTH) {
            throw CompileError{"Pattern length exceeds limit.", (int)p.index};
        }
        if (p.s.size() > LIMIT_LITERAL_LENGTH) {
            throw CompileError{"Resource limit exceeded.", (int)p.index};
        }
        if (opts.streaming && p.s.size() > 8) {
            /* in streaming mode literals beyond the literal matcher's 8 bytes need
             * the long-literal table and the full rose runtime
             * (src/rose/rose_build_bytecode.cpp:292-296 isPureFloating) */
            throw CompileError{"Streaming and vectored modes in this build support literals of up to 8 "
                               "bytes; longer literals need the long literal table.", (int)p.index};
        }
        checkHighlander(idHighlander, p.report, p.singlematch, p.index);
        PatInfo pi;
        pi.p = &p;
        pi.folded = p.s;
        pi.anyAlpha = false;
        for (char &c : pi.folded) {
            if (isAsciiAlpha((u8)c)) {
                pi.anyAlpha = true;
                if (p.caseless) {
                    c = (char)asciiUpper((u8)c);
                }
            }
        }
        bool effNocase = p.caseless && pi.anyAlpha;
        if (!seen.insert(std::make_tuple(pi.folded, effNocase, p.report)).second) {
            continue; /* identical literal + report: one report source */
        }
        pi.ekey = pi.dkey = INVALID_EKEY;
        pats.push_back(pi);
    }
    return pats;
}

/* Exhaustion keys for the HS_FLAG_SINGLEMATCH ids, dedupe keys for ids that more than one pattern
 * raises -- or that `engineIds` (the ids an engine raises too) holds.  Returns whether every
 * pattern is single-match. */
bool assignLiteralKeys(std::vector<PatInfo> *patsIo, const std::set<u32> &engineIds, std::map<u32, u32> *ekeysOut,
                       std::map<u32, u32> *dkeysOut) {
    std::vector<PatInfo> &pats = *patsIo;
    std::map<u32, u32> &ekeys = *ekeysOut, &dkeys = *dkeysOut;
    std::map<u32, u32> perReport;
    for (const auto &pi : pats) {
        perReport[pi.p->report]++;
    }
    for (u32 id : engineIds) {
        perReport[id]++;
    }
    bool allHighlander = true;
    for (auto &pi : pats) {
        const u32 r = pi.p->report;
        if (pi.p->singlematch) {
            auto it = ekeys.find(r);
            if (it == ekeys.end()) {
                it = ekeys.emplace(r, (u32)ekeys.size()).first;
            }
            pi.ekey = it->second;
        } else {
            allHighlander = false;
        }
        if (perReport[r] > 1) {
            auto it = dkeys.find(r);
            if (it == dkeys.end()) {
                it = dkeys.emplace(r, (u32)dkeys.size()).first;
            }
            pi.dkey = it->second;
        }
    }
    return allHighlander;
}

/* The literal programs, one per fragment (literals grouped by their 8-byte suffix and effective
 * case), added to the blob; returns the floating matcher's literals (ids = program offsets).
 * catchUp: each report block starts with CATCH_UP (makeCatchup, src/rose/rose_build_program.cpp:412-434),
 * as in a database with an outfix (needsCatchup, src/rose/rose_build_bytecode.cpp:226). */
std::vector<HwlmLit> writeLiteralPrograms(Blob &blob, const std::vector<PatInfo> &pats, const LogicalSet *logic,
                                          bool catchUp, u32 *minLen, u32 *maxLen) {
    const u32 catchUpSize = catchUp ? instrSize<InstrCatchUp>() : 0;
    /* --- group into fragments by (8-byte suffix, effective nocase) --- */
    struct Fragment {
        std::string suffix;
        bool nocase;
        std::vector<u32> pats;
        u32 program = 0;
    };
    std::vector<Fragment> frags;
    std::map<std::pair<std::string, bool>, u32> fragIndex;
    for (u32 i = 0; i < pats.size(); i++) {
        const std::string &f = pats[i].folded;
        std::string suf = f.size() > 8 ? f.substr(f.size() - 8) : f;
        bool nc = false;
        if (pats[i].p->caseless) {
            for (char c : suf) {
                nc |= isAsciiAlpha((u8)c);
            }
        }
        auto key = std::make_pair(suf, nc);
        auto it = fragIndex.find(key);
        if (it == fragIndex.end()) {
            it = fragIndex.emplace(key, (u32)frags.size()).first;
            frags.push_back({suf, nc, {}, 0});
        }
        frags[it->second].pats.push_back(i);
    }

    /* --- programs --- */
    struct PendingLit {
        u32 instrOff;
        std::string bytes;
    };
    std::vector<PendingLit> pendingLits;
    for (Fragment &fr : frags) {
        u32 total = instrSize<InstrEnd>();
        for (u32 pi : fr.pats) {
            total += blockSize(pats[pi], logic) + catchUpSize;
        }
        const u32 start = blob.reserve(total, INSTR_ALIGN);
        fr.program = start;
        u32 pc = start;
        for (size_t k = 0; k < fr.pats.size(); k++) {
            const PatInfo &pi = pats[fr.pats[k]];
            const u32 next = pc + blockSize(pi, logic) + catchUpSize; /* next pattern's block or END */
            if (pi.p->s.size() > 8) {
                InstrCheckLit in;
                memset(&in, 0, sizeof(in));
                bool nc = pi.p->caseless && pi.anyAlpha;
                in.code = nc ? OP_CHECK_MED_LIT_NOCASE : OP_CHECK_MED_LIT;
                in.lit_length = (u32)pi.folded.size();
                in.fail_jump = next - pc;
                memcpy(blob.at(pc), &in, sizeof(in));
                pendingLits.push_back({pc, pi.folded});
                pc += instrSize<InstrCheckLit>();
            }
            if (catchUp) {
                *blob.at(pc) = OP_CATCH_UP;
                pc += catchUpSize;
            }
            writeReport(blob, pc, pi, next, logic);
            pc = next;
        }
        InstrEnd e;
        e.code = OP_END;
        memcpy(blob.at(pc), &e, sizeof(e));
    }
    for (const PendingLit &pl : pendingLits) {
        u32 off = blob.add(pl.bytes.data(), pl.bytes.size(), 1);
        InstrCheckLit in;
        memcpy(&in, blob.at(pl.instrOff), sizeof(in));
        in.lit_offset = off;
        memcpy(blob.at(pl.instrOff), &in, sizeof(in));
    }

    std::vector<HwlmLit> hl;
    /* --- the floating matcher's literals --- */
    for (const Fragment &fr : frags) {
        HwlmLit l;
        l.s = fr.suffix;
        l.nocase = fr.nocase;
        l.noruns = false;
        l.id = fr.program;
        l.groups = 1;
        hl.push_back(l);
    }
    *minLen = ~0u;
    *maxLen = 0;
    for (const auto &pi : pats) {
        *minLen = std::min<u32>(*minLen, (u32)pi.folded.size());
        *maxLen = std::max<u32>(*maxLen, (u32)pi.folded.size());
    }
    return hl;
}

/* the dkey -> external report id table (rose_internal.h:354), or 0 without dedupe keys */
u32 addInvDkeys(Blob &blob, const std::map<u32, u32> &dkeys) {
    if (dkeys.empty()) {
        return 0;
    }
    std::vector<u32> inv(dkeys.size());
    for (const auto &d : dkeys) {
        inv[d.second] = d.first;
    }
    return blob.add(inv.data(), inv.size() * sizeof(u32), 4);
}

/* Report keys of the expressions: one exhaustion key per HS_FLAG_SINGLEMATCH report id; one dedupe key per report
 * id, always -- several accepting positions (or expressions) may raise one id at one offset and
 * the reference delivers a report once (dedupe, src/report.h:55-119) */
bool assignRegexKeys(const std::vector<RegexPattern> &pats, HighlanderMap *highlander, std::map<u32, u32> *ekeys,
                     std::map<u32, u32> *dkeys) {
    bool allHighlander = true;
    for (const RegexPattern &p : pats) {
        const bool single = (p.flags & HS_FLAG_SINGLEMATCH) != 0;
        checkHighlander(highlander, p.report, single, p.index);
        if (single) {
            ekeys->emplace(p.report, (u32)ekeys->size());
        } else {
            allHighlander = false;
        }
        dkeys->emplace(p.report, (u32)dkeys->size());
    }
    return allHighlander;
}

/* The report programs of the expressions (added to the blob) and ONE engine over all of them, whose
 * reports are those programs' offsets: McClellan-8 / 16 when the determinised automaton stays small
 * and `opts.regexDfa`, else LimEx.  *minLen: the shortest match. */
std::vector<u8> buildRegexEngine(Blob &blob, const std::vector<RegexPattern> &pats, std::map<u32, u32> &ekeys,
                                 std::map<u32, u32> &dkeys, const LogicalSet *logic, const CompileOpts &opts,
                                 u32 *minLen) {
    RawNfa nfa;
    regexNfaInit(&nfa);
    *minLen = ~0u;
    std::map<std::tuple<u32, int, u64, u64>, u32> progOf; /* (report id, offset_adjust, bounds) -> its report program */
    auto program = [&](const RegexPattern &p, int adjust) -> u32 {
        const auto key = std::make_tuple(p.report, adjust, p.minOffset, p.maxOffset);
        auto pit = progOf.find(key);
        if (pit != progOf.end()) {
            return pit->second;
        }
        const bool single = (p.flags & HS_FLAG_SINGLEMATCH) != 0;
        const bool quiet = (p.flags & HS_FLAG_QUIET) != 0;
        const bool bounded = p.minOffset > 0 || p.maxOffset != ~0ull;
        u32 sz = instrSize<InstrEnd>() + (bounded ? instrSize<InstrCheckBounds>() : 0) + flushSize(logic) +
                 logicalSize(logic, p.report);
        sz += single ? instrSize<InstrCheckExhausted>() + instrSize<InstrDedupe>() + instrSize<InstrReportExhaust>()
                     : quiet ? instrSize<InstrDedupe>() : instrSize<InstrDedupeAndReport>();
        u32 pc = blob.reserve(sz, INSTR_ALIGN);
        const u32 prog = pc;
        const u32 endAt = pc + sz - instrSize<InstrEnd>();
        if (bounded) {
            /* makeReport (src/rose/rose_build_program.cpp:533-538): the bounds come first, and they are on the raw
             * match end -- min_offset / max_offset less the report's offset_adjust (ng_extparam.cpp:199-211) */
            InstrCheckBounds cb;
            memset(&cb, 0, sizeof(cb));
            cb.code = OP_CHECK_BOUNDS;
            cb.min_bound = p.minOffset - (u64)(long long)adjust;
            cb.max_bound = p.maxOffset == ~0ull ? ~0ull : p.maxOffset - (u64)(long long)adjust;
            cb.fail_jump = endAt - pc;
            memcpy(blob.at(pc), &cb, sizeof(cb));
            pc += instrSize<InstrCheckBounds>();
        }
        if (single) {
            InstrCheckExhausted ce;
            memset(&ce, 0, sizeof(ce));
            ce.code = OP_CHECK_EXHAUSTED;
            ce.ekey = ekeys[p.report];
            ce.fail_jump = endAt - pc;
            memcpy(blob.at(pc), &ce, sizeof(ce));
            pc += instrSize<InstrCheckExhausted>();
            pc = writeFlush(blob, pc, logic);
            InstrDedupe dd;
            memset(&dd, 0, sizeof(dd));
            dd.code = OP_DEDUPE;
            dd.dkey = dkeys[p.report];
            dd.offset_adjust = adjust;
            dd.fail_jump = endAt - pc;
            memcpy(blob.at(pc), &dd, sizeof(dd));
            pc += instrSize<InstrDedupe>();
            InstrReportExhaust re;
            memset(&re, 0, sizeof(re));
            re.code = OP_REPORT_EXHAUST;
            re.onmatch = p.report;
            re.offset_adjust = adjust;
            re.ekey = ekeys[p.report];
            memcpy(blob.at(pc), &re, sizeof(re));
            pc += instrSize<InstrReportExhaust>();
        } else if (quiet) {
            pc = writeFlush(blob, pc, logic);
            InstrDedupe dd;
            memset(&dd, 0, sizeof(dd));
            dd.code = OP_DEDUPE;
            dd.dkey = dkeys[p.report];
            dd.offset_adjust = adjust;
            dd.fail_jump = endAt - pc;
            memcpy(blob.at(pc), &dd, sizeof(dd));
            pc += instrSize<InstrDedupe>();
        } else {
            pc = writeFlush(blob, pc, logic);
            InstrDedupeAndReport dr;
            memset(&dr, 0, sizeof(dr));
            dr.code = OP_DEDUPE_AND_REPORT;
            dr.dkey = dkeys[p.report];
            dr.onmatch = p.report;
            dr.offset_adjust = adjust;
            dr.fail_jump = endAt - pc;
            memcpy(blob.at(pc), &dr, sizeof(dr));
            pc += instrSize<InstrDedupeAndReport>();
        }
        writeLogical(blob, pc, logic, p.report, adjust);
        InstrEnd e;
        e.code = OP_END;
        memcpy(blob.at(endAt), &e, sizeof(e));
        progOf[key] = prog;
        return prog;
    };
    for (const RegexPattern &p : pats) {
        try {
            const RegexInfo ri = regexInfo(p.re.c_str(), p.flags, false, p.minLength);
            /* extended parameters no match can satisfy (src/nfagraph/ng_extparam.cpp:820-880) */
            if (p.minLength && ri.maxLen != 0xffffffffu && p.minLength > ri.maxLen) {
                throw CompileError{"Expression has min_length=" + std::to_string(p.minLength) + " but can only produce matches of length " +
                                       std::to_string(ri.maxLen) + " bytes at most.", (int)p.index};
            }
            if (p.maxOffset != ~0ull && ri.minLen > p.maxOffset) {
                throw CompileError{"Expression has max_offset=" + std::to_string(p.maxOffset) + " but requires " +
                                       std::to_string(ri.minLen) + " bytes to match.", (int)p.index};
            }
            if (ri.anchored && p.minOffset && ri.maxLen != 0xffffffffu && p.minOffset > ri.maxLen) {
                throw CompileError{"Expression is anchored and cannot satisfy min_offset=" + std::to_string(p.minOffset) +
                                       " as it can only produce matches of length " + std::to_string(ri.maxLen) + " bytes at most.",
                                   (int)p.index};
            }
            if (p.minLength || p.maxOffset != ~0ull) {
                /* ... and taken together: some alternative must have a match that is long enough and can end early
                 * enough (the reference prunes the graph by the parameters and reports what is left) */
                bool some = false;
                for (const auto &w : ri.armWidths) {
                    some |= (w.second == 0xffffffffu || w.second >= p.minLength) &&
                            std::max<u64>(w.first, p.minLength) <= p.maxOffset;
                }
                if (!some) {
                    throw CompileError{"Extended parameter constraints can not be satisfied for any match from this "
                                       "expression.", (int)p.index};
                }
            }
            {
                /* "Pattern can never match." (can_never_match after resolveAsserts, src/nfagraph/ng.cpp:330-350): the
                 * expression's own automaton, determinised and minimised, is the dead state alone */
                RawNfa own;
                regexNfaInit(&own);
                regexNfaAdd(&own, p.re.c_str(), p.flags, 1, ri.needsAdjust ? 2 : 0, p.minLength);
                RawDfa d;
                if (determinize(own, 1024, &d)) {
                    minimizeDfa(&d);
                    if (d.size() < 2) {
                        throw CompileError{"Pattern can never match.", (int)p.index};
                    }
                }
            }
            *minLen = std::min<u32>(*minLen, (u32)std::max<u64>(ri.minLen, std::min<u64>(p.minLength, 0xffffffffu)));
            regexNfaAdd(&nfa, p.re.c_str(), p.flags, program(p, 0), ri.needsAdjust ? program(p, -1) : 0, p.minLength);
        } catch (const RegexError &e) {
            throw CompileError{e.msg, (int)p.index};
        }
    }
    try {
        /* small automata run as DFAs, as in the reference (ng_mcclellan before LimEx); the report programs are
         * the same either way */
        RawDfa dfa;
        bool asDfa = opts.regexDfa && determinize(nfa, 1024, &dfa);
        if (asDfa) {
            minimizeDfa(&dfa);
            /* (nothing left but the dead state: an expression set that cannot match; it stays an NFA) */
            asDfa = dfa.size() >= 2 && dfa.size() <= 1024;
        }
        if (asDfa) {
            return emitDfa(dfa, dfa.size() <= 256 ? DFA_MCCLELLAN8 : DFA_MCCLELLAN16, true);
        } else {
            return emitLimEx(nfa);
        }
    } catch (const std::runtime_error &e) {
        throw CompileError{std::string("Unable to build the NFA: ") + e.what(), -1};
    }
}

/* The expressions of a set too large for one engine, in groups whose position automaton fits one: packed
 * greedily in expression order -- an expression joins the last group while that group's automaton can take
 * its positions (regexNfaAdd stays within the 512-state model), else it opens the next group.  The same set
 * therefore always splits the same way.  Throws CompileError when an expression does not fit an engine of
 * its own. */
std::vector<std::vector<RegexPattern>> packEngineGroups(const std::vector<RegexPattern> &pats) {
    std::vector<std::vector<RegexPattern>> groups;
    RawNfa last; /* the automaton of the last group */
    for (const RegexPattern &p : pats) {
        try {
            const RegexInfo ri = regexInfo(p.re.c_str(), p.flags, false, p.minLength);
            /* the reports do not change the positions: placeholders stand in for the report programs */
            auto add = [&](RawNfa *n) { regexNfaAdd(n, p.re.c_str(), p.flags, 1, ri.needsAdjust ? 2 : 0, p.minLength); };
            if (!groups.empty()) {
                RawNfa trial = last;
                try {
                    add(&trial);
                    last = std::move(trial);
                    groups.back().push_back(p);
                    continue;
                } catch (const RegexError &) {
                }
            }
            regexNfaInit(&last);
            add(&last);
            groups.push_back({p});
        } catch (const RegexError &e) {
            throw CompileError{e.msg, (int)p.index};
        }
    }
    return groups;
}

} // namespace

std::vector<u8> buildLiteralRose(const std::vector<LitPattern> &patsIn,
                                 const CompileOpts &opts, HwlmBuildInfo *info, LogicalSet *logic) {
    HighlanderMap highlander;
    std::vector<PatInfo> pats = prepareLiterals(patsIn, opts, &highlander);
    std::map<u32, u32> ekeys, dkeys;
    const bool allHighlander = assignLiteralKeys(&pats, std::set<u32>(), &ekeys, &dkeys);
    assignCombinationEkeys(logic, &ekeys);

    if (opts.outfixKind) {
        /* --- single-outfix database: report programs ([CHECK_EXHAUSTED] [DEDUPE] REPORT_EXHAUST |
         * DEDUPE_AND_REPORT | REPORT, END -- run by roseReportAdaptor / roseRunProgram), one engine
         * over the whole literals whose reports are those programs' offsets --- */
        if (opts.streaming) {
            throw CompileError{"Single-engine databases are built for block mode only.", -1};
        }
        Blob blob((u32)HSB_ROUNDUP(sizeof(RoseEngine), 64));
        std::vector<DfaLiteral> dl;
        u32 minLen = ~0u, maxLen = 0;
        for (const PatInfo &pi : pats) {
            minLen = std::min<u32>(minLen, (u32)pi.p->s.size());
            maxLen = std::max<u32>(maxLen, (u32)pi.p->s.size());
            const u32 sz = reportSize(pi, logic) + instrSize<InstrEnd>();
            const u32 prog = blob.reserve(sz, INSTR_ALIGN), endAt = prog + sz - instrSize<InstrEnd>();
            writeReport(blob, prog, pi, endAt, logic);
            InstrEnd e;
            e.code = OP_END;
            memcpy(blob.at(endAt), &e, sizeof(e));
            DfaLiteral l;
            l.s = pi.p->s;
            l.caseless = pi.p->caseless && pi.anyAlpha;
            l.report = prog;
            dl.push_back(l);
        }
        RoseTail t;
        t.minLen = minLen;
        t.maxLen = maxLen;
        t.ekeyCount = (u32)ekeys.size();
        t.dkeyCount = (u32)dkeys.size();
        t.invDkeyOffset = addInvDkeys(blob, dkeys);
        t.canExhaust = allHighlander;
        t.logic = logic;
        std::vector<u8> nfa;
        try {
            if (opts.outfixKind == OUTFIX_LIMEX32) {
                nfa = emitLimEx(nfaFromLiterals(dl));
            } else {
                const DfaKind k = opts.outfixKind == OUTFIX_MCCLELLAN8    ? DFA_MCCLELLAN8
                                  : opts.outfixKind == OUTFIX_MCCLELLAN16 ? DFA_MCCLELLAN16
                                  : opts.outfixKind == OUTFIX_SHENG       ? DFA_SHENG
                                                                          : DFA_AUTO;
                nfa = emitDfa(dfaFromLiterals(dl, false), k, false);
            }
        } catch (const std::runtime_error &e) {
            throw CompileError{std::string("Unable to build the engine: ") + e.what(), -1};
        }
        if (info) {
            memset(info, 0, sizeof(*info));
        }
        return finishOutfixRose(blob, nfa, t);
    }

    Blob blob((u32)HSB_ROUNDUP(sizeof(RoseEngine), 64));
    u32 minLen = 0, maxLen = 0;
    const std::vector<HwlmLit> hl = writeLiteralPrograms(blob, pats, logic, false, &minLen, &maxLen);
    const u32 invDkeyOffset = addInvDkeys(blob, dkeys);
    RoseTail t;
    t.minLen = minLen;
    t.maxLen = maxLen;
    t.ekeyCount = (u32)ekeys.size();
    t.dkeyCount = (u32)dkeys.size();
    t.invDkeyOffset = invDkeyOffset;
    t.canExhaust = allHighlander;
    t.logic = logic;

    /* --- small-write engine (src/smallwrite/smallwrite_build.cpp; used by hs_scan for
     * buffers shorter than largestBuffer, src/runtime.c:401-413): one DFA over the WHOLE
     * literals whose reports are the offsets of report programs -- the literal's program
     * without the literal check, which the DFA has already done -- run through
     * roseReportAdaptor (src/rose/match.c:611-633).  Only while the automaton stays small
     * (12 000 literal bytes, 16 K states); otherwise no engine, like the reference when its
     * DFA limits are exceeded. --- */
    if (opts.smallWrite && !opts.streaming) {
        const u32 LARGEST_BUFFER = 70; /* Grey::smallWriteLargestBuffer, src/grey.cpp:135 */
        std::vector<DfaLiteral> dl;
        size_t budget = 0;
        bool ok = true;
        for (const PatInfo &pi : pats) {
            if (pi.p->s.size() >= LARGEST_BUFFER) {
                continue; /* cannot match in a buffer that short */
            }
            const bool nc = pi.p->caseless && pi.anyAlpha;
            budget += pi.p->s.size();
            if (budget > 12000) { /* positions of the automaton; it may still grow past 16 K states */
                ok = false;
                break;
            }
            /* report program: [CHECK_EXHAUSTED] [DEDUPE] REPORT_EXHAUST | DEDUPE_AND_REPORT | REPORT, END */
            const u32 sz = reportSize(pi, logic) + instrSize<InstrEnd>();
            const u32 prog = blob.reserve(sz, INSTR_ALIGN), endAt = prog + sz - instrSize<InstrEnd>();
            writeReport(blob, prog, pi, endAt, logic);
            InstrEnd e;
            e.code = OP_END;
            memcpy(blob.at(endAt), &e, sizeof(e));
            DfaLiteral l;
            l.s = pi.p->s;
            l.caseless = nc;
            l.report = prog;
            dl.push_back(l);
        }
        if (ok && !dl.empty()) {
            try {
                const std::vector<u8> nfa = emitDfa(dfaFromLiterals(dl, false), DFA_AUTO, false);
                SmallWriteEngine sw;
                memset(&sw, 0, sizeof(sw));
                sw.largestBuffer = LARGEST_BUFFER;
                sw.start_offset = 0;
                sw.size = (u32)(sizeof(SmallWriteEngine) + nfa.size());
                t.smallWriteOffset = blob.add(&sw, sizeof(sw), 64);
                blob.add(nfa.data(), nfa.size(), 64);
            } catch (const std::runtime_error &) {
                /* automaton too large: no small-write engine */
            }
        }
    }
    return finishRose(blob, hl, t, opts, info);
}

std::vector<u8> buildRegexRose(const std::vector<RegexPattern> &pats, const CompileOpts &opts, LogicalSet *logic) {
    if (pats.empty()) {
        throw CompileError{"Invalid parameter: elements is zero", -1};
    }
    if (opts.streaming) {
        throw CompileError{"Expressions that need an NFA engine are compiled for block mode only in this build.", -1};
    }
    HighlanderMap highlander;
    std::map<u32, u32> ekeys, dkeys;
    const bool allHighlander = assignRegexKeys(pats, &highlander, &ekeys, &dkeys);
    assignCombinationEkeys(logic, &ekeys);
    Blob blob((u32)HSB_ROUNDUP(sizeof(RoseEngine), 64));
    u32 minLen = 0;
    const std::vector<u8> eng = buildRegexEngine(blob, pats, ekeys, dkeys, logic, opts, &minLen);
    RoseTail t;
    t.minLen = minLen;
    t.maxLen = 0;
    t.ekeyCount = (u32)ekeys.size();
    t.dkeyCount = (u32)dkeys.size();
    std::vector<u32> inv(dkeys.size());
    for (const auto &d : dkeys) {
        inv[d.second] = d.first;
    }
    t.invDkeyOffset = blob.add(inv.data(), inv.size() * sizeof(u32), 4);
    t.canExhaust = allHighlander;
    t.logic = logic;
    return finishOutfixRose(blob, eng, t);
}

std::vector<u8> buildMixedRose(const std::vector<LitPattern> &lits, const std::vector<RegexPattern> &regexes,
                               const CompileOpts &opts, HwlmBuildInfo *info) {
    if (regexes.empty() || opts.streaming) {
        throw CompileError{"A literal matcher with an engine is built for block mode only.", -1};
    }
    /* one report id is one exhaustion key and one dedupe key, whichever half raises it */
    HighlanderMap highlander;
    std::vector<PatInfo> pats = prepareLiterals(lits, opts, &highlander);
    std::set<u32> engineIds;
    for (const RegexPattern &p : regexes) {
        engineIds.insert(p.report);
    }
    std::map<u32, u32> ekeys, dkeys;
    const bool litHighlander = assignLiteralKeys(&pats, engineIds, &ekeys, &dkeys);
    const bool regexHighlander = assignRegexKeys(regexes, &highlander, &ekeys, &dkeys);
    Blob blob((u32)HSB_ROUNDUP(sizeof(RoseEngine), 64));
    u32 litMin = 0, litMax = 0, regexMin = 0;
    const std::vector<HwlmLit> hl = writeLiteralPrograms(blob, pats, nullptr, true, &litMin, &litMax);
    const std::vector<u8> eng = buildRegexEngine(blob, regexes, ekeys, dkeys, nullptr, opts, &regexMin);
    RoseTail t;
    t.minLen = std::min(litMin, regexMin);
    t.maxLen = litMax;
    t.ekeyCount = (u32)ekeys.size();
    t.dkeyCount = (u32)dkeys.size();
    t.invDkeyOffset = addInvDkeys(blob, dkeys);
    t.canExhaust = litHighlander && regexHighlander;
    return finishFullRose(blob, hl, litMin, {eng}, t, opts, info);
}

std::vector<u8> buildMultiOutfixRose(const std::vector<RegexPattern> &pats, const CompileOpts &opts) {
    if (pats.empty() || opts.streaming) {
        throw CompileError{"Expression sets of several engines are built for block mode only.", -1};
    }
    /* one report id is one exhaustion key and one dedupe key, whichever engine raises it */
    HighlanderMap highlander;
    std::map<u32, u32> ekeys, dkeys;
    const bool allHighlander = assignRegexKeys(pats, &highlander, &ekeys, &dkeys);
    const std::vector<std::vector<RegexPattern>> groups = packEngineGroups(pats);
    Blob blob((u32)HSB_ROUNDUP(sizeof(RoseEngine), 64));
    std::vector<std::vector<u8>> engines;
    u32 minLen = ~0u;
    for (const std::vector<RegexPattern> &g : groups) {
        u32 groupMin = 0;
        engines.push_back(buildRegexEngine(blob, g, ekeys, dkeys, nullptr, opts, &groupMin));
        minLen = std::min(minLen, groupMin);
    }
    RoseTail t;
    t.minLen = minLen;
    t.maxLen = 0;
    t.ekeyCount = (u32)ekeys.size();
    t.dkeyCount = (u32)dkeys.size();
    t.invDkeyOffset = addInvDkeys(blob, dkeys);
    t.canExhaust = allHighlander;
    return finishFullRose(blob, std::vector<HwlmLit>(), 0, engines, t, opts, nullptr);
}

/* Test hook (hs_b200_test_compile_programs): a pure-literal block database whose
 * literal programs are given as raw instruction bytes -- the way to reach every
 * opcode of roseRunProgram_l (src/rose/program_runtime.c:3101-3522) that this
 * compiler does not emit itself.  lits[i].id = offset of its program inside
 * `area`, which is placed at programAreaBase(); absolute offsets inside the
 * programs (lit_offset, child_offset) are the caller's business. */
u32 programAreaBase() { return (u32)HSB_ROUNDUP(sizeof(RoseEngine), 64); }

std::vector<u8> buildRawProgramRose(std::vector<HwlmLit> lits, const std::vector<u8> &area,
                                    u32 ekeyCount, const std::vector<u32> &invDkey,
                                    const CompileOpts &opts, HwlmBuildInfo *info) {
    if (lits.empty()) {
        throw CompileError{"Invalid parameter: elements is zero", -1};
    }
    Blob blob(programAreaBase());
    blob.add(area.data(), area.size(), INSTR_ALIGN);
    RoseTail t;
    t.minLen = ~0u;
    t.maxLen = 0;
    for (HwlmLit &l : lits) {
        if (l.s.empty() || l.s.size() > 8 || l.id >= area.size() || (l.id % INSTR_ALIGN)) {
            throw CompileError{"bad literal or program offset", -1};
        }
        l.id += blob.base;
        t.minLen = std::min<u32>(t.minLen, (u32)l.s.size());
        t.maxLen = std::max<u32>(t.maxLen, (u32)l.s.size());
    }
    t.ekeyCount = ekeyCount;
    t.dkeyCount = (u32)invDkey.size();
    t.invDkeyOffset = invDkey.empty() ? 0 : blob.add(invDkey.data(), invDkey.size() * sizeof(u32), 4);
    t.canExhaust = false;
    return finishRose(blob, lits, t, opts, info);
}

} // namespace hsb
