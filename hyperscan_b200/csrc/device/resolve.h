/*
 * resolve.h -- the report tables of a database on the device (DeviceRules, uploaded with its image), and what one
 * match becomes through them: the look-ups the ordering (order_kernels.h) and the match mask (scan_kernels.cu,
 * dfa_kernels.cu) share.  Each translation unit that includes it gets its own copy of these inline functions.
 */
#ifndef HSB200_RESOLVE_H
#define HSB200_RESOLVE_H

#include "kernels.h"

namespace hsb {

namespace {

/* index of v in the ascending table[0, n), or -1 (a program offset in progOff, a report id in ids) */
__device__ __forceinline__ int indexOf(const u32 *table, u32 n, u32 v) {
    u32 lo = 0, hi = n;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        const u32 t = __ldg(table + mid);
        if (t == v) {
            return (int)mid;
        }
        if (t < v) {
            lo = mid + 1;
        } else {
            hi = mid;
        }
    }
    return -1;
}

/* The reports an engine's record raises (ReportRules::deliver): f(rep) for each report instruction of program k
 * (its index in progOff; -1 = none) whose CHECK_BOUNDS admits the record's end offset `to`.  Returns how many. */
template <class F>
__device__ __forceinline__ u32 programReports(const u32 *progStart, const OrderRep *reps, int k, u64 to, F f) {
    if (k < 0) {
        return 0;
    }
    u32 n = 0;
    const u32 e = __ldg(progStart + k + 1);
    for (u32 q = __ldg(progStart + k); q < e; q++) {
        const OrderRep &rp = reps[q];
        const bool in = to >= rp.lo && to <= rp.hi;
        if (in) {
            f(rp);
        }
        n += in;
    }
    return n;
}

/* A mask pass: set the bit of report id `id` in row `block` (an id outside the table sets none).  The word is
 * read first, so that an id that fires again in the same block costs a load, not an atomic: bits only go from 0
 * to 1 during the pass, so a stale read can only send a match to the atomic. */
__device__ __forceinline__ void maskReport(const MaskOut &m, u32 id, u32 block) {
    const int r = indexOf(m.ids, m.nIds, id);
    if (r < 0) {
        return;
    }
    u32 *w = m.bits + (u64)block * m.words + ((u32)r >> 5);
    const u32 bit = 1u << ((u32)r & 31);
    if (!(*w & bit)) {
#ifdef HSB_HOST_EMU /* the SIMT emulator of tests/emu runs one thread at a time between its barriers */
        *w |= bit;
#else
        atomicOr(w, bit);
#endif
    }
}

/* A first-match pass: lower block `block`'s entry to (to << 32) | id, the delivery order's key within a block (every
 * id counts, as in the ordering, known to the id table or not).  The entry is read first, so that a match that
 * cannot win costs a load, not an atomic: entries only go down during the pass, so a stale read can only send a
 * match to the atomic. */
__device__ __forceinline__ void firstReport(const MaskOut &m, u32 id, u32 block, u64 to) {
    unsigned long long *e = m.first + block;
    const unsigned long long key = (to << 32) | id;
    if (*(volatile unsigned long long *)e > key) {
#ifdef HSB_HOST_EMU /* the SIMT emulator of tests/emu runs one thread at a time between its barriers */
        *e = key;
#else
        atomicMin(e, key);
#endif
    }
}

/* the `to` of block `block`'s entry so far (~0 >> 32 = none): a match that ends later cannot win */
__device__ __forceinline__ u32 firstTo(const MaskOut &m, u32 block) {
    return (u32)(*(volatile unsigned long long *)(m.first + block) >> 32);
}

/* A first-match pass: no report raised at a raw end offset `pos` or later can come first in block `block` -- its
 * offset (pos + offset_adjust >= pos - slack) lies past the entry's.  A tie on `to` is not past: a smaller id may win
 * it. */
__device__ __forceinline__ bool firstPast(const MaskOut &m, u32 block, u64 pos) {
    return (u64)firstTo(m, block) + m.slack < pos;
}

/* A stream-set mask pass over rows: a match of report id `id` that ends at `to` of group g's block.  An end inside
 * the look-behind was delivered by an earlier pass; any other sets its bit in the row that holds its last byte, the
 * row srRewriteKernel gives the same match's record. */
__device__ __forceinline__ void maskRowReport(const MaskOut &m, u32 id, u32 g, u64 to) {
    const StreamRowsMap &rm = m.rows;
    const u32 hl = rm.gHl[g];
    if (to <= hl) {
        return;
    }
    maskReport(m, id, rm.sorted[streamRowAt(rm.gFirst, rm.posOf, g, rm.gPos[g] + (to - 1 - hl))].y);
}

} // namespace

} // namespace hsb
#endif
