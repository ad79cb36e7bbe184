/*
 * scan_kernels.cu -- sm_90a scan kernels for the floating literal matcher:
 * first-stage shift-OR filter (FDR / Teddy / noodle tables), hash confirm and
 * the pure-literal rose program, all on the device.
 *
 * Replaces the reference's hwlmExec() and everything below it
 * (src/hwlm/hwlm.c:172-199 -> src/hwlm/noodle_engine.c, src/fdr/fdr.c,
 * src/fdr/teddy.c, src/fdr/fdr_confirm_runtime.h) together with the
 * per-literal callback chain roseCallback -> roseRunProgram_l
 * (src/rose/match.c:479-527, src/rose/program_runtime.c:3101-3522).
 *
 * Execution model (DESIGN.md section 3):
 *   - persistent grid, one CTA per SM; the first-stage tables are pinned in
 *     shared memory once per CTA;
 *   - the packed corpus is cut into fixed-size tiles regardless of block
 *     boundaries (the first stage is position-only; block membership is
 *     checked in the confirm stage); every warp owns a CONTIGUOUS run of
 *     tiles so the shift-OR state carries across tiles;
 *   - every lane loads its bytes straight from HBM into registers, a step or
 *     two ahead, with prefetch.global.L2 pfDist steps ahead;
 *   - three first stages, chosen by the host from the database:
 *       scanKernelWide (FK_BYTE32: noodle, 8-bucket Teddy): 32 bytes per lane
 *         and 1 KiB per warp iteration, one per-lane-replicated byte table;
 *       scanKernelPair (FK_PAIR32: FDR sets, fat Teddy with its buckets
 *         folded): two conflict-free class lookups and one pair lookup per byte;
 *       scanKernelGram (FK_GRAM4: large FDR sets): class 4-gram membership in
 *         a 1 Mbit shared-memory bitmap;
 *     a zero bit of the shift-OR state = candidate (bucket, end);
 *   - candidates (rare) go through a per-warp queue in shared memory, probe a
 *     bitmap over hashes of literal tails (shared memory, + a sparser second
 *     level in L2 for large sets), and the survivors are appended to a
 *     candidate list in HBM;
 *   - confirmKernel, launched after every scan, finishes the list: FDRConfirm
 *     hash -> LitInfo chain -> block lookup -> rose literal program -> 16-byte
 *     match record appended to a ring in HBM and, in multi-GPU runs, stored
 *     into every rank's exchange buffer over NVLink peer mappings (the scan IS
 *     the all-gather).
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.h"
#include "resolve.h"

namespace hsb {

namespace {

/* ---- PTX wrappers: shared-memory addresses, streaming loads.  The HSB_HOST_EMU
 * forms belong to the SIMT emulator of tests/emu (test infrastructure):
 * shared-memory "addresses" are offsets into the block's window. */
#ifdef HSB_HOST_EMU
__device__ __forceinline__ u32 smemAddr(const void *p) {
    return (u32)((const u8 *)p - hsb_emu::dynamicSmem());
}
__device__ __forceinline__ uint4 ldCs128(const u8 *p) { return *reinterpret_cast<const uint4 *>(p); }
__device__ __forceinline__ void prefetchL2(const void *) {}
#else
__device__ __forceinline__ u32 smemAddr(const void *p) {
    return (u32)__cvta_generic_to_shared(p);
}
/* volatile: keeps the load where it is written (ptxas otherwise sinks it next to
 * its first use and the prefetch is lost) */
__device__ __forceinline__ uint4 ldCs128(const u8 *p) {
    uint4 r;
    asm volatile("ld.global.cs.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void prefetchL2(const void *p) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
#endif

/* ---- read-only loads of the database image ------------------------------- */

__device__ __forceinline__ u32 ld32(const u8 *p) { return __ldg((const u32 *)p); }
__device__ __forceinline__ u64 ld64(const u8 *p) {
    const uint2 v = __ldg((const uint2 *)p);
    return ((u64)v.y << 32) | v.x;
}
__device__ __forceinline__ u8 ld8(const u8 *p) { return __ldg(p); }

/* ---- confirm stage -------------------------------------------------------- */

struct BlockRef {
    const u8 *base; /* first byte of the block */
    u32 len;
    u32 index;
    u32 hist;       /* stream sets: leading bytes that are look-behind (already scanned) */
    u64 toBase;     /* added to block-relative `to` in emitted records (stream offset) */
};

/* Which block holds corpus position g?  (Blocks are 16-byte aligned, sorted,
 * disjoint; gaps belong to no block.) */
__device__ bool findBlock(const ScanParams &p, u64 g, BlockRef *out) {
    if (g >= p.corpusBytes) {
        return false;
    }
    out->hist = 0;
    out->toBase = 0;
    if (p.streamPitch) {
        /* stream set: stream b's write sits at b * pitch + 16, its look-behind
         * (<= 7 bytes kept in HBM) right in front of it */
        const u32 b = (u32)(g / p.streamPitch);
        if (b >= p.nblocks) {
            return false;
        }
        const u32 hl = __ldg(p.streamHist + (size_t)b * 8 + 7);
        const u32 wl = p.uniformLen ? p.uniformLen : __ldg(p.blockLen + b);
        const u64 off = (u64)b * p.streamPitch + 16 - hl;
        if (g < off || g - off >= hl + wl) {
            return false;
        }
        out->base = p.corpus + off;
        out->len = hl + wl;
        out->index = b;
        out->hist = hl;
        out->toBase = __ldg(p.streamOffset + b) - hl;
        return true;
    }
    u32 b;
    if (p.uniformPitch) {
        b = (u32)(g / p.uniformPitch);
    } else {
        u32 lo = 0, hi = p.nblocks; /* largest b with off[b] <= g */
        while (hi - lo > 1) {
            const u32 mid = lo + ((hi - lo) >> 1);
            if (__ldg(p.blockOff + mid) <= g) {
                lo = mid;
            } else {
                hi = mid;
            }
        }
        b = lo;
    }
    if (b >= p.nblocks) {
        return false;
    }
    u64 off;
    u32 len;
    if (p.uniformPitch && p.uniformLen) { /* no table needed */
        off = (u64)b * p.uniformPitch;
        len = p.uniformLen;
    } else {
        off = __ldg(p.blockOff + b);
        len = __ldg(p.blockLen + b);
    }
    if (g < off || g - off >= len) {
        return false;
    }
    out->base = p.corpus + off;
    out->len = len;
    out->index = b;
    return true;
}

/* The confirm paths: CONF_PLAIN writes records, or sets the bits of a mask pass (p.mask.bits); CONF_ROWS_MASK is the
 * confirm kernel of a stream-set mask pass over rows (confirmRowsMaskKernel), whose blocks are the batch's groups;
 * CONF_FIRST is the confirm kernel of a first-match pass (confirmFirstKernel) */
enum { CONF_PLAIN = 0, CONF_ROWS_MASK = 1, CONF_FIRST = 2 };
template <int CONF> __device__ __forceinline__ void emitMatch(const ScanParams &p, u32 id, u32 block, u64 to) {
    if (CONF == CONF_ROWS_MASK) {
        maskRowReport(p.mask, id, block, to);
        return;
    }
    if (CONF == CONF_FIRST) {
        firstReport(p.mask, id, block, to); /* (no logical-key record: a database with combinations is refused) */
        return;
    }
    if (p.mask.bits) {
        maskReport(p.mask, id, block); /* (no logical-key record: a database with combinations is refused) */
        return;
    }
    const u32 i = atomicAdd(p.counters + CTR_MATCHES, 1u);
    if (i < p.outCap) {
        DevMatch m;
        m.id = id;
        m.block = block;
        m.to = to;
        *reinterpret_cast<uint4 *>(p.out + i) = *reinterpret_cast<const uint4 *>(&m);
    }
    if (p.nPeers && i < p.peerCap) {
        /* fused all-gather: the record goes straight into every rank's
         * exchange buffer (posted 16-byte stores over NVLink peer mappings) */
        DevMatch g = {id, block + p.blockBase, to};
        const size_t slot = (size_t)p.myRank * (p.peerCap + 1) + 1 + i;
#pragma unroll 1
        for (u32 r = 0; r < p.nPeers; r++) {
            *reinterpret_cast<uint4 *>(p.peers[r] + slot) = *reinterpret_cast<const uint4 *>(&g);
        }
    }
}

__device__ __forceinline__ u8 upperAscii(u8 c) {
    return (c >= 'a' && c <= 'z') ? (u8)(c - 0x20) : c;
}

/* CHECK_MED_LIT / CHECK_LONG_LIT, block mode: the lit_length bytes ending at
 * `to` must equal the stored literal, which is stored upper-cased for the
 * _NOCASE variants (src/rose/program_runtime.c:1883-2014). */
__device__ bool checkLiteral(const u8 *bc, const BlockRef &blk, u64 to, u32 litOff, u32 litLen,
                             bool nocase) {
    if (to < litLen) {
        return false;
    }
    const u8 *lit = bc + litOff;
    const u8 *d = blk.base + (to - litLen);
    for (u32 i = 0; i < litLen; i++) {
        u8 c = d[i];
        if (nocase) {
            c = upperAscii(c);
        }
        if (c != ld8(lit + i)) {
            return false;
        }
    }
    return true;
}

/* CHECK_MASK: 8 bytes at to+offset; byte lanes outside the block are ignored
 * (src/rose/program_runtime.c:644-726, src/rose/validate_mask.h:83-103). */
__device__ bool checkMask8(const BlockRef &blk, u64 to, u64 andM, u64 cmpM, u64 negM, s32 off) {
    const long long start = (long long)to + off;
    if (start < 0) {
        return false; /* "too early, fail": block mode has no history */
    }
    for (int i = 0; i < 8; i++) {
        const long long q = start + i;
        if (q < 0 || q >= (long long)blk.len) {
            continue;
        }
        const u8 d = blk.base[q];
        const u8 a = (u8)(andM >> (8 * i)), c = (u8)(cmpM >> (8 * i));
        const bool eq = ((d & a) ^ c) == 0;
        const bool neg = ((negM >> (8 * i)) & 0xff) != 0;
        if (eq == neg) {
            return false;
        }
    }
    return true;
}

/* CHECK_MASK_32 / CHECK_MASK_64: N bytes at to+offset, one negation BIT per byte; bytes
 * in the future are ignored, a window starting before the block fails
 * (src/rose/program_runtime.c:729-801 and :805-877, src/rose/validate_mask.h:106-153).
 * The masks are read from the instruction in the bytecode. */
__device__ bool checkMaskWide(const BlockRef &blk, u64 to, const u8 *andM, const u8 *cmpM, u64 negM, s32 off,
                              int nbytes) {
    const long long start = (long long)to + off;
    if (start < 0) {
        return false; /* "too early, fail": block mode has no history */
    }
    for (int i = 0; i < nbytes; i++) {
        const long long q = start + i;
        if (q >= (long long)blk.len) {
            break;
        }
        const bool ne = (blk.base[q] & __ldg(andM + i)) != __ldg(cmpM + i);
        if (ne != (bool)((negM >> i) & 1)) {
            return false;
        }
    }
    return true;
}

/* CHECK_BYTE (src/rose/program_runtime.c:600-641). */
__device__ bool checkByte(const BlockRef &blk, u64 to, u8 andM, u8 cmpM, u8 neg, s32 off) {
    const long long q = (long long)to + off;
    if (q < 0) {
        return false; /* "too early, fail" (no history in block mode) */
    }
    if (q >= (long long)blk.len) {
        return true;  /* in the future: passes */
    }
    const u8 c = blk.base[q];
    return !(((andM & c) != cmpM) ^ (neg != 0));
}

template <class T> __device__ __forceinline__ T loadInstr(const u8 *pc) {
    T t;
    const u32 *s = (const u32 *)pc; /* instructions are 8-byte aligned */
    u32 *d = (u32 *)&t;
#pragma unroll
    for (u32 i = 0; i < (sizeof(T) + 3) / 4; i++) {
        d[i] = __ldg(s + i);
    }
    return t;
}

/* Literal program at bytecode offset `prog` for a literal whose last byte is
 * block offset `end` (to = end + 1: lit_offset_adjust, src/rose/match.c:483).
 * The stateless part of roseRunProgram_l: exhaustion (CHECK_EXHAUSTED /
 * REPORT_EXHAUST) and dedupe (DEDUPE*) are order-dependent and are applied
 * when the records are ordered for delivery (host, DESIGN.md section 5); here
 * they pass. */
template <int CONF> __device__ void runProgram(const ScanParams &p, const BlockRef &blk, u32 prog, u64 to) {
    const u8 *pc = p.bc + prog;
#define NEXT(T) pc += HSB_ROUNDUP(sizeof(T), INSTR_ALIGN)
    for (int guard = 0; guard < 4096; guard++) {
        const u8 code = ld8(pc);
        switch (code) {
        case OP_END:
            return;
        case OP_CHECK_GROUPS: {
            const InstrCheckGroups in = loadInstr<InstrCheckGroups>(pc);
            if (!(in.groups & p.groups)) {
                return;
            }
            NEXT(InstrCheckGroups);
            break;
        }
        case OP_CHECK_MASK: {
            const InstrCheckMask in = loadInstr<InstrCheckMask>(pc);
            if (!checkMask8(blk, to, in.and_mask, in.cmp_mask, in.neg_mask, in.offset)) {
                pc += in.fail_jump;
            } else {
                NEXT(InstrCheckMask);
            }
            break;
        }
        case OP_CHECK_MASK_32: {
            const u32 neg = __ldg((const u32 *)(pc + offsetof(InstrCheckMask32, neg_mask)));
            const s32 off = (s32)__ldg((const u32 *)(pc + offsetof(InstrCheckMask32, offset)));
            if (!checkMaskWide(blk, to, pc + offsetof(InstrCheckMask32, and_mask),
                               pc + offsetof(InstrCheckMask32, cmp_mask), neg, off, 32)) {
                pc += __ldg((const u32 *)(pc + offsetof(InstrCheckMask32, fail_jump)));
            } else {
                NEXT(InstrCheckMask32);
            }
            break;
        }
        case OP_CHECK_MASK_64: {
            const u64 neg = __ldg((const u64 *)(pc + offsetof(InstrCheckMask64, neg_mask)));
            const s32 off = (s32)__ldg((const u32 *)(pc + offsetof(InstrCheckMask64, offset)));
            if (!checkMaskWide(blk, to, pc + offsetof(InstrCheckMask64, and_mask),
                               pc + offsetof(InstrCheckMask64, cmp_mask), neg, off, 64)) {
                pc += __ldg((const u32 *)(pc + offsetof(InstrCheckMask64, fail_jump)));
            } else {
                NEXT(InstrCheckMask64);
            }
            break;
        }
        case OP_CHECK_BYTE: {
            const InstrCheckByte in = loadInstr<InstrCheckByte>(pc);
            if (!checkByte(blk, to, in.and_mask, in.cmp_mask, in.negation, in.offset)) {
                pc += in.fail_jump;
            } else {
                NEXT(InstrCheckByte);
            }
            break;
        }
        case OP_CHECK_MED_LIT:
        case OP_CHECK_MED_LIT_NOCASE:
        case OP_CHECK_LONG_LIT:
        case OP_CHECK_LONG_LIT_NOCASE: {
            const InstrCheckLit in = loadInstr<InstrCheckLit>(pc);
            const bool nc = code == OP_CHECK_MED_LIT_NOCASE || code == OP_CHECK_LONG_LIT_NOCASE;
            if (!checkLiteral(p.bc, blk, to, in.lit_offset, in.lit_length, nc)) {
                pc += in.fail_jump;
            } else {
                NEXT(InstrCheckLit);
            }
            break;
        }
        case OP_CHECK_EXHAUSTED:
            NEXT(InstrCheckExhausted);
            break;
        case OP_DEDUPE:
            NEXT(InstrDedupe);
            break;
        case OP_REPORT: {
            const InstrReport in = loadInstr<InstrReport>(pc);
            emitMatch<CONF>(p, in.onmatch, blk.index, blk.toBase + to + in.offset_adjust);
            NEXT(InstrReport);
            break;
        }
        case OP_REPORT_EXHAUST: {
            const InstrReportExhaust in = loadInstr<InstrReportExhaust>(pc);
            emitMatch<CONF>(p, in.onmatch, blk.index, blk.toBase + to + in.offset_adjust);
            NEXT(InstrReportExhaust);
            break;
        }
        case OP_DEDUPE_AND_REPORT: {
            const InstrDedupeAndReport in = loadInstr<InstrDedupeAndReport>(pc);
            emitMatch<CONF>(p, in.onmatch, blk.index, blk.toBase + to + in.offset_adjust);
            NEXT(InstrDedupeAndReport);
            break;
        }
        case OP_FINAL_REPORT: {
            const InstrFinalReport in = loadInstr<InstrFinalReport>(pc);
            emitMatch<CONF>(p, in.onmatch, blk.index, blk.toBase + to + in.offset_adjust);
            return;
        }
        case OP_SQUASH_GROUPS: /* group squashing only prunes work */
            NEXT(InstrSquashGroups);
            break;
        case OP_CLEAR_WORK_DONE:
            pc += INSTR_ALIGN;
            break;
        case OP_INCLUDED_JUMP: /* the child literal is confirmed on its own */
            NEXT(InstrIncludedJump);
            break;
        case OP_SET_LOGICAL: {
            /* a logical-key record (id = lkey, bit 63 of `to` set): the combinations are
             * evaluated on the host when the records are ordered (postprocessCombinations) */
            const InstrSetLogical in = loadInstr<InstrSetLogical>(pc);
            emitMatch<CONF>(p, in.lkey, blk.index, (blk.toBase + to + in.offset_adjust) | (1ull << 63));
            NEXT(InstrSetLogical);
            break;
        }
        case OP_SET_COMBINATION: /* follows from the lkey on the host */
            NEXT(InstrSetCombination);
            break;
        case OP_FLUSH_COMBINATION:
            NEXT(InstrFlushCombination);
            break;
        case OP_CATCH_UP: /* (databases with an outfix only: the host orders its records among these) */
            NEXT(InstrCatchUp);
            break;
        default:
            atomicExch(p.counters + CTR_ERROR, (u32)ERR_BAD_OPCODE);
            return;
        }
    }
#undef NEXT
    atomicExch(p.counters + CTR_ERROR, (u32)ERR_BAD_OPCODE);
}

/* Second stage for one candidate (bucket, corpus position g of the last
 * byte); confVal = little-endian u64 of the bytes [g-7, g].  Restates
 * confWithBit (src/fdr/fdr_confirm_runtime.h:43-102) minus the callback
 * feedback: bytes before the block start never decide (every accepted
 * literal lies inside the block, item 3 of SURVEY.md A.1). */
template <int CONF> __device__ void confirmFdr(const ScanParams &p, u32 bucket, u64 g, u64 confVal, u32 *nconf) {
    const u8 *confBase = p.bc + p.confOff;
    const u32 cf = ld32(confBase + 4 * bucket);
    if (!cf) {
        return;
    }
    const u8 *fc = confBase + cf; /* struct FDRConfirm */
    if (!(ld64(fc + 24) & p.groups)) {
        return;
    }
    const u64 andmsk = ld64(fc + 0), mult = ld64(fc + 8);
    const u32 nBits = ld32(fc + 16);
    const u32 c = (u32)(((confVal & andmsk) * mult) >> (64 - nBits));
    const u32 start = ld32(fc + sizeof(FDRConfirm) + 4 * c);
    if (!start) {
        return;
    }
    const u8 *li = fc + start; /* struct LitInfo chain */
    bool haveBlock = false, inBlock = false;
    BlockRef blk;
    for (;;) {
        const u64 v = ld64(li + 0), msk = ld64(li + 8);
        const u32 tail = ld32(li + 28); /* size | flags << 8 | next << 16 */
        if ((confVal & msk) == v && (ld64(li + 16) & p.groups)) {
            if (!haveBlock) {
                inBlock = findBlock(p, g, &blk);
                haveBlock = true;
            }
            if (inBlock) {
                const u64 end = (u64)(p.corpus + g - blk.base);
                if (CONF == CONF_FIRST && firstPast(p.mask, blk.index, end + 1)) {
                    break; /* no report of a literal ending here can come before the block's entry */
                }
                if ((tail & 0xff) <= end + 1 && end >= blk.hist) { /* ends inside the write */
                    (*nconf)++;
                    runProgram<CONF>(p, blk, ld32(li + 24), end + 1);
                }
            }
        }
        if (!((tail >> 16) & 0xff)) {
            break;
        }
        li += sizeof(LitInfo);
    }
}

/* Noodle second stage (src/hwlm/noodle_engine.c:114-141): the msk_len bytes
 * ending at g, first byte in the low lane, under msk must equal cmp. */
template <int CONF> __device__ void confirmNoodle(const ScanParams &p, u64 g, u64 confVal, u32 *nconf) {
    const u8 *n = p.bc + p.engineOff; /* struct noodTable */
    const u32 mskLen = ld8(n + 24);
    const u64 msk = ld64(n + 8), cmp = ld64(n + 16);
    const u64 v = mskLen >= 8 ? confVal : confVal >> (8 * (8 - mskLen));
    if ((v & msk) != cmp) {
        return;
    }
    BlockRef blk;
    if (!findBlock(p, g, &blk)) {
        return;
    }
    const u64 end = (u64)(p.corpus + g - blk.base);
    if (mskLen > end + 1 || end < blk.hist) {
        return;
    }
    if (CONF == CONF_FIRST && firstPast(p.mask, blk.index, end + 1)) {
        return; /* no report of the literal can come before the block's entry */
    }
    (*nconf)++;
    runProgram<CONF>(p, blk, ld32(n + 0), end + 1);
}

/* ---- first stage ----------------------------------------------------------- */

#ifdef HSB_HOST_EMU
__device__ __forceinline__ u32 lds32(u32 addr) {
    u32 v;
    memcpy(&v, hsb_emu::dynamicSmem() + addr, 4);
    return v;
}
__device__ __forceinline__ uint2 lds64(u32 addr) {
    uint2 v;
    memcpy(&v, hsb_emu::dynamicSmem() + addr, 8);
    return v;
}
__device__ __forceinline__ uint4 lds128(u32 addr) {
    uint4 v;
    memcpy(&v, hsb_emu::dynamicSmem() + addr, 16);
    return v;
}
__device__ __forceinline__ void sts128(u32 addr, u32 x, u32 y, u32 z, u32 w) {
    const u32 v[4] = {x, y, z, w};
    memcpy(hsb_emu::dynamicSmem() + addr, v, 16);
}
__device__ __forceinline__ void sts64(u32 addr, u32 x, u32 y) {
    const u32 v[2] = {x, y};
    memcpy(hsb_emu::dynamicSmem() + addr, v, 8);
}
__device__ __forceinline__ void sts32(u32 addr, u32 x) { memcpy(hsb_emu::dynamicSmem() + addr, &x, 4); }
#else
__device__ __forceinline__ u32 lds32(u32 addr) {
    u32 v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint2 lds64(u32 addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint4 lds128(u32 addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(u32 addr, u32 x, u32 y, u32 z, u32 w) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w)
                 : "memory");
}
__device__ __forceinline__ void sts64(u32 addr, u32 x, u32 y) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(addr), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void sts32(u32 addr, u32 x) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(x) : "memory");
}
#endif

/* OR the 128-bit stream E[0..3] (one entry per word of the lane, all at the
 * same in-word position) into a[] at byte offset O (0..3): one funnel shift
 * per output word instead of two shifts per entry. */
template <int O> __device__ __forceinline__ void orStream(u32 (&a)[6], const u32 (&E)[4]) {
    if constexpr (O == 0) {
#pragma unroll
        for (int k = 0; k < 4; k++) a[k] |= E[k];
    } else {
        a[0] |= E[0] << (8 * O);
#pragma unroll
        for (int k = 1; k < 4; k++) a[k] |= __funnelshift_l(E[k - 1], E[k], 8 * O);
        a[4] |= E[3] >> (32 - 8 * O);
    }
}

/* Shift-OR contributions of one lane's 16 positions through the FK_BYTE32 table.
 * a[0..3]: bytes for the lane's own 16 end positions (bit set = bucket
 * impossible); a[4]: overflow that belongs to the NEXT lane's first positions.
 * An entry read at position x applies to end positions x .. x+3. */
__device__ __forceinline__ void laneFilter(const u32 (&w)[5], u32 tabAddr, u32 laneOff, u32 (&a)[6]) {
#pragma unroll
    for (int i = 0; i < 6; i++) {
        a[i] = 0;
    }
    /* gather the entries of in-word position r for all four words, then merge
     * the stream with funnel shifts */
#pragma unroll
    for (int r = 0; r < 4; r++) {
        u32 E[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            /* row b of the table is 256 bytes: lane l's copy of the entry at
             * l * 4, so the row offset b << 8 | l << 2 is ONE byte permute of
             * (word, laneOff) and every lookup is bank-conflict free */
            E[k] = lds32(tabAddr + __byte_perm(w[k], laneOff, 0x5504 + (r << 4)));
        }
        if (r == 0) orStream<0>(a, E);
        if (r == 1) orStream<1>(a, E);
        if (r == 2) orStream<2>(a, E);
        if (r == 3) orStream<3>(a, E);
    }
}

/* ---- candidate handling (rare path) ------------------------------------------- */

/* little-endian u64 of corpus bytes [g-7, g]; positions before the corpus
 * read as zero (a wrapped caller buffer has nothing readable before it), and so
 * do positions past its readable end: a first-stage candidate can sit in the
 * padding after the last block (it is rejected later, by the block lookup) */
__device__ __forceinline__ u64 confValAt(const ScanParams &p, u64 g) {
    if (g < 11 || g + 5 > p.readableEnd) { /* rare: the aligned 12-byte window would leave the buffer */
        u64 v = 0;
        for (int z = 0; z < 8; z++) {
            const long long q = (long long)g - 7 + z;
            if (q >= 0 && (u64)q < p.readableEnd) {
                v |= (u64)__ldg(p.corpus + q) << (8 * z);
            }
        }
        return v;
    }
    const u8 *a = p.corpus + g - 7;
    const u32 mis = (u32)((uintptr_t)a & 3);
    const u32 *aw = reinterpret_cast<const u32 *>(a - mis);
    const u32 w0 = __ldg(aw), w1 = __ldg(aw + 1), w2 = __ldg(aw + 2);
    const u32 lo = __funnelshift_r(w0, w1, 8 * mis);
    const u32 hi = __funnelshift_r(w1, w2, 8 * mis);
    return ((u64)hi << 32) | lo;
}

/* Candidates of one lane's 16 bytes: c[k] has a set bit per (bucket, byte) of word
 * k, w[k] is the word itself and `pw` the word before it.  Per candidate byte: hash
 * the last keyBytes bytes into the prefilter bitmap (shared memory); survivors are
 * appended to the candidate list (second half of the record ring) for confirmKernel. */
__device__ __forceinline__ void laneCandidates(const ScanParams &p, u32 bitmapAddr, u32 c0, u32 c1, u32 c2,
                                               u32 c3, u32 w0, u32 w1, u32 w2, u32 w3, u32 pw, u64 g0,
                                               u32 *stats) {
    /* 16-bit map of bytes that carry a candidate */
    u32 cm = 0;
    {
        const u32 n[4] = {c0, c1, c2, c3};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            u32 t = n[k] | (n[k] >> 4);
            t |= t >> 2;
            t |= t >> 1;
            t &= 0x01010101u;
            cm |= ((t * 0x01020408u) >> 24) << (4 * k);
        }
    }
    while (cm) {
        const u32 x = __ffs(cm) - 1;
        cm &= cm - 1;
        const u32 k = x >> 2, q = x & 3;
        const u32 cur = k == 0 ? w0 : k == 1 ? w1 : k == 2 ? w2 : w3;
        const u32 prv = k == 0 ? pw : k == 1 ? w0 : k == 2 ? w1 : w2;
        const u32 b0 = k == 0 ? c0 : k == 1 ? c1 : k == 2 ? c2 : c3;
        const u32 buckets = (b0 >> (8 * q)) & 0xff;
        stats[0]++;
        if (p.bitmapBytes) {
            /* the 4 bytes ending at x, then the last keyBytes of them */
            const u32 last4 = q == 3 ? cur : __funnelshift_r(prv, cur, 8 * (q + 1));
            const u32 key = last4 >> (8 * (4 - p.keyBytes));
            const u32 hsh = (key * 0x9E3779B1u) >> p.bitmapShift;
            if (!((lds32(bitmapAddr + ((hsh >> 5) << 2)) >> (hsh & 31)) & 1)) {
                continue; /* no literal of any bucket ends here */
            }
            if (p.bitmap2Shift) {
                /* large sets overload the shared-memory bitmap: a second, much
                 * sparser one lives in HBM and stays L2-resident */
                const u32 h2 = (key * 0x85EBCA6Bu) >> p.bitmap2Shift;
                if (!((__ldg(p.bitmap2 + (h2 >> 5)) >> (h2 & 31)) & 1)) {
                    continue;
                }
            }
        }
        stats[1]++;
        const u32 i = atomicAdd(p.counters + CTR_CANDQ, 1u);
        if (i < p.outCap) {
            DevCand cnd;
            cnd.g = g0 + x;
            cnd.buckets = buckets;
            cnd.pad = 0;
            *reinterpret_cast<uint4 *>(reinterpret_cast<DevCand *>(p.out + p.outCap) + i) =
                *reinterpret_cast<const uint4 *>(&cnd);
        }
    }
}

/* State entering a run of tiles: every lane evaluates the 16 bytes before the
 * run (v, then w4 = the run's first word) as if it were "lane -1" and keeps only
 * the overflow. */
__device__ __forceinline__ u32 haloStep(const uint4 v, u32 w4, u32 tabAddr, u32 laneOff) {
    const u32 w[5] = {v.x, v.y, v.z, v.w, w4};
    u32 a[6];
    laneFilter(w, tabAddr, laneOff, a);
    return a[4];
}

/* ---- wide-step kernel (FK_BYTE32) ------------------------------------------------
 *
 * Every lane owns 32 CONTIGUOUS bytes (8 words) per iteration and the warp 1 KiB:
 * the per-step overhead (carry shuffle, vote, loop, prefetch) is paid once per 1 KiB
 * instead of once per 512 bytes and the overflow into the next lane once per 32
 * bytes.  Candidates go through the per-warp queue (entry = 8 candidate words + the
 * number of the 32-byte chunk). */
enum { BYTE_TABLE_BYTES = 256 * 256 }; /* 256 rows x 32 lane copies (+ 128 B unused) */

struct WideQueue {
    static constexpr u32 BYTES = 48;
    static constexpr u32 SLOTS = 64;
    static constexpr u32 RUN_START = BYTES * SLOTS;
    static constexpr u32 WARP_BYTES = RUN_START + 16;
};

template <int O> __device__ __forceinline__ void orStreamWide(u32 (&a)[9], const u32 (&E)[8]) {
    if constexpr (O == 0) {
#pragma unroll
        for (int k = 0; k < 8; k++) a[k] |= E[k];
    } else if constexpr (O == 4) {
#pragma unroll
        for (int k = 0; k < 8; k++) a[k + 1] |= E[k];
    } else {
        a[0] |= E[0] << (8 * O);
#pragma unroll
        for (int k = 1; k < 8; k++) a[k] |= __funnelshift_l(E[k - 1], E[k], 8 * O);
        a[8] |= E[7] >> (32 - 8 * O);
    }
}

/* a[0..7]: the lane's own 32 end positions, a[8]: overflow into the next lane */
__device__ __forceinline__ void laneFilterWide(const u32 (&w)[8], u32 tabAddr, u32 laneOff, u32 (&a)[9]) {
#pragma unroll
    for (int i = 0; i < 9; i++) {
        a[i] = 0;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
        u32 E[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            E[k] = lds32(tabAddr + __byte_perm(w[k], laneOff, 0x5504 + (r << 4)));
        }
        if (r == 0) orStreamWide<0>(a, E);
        if (r == 1) orStreamWide<1>(a, E);
        if (r == 2) orStreamWide<2>(a, E);
        if (r == 3) orStreamWide<3>(a, E);
    }
}

/* One queue entry per lane: the two 16-byte halves of its 32-byte chunk, bytes read
 * back from L2, through laneCandidates. */
__device__ __forceinline__ void drainWide(const ScanParams &p, u32 bitmapAddr, u32 qAddr, u32 first, u32 count,
                                          u32 lane, u32 *stats) {
    if (lane >= count) {
        return;
    }
    const uint2 rs = lds64(qAddr + WideQueue::RUN_START);
    const u64 runStart = ((u64)rs.y << 32) | rs.x;
    const u32 e = qAddr + (first + lane) * WideQueue::BYTES;
    const uint4 c0 = lds128(e), c1 = lds128(e + 16);
    const u64 g0 = runStart + (u64)lds32(e + 32) * 32;
    uint4 v0 = make_uint4(0, 0, 0, 0), v1 = make_uint4(0, 0, 0, 0);
    if (g0 + 16 <= p.readableEnd) {
        v0 = __ldg(reinterpret_cast<const uint4 *>(p.corpus + g0));
    }
    if (g0 + 32 <= p.readableEnd) {
        v1 = __ldg(reinterpret_cast<const uint4 *>(p.corpus + g0 + 16));
    }
    const u32 pw = g0 ? __ldg(reinterpret_cast<const u32 *>(p.corpus + g0 - 4)) : 0u;
    if (c0.x | c0.y | c0.z | c0.w) {
        laneCandidates(p, bitmapAddr, c0.x, c0.y, c0.z, c0.w, v0.x, v0.y, v0.z, v0.w, pw, g0, stats);
    }
    if (c1.x | c1.y | c1.z | c1.w) {
        laneCandidates(p, bitmapAddr, c1.x, c1.y, c1.z, c1.w, v1.x, v1.y, v1.z, v1.w, v0.w, g0 + 16, stats);
    }
}

template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1) scanKernelWide(const HSB_GRID_CONSTANT ScanParams p) {
    HSB_DYNAMIC_SMEM(smem);
    const u32 lane = threadIdx.x & 31;
    const u32 warp = threadIdx.x >> 5;
    const u32 nwarps = blockDim.x >> 5;

    {
        const u32 *g = reinterpret_cast<const u32 *>(p.table);
        u32 *s = reinterpret_cast<u32 *>(smem);
        for (u32 i = threadIdx.x; i < 256 * 64; i += blockDim.x) {
            s[i] = ((i >> 5) & 1) ? 0xffffffffu : __ldg(g + (i >> 6));
        }
    }
    /* second-stage prefilter: one bit per hash of a literal's last bytes */
    if (p.bitmapBytes) {
        const uint4 *g = reinterpret_cast<const uint4 *>(p.bitmap);
        uint4 *sdst = reinterpret_cast<uint4 *>(smem + BYTE_TABLE_BYTES);
        for (u32 i = threadIdx.x; i < p.bitmapBytes / 16; i += blockDim.x) {
            sdst[i] = __ldg(g + i);
        }
    }
    __syncthreads();

    const u32 tabAddr = smemAddr(smem);
    const u32 bitmapAddr = tabAddr + BYTE_TABLE_BYTES;
    const u32 laneOff = lane * 4; /* the lane's column of a table row */
    const u32 qAddr = bitmapAddr + p.bitmapBytes + warp * WideQueue::WARP_BYTES;

    /* this warp's contiguous run of tiles (tileBytes is a multiple of 1024 here) */
    const u32 gwarp = blockIdx.x * nwarps + warp;
    const u32 totalWarps = gridDim.x * nwarps;
    const u32 q = p.ntiles / totalWarps, rem = p.ntiles % totalWarps;
    const u32 myCount = q + (gwarp < rem ? 1u : 0u);
    const u32 myFirst = p.tileFirst + gwarp * q + min(gwarp, rem);
    if (myCount == 0) {
        return;
    }
    const u64 runStart = (u64)myFirst * p.tileBytes;
    u64 runEnd = runStart + (u64)myCount * p.tileBytes;
    if (runEnd > p.corpusBytes) {
        runEnd = p.corpusBytes;
    }
    const u32 niter = (u32)((runEnd - runStart + 1023) >> 10);
    const u8 *base = p.corpus + runStart + lane * 32;
    const u64 lanePos = runStart + lane * 32;
    if (lane == 0) {
        sts64(qAddr + WideQueue::RUN_START, (u32)runStart, (u32)(runStart >> 32));
    }

    u32 carry = 0; /* lane 31's overflow of the previous iteration */
    u32 stats[2] = {0, 0}; /* candidates, prefilter passes */
    u32 qn = 0;

    auto load = [&](u32 it, uint4 &lo, uint4 &hi) {
        const u64 pos = lanePos + (u64)it * 1024;
        lo = make_uint4(0, 0, 0, 0);
        hi = make_uint4(0, 0, 0, 0);
        const u8 *q0 = base + (size_t)it * 1024;
        if (pos + 32 <= p.readableEnd) {
            lo = ldCs128(q0);
            hi = ldCs128(q0 + 16);
        } else if (pos + 16 <= p.readableEnd) {
            lo = ldCs128(q0);
        }
    };
    const u32 pfDist = p.pfDist; /* in 1 KiB iterations */
    uint4 nlo, nhi;
    load(0, nlo, nhi);
    if (runStart != 0) {
        /* only the 4 bytes before the run (and its first word) reach into it */
        const uint4 hv = __ldg(reinterpret_cast<const uint4 *>(p.corpus + runStart - 16));
        const u32 first = __shfl_sync(0xffffffffu, nlo.x, 0);
        carry = haloStep(hv, first, tabAddr, laneOff);
    }
    /* one iteration; `fast` (every iteration but the last ones of the corpus): the
     * load of iteration it + 1 needs no bounds check because that whole KiB is
     * readable for every lane */
    auto iteration = [&](const u32 it, const bool fast) {
        const uint4 lo = nlo, hi = nhi;
        if (fast) {
            const u8 *q0 = base + (size_t)(it + 1) * 1024;
            nlo = ldCs128(q0);
            nhi = ldCs128(q0 + 16);
        } else {
            load(it + 1, nlo, nhi);
        }
        if ((lane & 3) == 0) {
            const u64 pos = lanePos + (u64)(it + pfDist) * 1024;
            if (pos < p.readableEnd) {
                prefetchL2(p.corpus + pos);
            }
        }
        const u32 w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        u32 a[9];
        laneFilterWide(w, tabAddr, laneOff, a);
        {
            u32 in = __shfl_sync(0xffffffffu, a[8], (lane + 31) & 31);
            if (lane == 0) {
                const u32 next = in;
                in = carry;
                carry = next;
            }
            a[0] |= in;
        }
        u32 any = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            a[k] = ~a[k];
            any |= a[k];
        }
        const u32 bal = __ballot_sync(0xffffffffu, any != 0);
        if (bal) {
            if (any) {
                const u32 e = qAddr + (qn + __popc(bal & ((1u << lane) - 1))) * WideQueue::BYTES;
                sts128(e, a[0], a[1], a[2], a[3]);
                sts128(e + 16, a[4], a[5], a[6], a[7]);
                sts32(e + 32, it * 32 + lane);
            }
            qn += __popc(bal);
            if (qn >= 32) {
                __syncwarp();
                qn -= 32;
                drainWide(p, bitmapAddr, qAddr, qn, 32, lane, stats);
                __syncwarp();
            }
        }
    };
    const u64 readableIters = (p.readableEnd - runStart) >> 10;
    const u32 nFast = readableIters >= (u64)niter + 1 ? niter : (readableIters ? (u32)readableIters - 1 : 0);
    u32 it = 0;
#pragma unroll 1
    for (; it < nFast; it++) {
        iteration(it, true);
    }
#pragma unroll 1
    for (; it < niter; it++) {
        iteration(it, false);
    }
    if (qn) {
        __syncwarp();
        drainWide(p, bitmapAddr, qAddr, 0, qn, lane, stats);
    }
    if (stats[0]) {
        atomicAdd(p.counters + CTR_CANDIDATES, stats[0]);
    }
    if (stats[1]) {
        atomicAdd(p.counters + CTR_PREFILTER_PASS, stats[1]);
    }
}

/* ---- class-pair kernel (FK_PAIR32): conflict-free two-byte first stage -------------
 *
 * An FDR hash lookup costs ~3.3 shared-memory wavefronts (random 4-byte gather of
 * 32 lanes into 32 banks; replicas only help once every lane has its own copy).
 * A copy per lane needs a table of <= 1024 entries, i.e. a 10-bit key for the two
 * bytes: each byte is first mapped to a 5-bit CLASS by a per-lane byte table
 * (conflict free, like the Teddy rows), two classes index a per-lane pair table
 * (conflict free): 2 wavefronts per input byte instead of 3.3, for a candidate
 * rate of the same order (the classes are chosen for the literal set on the host:
 * bytes that no literal uses share one class, api_device.cu buildPairTables).
 *
 *   class row b (256 B): [lane l: c0(b) << 7 | c1(b) << 12 | l << 2] x 32 | 128 B of the
 *                        first-level prefilter bitmap (32 KB in the 256 rows' upper halves)
 *   pair row (c1 << 5 | c0) (128 B): [u32 entry: 4 slots x 8 buckets] x 32 lanes
 *
 * so the pair address is ONE logic op of the two class words and every lookup is
 * PRMT/LOP3 + LDS.  A sample is keyed (c0(first byte), c1(second byte)); entry byte i
 * says which buckets cannot END i + SB bytes after the FIRST byte (SB = slot base: 1 when
 * every literal has at least two bytes, so that all four slots see both bytes of a pair).
 * The sample is placed so that its entry applies to the end positions x .. x + 3: SB = 1
 * keys x by the bytes (x - 1, x) -- one class lookup per byte of the lane, the class word
 * of the byte before it comes from the left neighbour --, SB = 0 by (x, x + 1).
 * Candidates: per-warp queue -> prefilter bitmaps -> candidate list in HBM ->
 * confirmKernel (the hot kernel carries no confirm code). */

struct PairQueue {
    static constexpr u32 SLOTS = 64;                      /* < 32 pending + <= 32 appended per step */
    static constexpr u32 CHUNK = 16 * SLOTS;              /* u32 chunk[SLOTS] after uint4 cand[SLOTS] */
    static constexpr u32 RUN_START = CHUNK + 4 * SLOTS;   /* u64: corpus position of the run's chunk 0 */
    static constexpr u32 WARP_BYTES = RUN_START + 16;
};
enum { PAIR_CLASS_BYTES = 256 * 256, PAIR_TABLE_BYTES = 1024 * 128 };

/* Row offset in the pair table: l << 2 | c0 << 7 from the first byte's class word,
 * c1 << 12 from the second's -- bit-field select (a & 0xfff) | (b & ~0xfff), ONE
 * LOP3 (left to itself the compiler emits and / and / add3). */
__device__ __forceinline__ u32 pairIndex(u32 a, u32 b) {
#ifdef HSB_HOST_EMU
    return (a & 0xfffu) | (b & ~0xfffu);
#else
    u32 d;
    asm("lop3.b32 %0, %1, %2, 0xfff, 0xE4;" : "=r"(d) : "r"(a), "r"(b));
    return d;
#endif
}

/* Class words of the 16 bytes of v into E[O .. O + 15] (the lane's own copies: row
 * offset byte << 8 | laneOff, conflict free). */
template <int O>
__device__ __forceinline__ void laneClasses(const uint4 v, u32 clsAddr, u32 laneOff, u32 (&E)[17]) {
    const u32 w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            E[O + 4 * k + r] = lds32(clsAddr + __byte_perm(w[k], laneOff, 0x5504 + (r << 4)));
        }
    }
}

/* Shift-OR contributions of one lane's 16 positions from the class words E[0..16] of 17
 * consecutive bytes: sample j keyed (E[j], E[j + 1]) applies to the lane's end positions
 * j .. j + 3 (SB = 1: E[0] is the byte before the lane; SB = 0: E[16] the byte after it).
 * a[0..3]: own end positions, a[4]: overflow into the next lane (bit set = bucket
 * impossible).  The pair lookups are conflict free as long as the lanes' first operands
 * carry lane fields that are a permutation of 0..31: E[0] of SB = 1 is the left
 * neighbour's word, a rotation by one. */
__device__ __forceinline__ void pairFilter(const u32 (&E)[17], u32 clsAddr, u32 (&a)[6]) {
#pragma unroll
    for (int i = 0; i < 6; i++) {
        a[i] = 0;
    }
    const u32 pairAddr = clsAddr + PAIR_CLASS_BYTES;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        u32 P[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            /* lane << 2 | c0 << 7 from the first byte's word, c1 << 12 from the second's */
            P[k] = lds32(pairAddr + pairIndex(E[4 * k + r], E[4 * k + r + 1]));
        }
        if (r == 0) orStream<0>(a, P);
        if (r == 1) orStream<1>(a, P);
        if (r == 2) orStream<2>(a, P);
        if (r == 3) orStream<3>(a, P);
    }
}

/* First-level bitmap word of the class-pair kernel: index = mulhi(key * K, bits);
 * word i lives in class row i >> 5 at byte 128 + 4 * (i & 31). */
__device__ __forceinline__ bool pairBitmapTest(const ScanParams &p, u32 bitmapAddr, u32 key) {
    const u32 h = __umulhi(key * 0x9E3779B1u, p.bitmapBits);
    const u32 wi = h >> 5;
    return (lds32(bitmapAddr + ((wi >> 5) << 8) + ((wi & 31u) << 2)) >> (h & 31)) & 1;
}

/* One queue entry per lane: the lane's candidate bytes go through the prefilter
 * bitmaps; survivors are appended to the candidate list in HBM (confirmKernel). */
__device__ HSB_NOINLINE void drainPair(const ScanParams &p, u32 bitmapAddr, u32 qAddr, u32 first,
                                       u32 count, u32 lane, u32 *stats) {
    if (lane >= count) {
        return;
    }
    const uint2 rs = lds64(qAddr + PairQueue::RUN_START);
    const u64 runStart = ((u64)rs.y << 32) | rs.x;
    const uint4 c = lds128(qAddr + (first + lane) * 16);
    const u64 g0 = runStart + (u64)lds32(qAddr + PairQueue::CHUNK + (first + lane) * 4) * 16;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (g0 + 16 <= p.readableEnd) {
        v = __ldg(reinterpret_cast<const uint4 *>(p.corpus + g0));
    }
    const u32 pw = g0 ? __ldg(reinterpret_cast<const u32 *>(p.corpus + g0 - 4)) : 0u;
    const u32 cw[4] = {c.x, c.y, c.z, c.w};
    const u32 w[5] = {pw, v.x, v.y, v.z, v.w};
    const u32 keyShift = 8 * (4 - p.keyBytes);
    u32 ncand = 0, npass = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        u32 m = cw[k];
        while (m) { /* one candidate byte (8 bucket bits) of word k per iteration */
            const u32 q = (u32)(__ffs(m) - 1) >> 3;
            const u32 buckets = (m >> (8 * q)) & 0xffu;
            m &= ~(0xffu << (8 * q));
            ncand++;
            if (p.bitmapBytes) {
                /* the 4 bytes ending at byte q of word k, then the last keyBytes of them */
                const u32 last4 = __funnelshift_rc(w[k], w[k + 1], 8 * (q + 1));
                const u32 key = last4 >> keyShift;
                if (!pairBitmapTest(p, bitmapAddr, key)) {
                    continue; /* no literal of any bucket ends here */
                }
                if (p.bitmap2Shift) {
                    const u32 h2 = (key * 0x85EBCA6Bu) >> p.bitmap2Shift;
                    if (!((__ldg(p.bitmap2 + (h2 >> 5)) >> (h2 & 31)) & 1)) {
                        continue;
                    }
                }
            }
            npass++;
            const u32 i = atomicAdd(p.counters + CTR_CANDQ, 1u);
            if (i < p.outCap) {
                DevCand cnd;
                cnd.g = g0 + 4 * k + q;
                cnd.buckets = buckets;
                cnd.pad = 0;
                *reinterpret_cast<uint4 *>(reinterpret_cast<DevCand *>(p.out + p.outCap) + i) =
                    *reinterpret_cast<const uint4 *>(&cnd);
            }
        }
    }
    stats[0] += ncand;
    stats[1] += npass;
}

/* Word-entry drains (heavy pair kernel, 4-gram kernel): every lane holds up to four
 * survivors {position, buckets[q] != 0}.  ONE atomicAdd per warp reserves their slots in
 * the candidate list (ballot prefix per round), instead of one same-address atomic -- and
 * one dependent L2 round trip -- per candidate. */
__device__ __forceinline__ void appendWordCandidates(const ScanParams &p, u64 g0, const u32 (&bk)[4], u32 lane) {
    const u32 full = 0xffffffffu;
    const u32 b0 = __ballot_sync(full, bk[0] != 0), b1 = __ballot_sync(full, bk[1] != 0);
    const u32 b2 = __ballot_sync(full, bk[2] != 0), b3 = __ballot_sync(full, bk[3] != 0);
    const u32 o1 = __popc(b0), o2 = o1 + __popc(b1), o3 = o2 + __popc(b2), total = o3 + __popc(b3);
    if (total == 0) {
        return;
    }
    u32 base = 0;
    if (lane == 0) {
        base = atomicAdd(p.counters + CTR_CANDQ, total);
    }
    base = __shfl_sync(full, base, 0);
    const u32 below = (1u << lane) - 1;
    const u32 idx[4] = {base + __popc(b0 & below), base + o1 + __popc(b1 & below), base + o2 + __popc(b2 & below),
                        base + o3 + __popc(b3 & below)};
    DevCand *const list = reinterpret_cast<DevCand *>(p.out + p.outCap);
#pragma unroll
    for (int q = 0; q < 4; q++) {
        if (bk[q] && idx[q] < p.outCap) {
            DevCand cnd;
            cnd.g = g0 + q;
            cnd.buckets = bk[q];
            cnd.pad = 0;
            *reinterpret_cast<uint4 *>(list + idx[q]) = *reinterpret_cast<const uint4 *>(&cnd);
        }
    }
}

/* Heavy variant (large / saturating sets: tens of candidates per 512-byte step).  A queue
 * entry is ONE WORD of one lane with at least one candidate byte: {offset of the word in
 * the warp's run, its candidate bits, the word before it, the word} -- the bytes travel
 * with the entry, so the drain needs no corpus read.  The four bytes of the word are
 * tested in four static rounds (an entry holds 1.1 candidates on average): the shared-
 * memory probes, then ALL second-level probes in flight together, then one reservation. */
__device__ HSB_NOINLINE void drainPairWords(const ScanParams &p, u32 bitmapAddr, u32 qAddr, u32 first,
                                            u32 count, u32 lane, u32 *stats) {
    const uint2 rs = lds64(qAddr + PairQueue::RUN_START);
    const u64 runStart = ((u64)rs.y << 32) | rs.x;
    uint4 e = make_uint4(0, 0, 0, 0); /* x = offset, y = candidate bits, z = previous word, w = word */
    if (lane < count) {
        e = lds128(qAddr + (first + lane) * 16);
    }
    const u32 keyShift = 8 * (4 - p.keyBytes);
    u32 bk[4], key[4];
    u32 ncand = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        bk[q] = (e.y >> (8 * q)) & 0xffu;
        ncand += bk[q] != 0;
        key[q] = __funnelshift_rc(e.z, e.w, 8 * (q + 1)) >> keyShift;
        if (bk[q] && p.bitmapBytes && !pairBitmapTest(p, bitmapAddr, key[q])) {
            bk[q] = 0;
        }
    }
    if (p.bitmapBytes && p.bitmap2Shift) {
        u32 w2[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const u32 h2 = (key[q] * 0x85EBCA6Bu) >> p.bitmap2Shift;
            w2[q] = bk[q] ? (__ldg(p.bitmap2 + (h2 >> 5)) >> (h2 & 31)) & 1u : 0u;
        }
#pragma unroll
        for (int q = 0; q < 4; q++) {
            bk[q] = w2[q] ? bk[q] : 0u;
        }
    }
    stats[0] += ncand;
    stats[1] += (bk[0] != 0) + (bk[1] != 0) + (bk[2] != 0) + (bk[3] != 0);
    appendWordCandidates(p, runStart + e.x, bk, lane);
}

template <int SB, int MAXT, int HEAVY>
__global__ void __launch_bounds__(MAXT, 1) scanKernelPair(const HSB_GRID_CONSTANT ScanParams p) {
    HSB_DYNAMIC_SMEM(smem);
    const u32 lane = threadIdx.x & 31;
    const u32 warp = threadIdx.x >> 5;
    const u32 nwarps = blockDim.x >> 5;

    /* this warp's contiguous run of tiles */
    const u32 gwarp = blockIdx.x * nwarps + warp;
    const u32 totalWarps = gridDim.x * nwarps;
    const u32 q = p.ntiles / totalWarps, rem = p.ntiles % totalWarps;
    const u32 myCount = q + (gwarp < rem ? 1u : 0u);
    const u32 myFirst = p.tileFirst + gwarp * q + min(gwarp, rem);
    const u64 runStart = (u64)myFirst * p.tileBytes;
    const u8 *ptr = p.corpus + runStart + lane * 16; /* this lane's 16 bytes of the current step */
    const u8 *const endPtr = p.corpus + p.readableEnd;

    auto load = [&](const u8 *src, bool guard) -> uint4 {
        uint4 r = make_uint4(0, 0, 0, 0);
        if (!guard || src + 16 <= endPtr) {
            r = ldCs128(src);
        }
        return r;
    };
    /* L2 prefetch of the 2 KiB (four steps) that lie pfDist steps after the lane's
     * position `at`: even lanes, 16 x 128 B */
    const size_t pfBytes = (size_t)p.pfDist * 512 + lane * 48;
    auto prefetchAhead = [&](const u8 *at) {
        if ((lane & 1) == 0) {
            const u8 *pf = at + pfBytes;
            if (pf < endPtr) {
                prefetchL2(pf);
            }
        }
    };

    /* the stream starts before the tables are expanded: steps 0 and 1, the 16 bytes
     * before the run and the first prefetch are in flight during the expansion */
    uint4 cur = make_uint4(0, 0, 0, 0), nxt = cur, hv = cur;
    if (myCount != 0) {
        cur = load(ptr, true);
        nxt = load(ptr + 512, true);
        if (runStart != 0) {
            hv = __ldg(reinterpret_cast<const uint4 *>(p.corpus + runStart - 16));
        }
        prefetchAhead(ptr);
    }

    /* expand the tables: p.table = 256 class words, then 1024 pair entries; the
     * (32 KiB) prefilter bitmap, if any, fills the class rows' upper halves.  In 16-byte
     * units: a class row is 8 units of {c | l << 2} for four lanes l and 8 units of the
     * bitmap, a pair row 8 units of its entry four times */
    {
        const u32 *g = reinterpret_cast<const u32 *>(p.table);
        const uint4 *bm = reinterpret_cast<const uint4 *>(p.bitmap);
        const u32 sBase = smemAddr(smem);
        const bool keyed = p.bitmapBytes != 0;
        for (u32 u = threadIdx.x; u < PAIR_CLASS_BYTES / 32; u += blockDim.x) {
            const u32 c = __ldg(g + (u >> 3));
            const uint4 b = keyed ? __ldg(bm + u) : make_uint4(0, 0, 0, 0);
            const u32 a = sBase + (u >> 3) * 256 + (u & 7) * 16, l = (u & 7) * 16;
            sts128(a, c | l, c | (l + 4), c | (l + 8), c | (l + 12));
            sts128(a + 128, b.x, b.y, b.z, b.w);
        }
        for (u32 u = threadIdx.x; u < p.pairBytes / 16; u += blockDim.x) {
            const u32 e = __ldg(g + 256 + (u >> 3));
            sts128(sBase + PAIR_CLASS_BYTES + u * 16, e, e, e, e);
        }
    }
    __syncthreads();

    const u32 clsAddr = smemAddr(smem);
    const u32 bitmapAddr = clsAddr + 128;
    const u32 laneOff = lane * 4;
    const u32 qAddr = clsAddr + PAIR_CLASS_BYTES + p.pairBytes + warp * PairQueue::WARP_BYTES;
    if (myCount == 0) {
        return;
    }
    u64 runEnd = runStart + (u64)myCount * p.tileBytes;
    if (runEnd > p.corpusBytes) {
        runEnd = p.corpusBytes;
    }
    const u32 nsteps = (u32)((runEnd - runStart + 511) >> 9);
    if (lane == 0) {
        sts64(qAddr + PairQueue::RUN_START, (u32)runStart, (u32)(runStart >> 32));
    }

    u32 carry = 0; /* lane 31's overflow of the previous step */
    u32 stats[3] = {0, 0, 0};
    u32 qn = 0;

    /* SB = 1: lane 31's last class word of the previous step (lane field 31: the pair
     * lookups stay a rotation of the banks).  Entering the run at the start of the corpus
     * byte 0x00 stands in for the byte before it, as it does in confirm (confValAt); a slot
     * that reaches before a literal's first byte never constrains its bucket anyway. */
    u32 prevCls = SB == 1 ? lds32(clsAddr + 31 * 4) : 0u;
    u32 prevW = 0; /* heavy: the last word of the previous step (own lane's; lane 31's is the one used) */
    if (runStart != 0) {
        /* state entering the run: the 16 bytes before it, as "lane -1" */
        u32 hE[17];
        if constexpr (SB == 1) {
            laneClasses<1>(hv, clsAddr, laneOff, hE);
            hE[0] = hE[1]; /* sample 0 does not overflow */
            prevCls = __shfl_sync(0xffffffffu, hE[16], 31);
        } else {
            laneClasses<0>(hv, clsAddr, laneOff, hE);
            hE[16] = lds32(clsAddr + __byte_perm(__shfl_sync(0xffffffffu, cur.x, 0), laneOff, 0x5504));
        }
        u32 ha[6];
        pairFilter(hE, clsAddr, ha);
        carry = ha[4];
        prevW = hv.w;
    }
    u32 step = 0;
    u32 prevRecv = carry;
    /* one 512-byte step: v = the lane's 16 bytes, nextFirst = first word of the NEXT
     * step (SB = 0: lane 0 hands it to lane 31 in the rotate shuffle) */
    auto compute = [&](const uint4 v, const u32 nextFirst, const u32 chunk) {
        u32 E[17];
        if constexpr (SB == 1) {
            laneClasses<1>(v, clsAddr, laneOff, E);
            /* the class word of the byte before the lane: the left neighbour's last (ONE
             * rotate shuffle); lane 0 takes lane 31's of the previous step */
            const u32 left = __shfl_sync(0xffffffffu, E[16], (lane + 31) & 31);
            E[0] = lane == 0 ? prevCls : left;
            prevCls = left;
        } else {
            const u32 w4 = __shfl_sync(0xffffffffu, lane == 0 ? nextFirst : v.x, (lane + 1) & 31);
            laneClasses<0>(v, clsAddr, laneOff, E);
            E[16] = lds32(clsAddr + __byte_perm(w4, laneOff, 0x5504));
        }
        u32 a[6];
        pairFilter(E, clsAddr, a);
        /* ONE rotate-by-one shuffle: lanes 1..31 receive their left neighbour's
         * overflow, lane 0 receives lane 31's = the carry into the NEXT step */
        const u32 recv = __shfl_sync(0xffffffffu, a[4], (lane + 31) & 31);
        a[0] |= lane == 0 ? prevRecv : recv;
        prevRecv = recv;
        /* a zero bit anywhere = candidate: test the AND of the four words */
        const u32 all = a[0] & a[1] & a[2] & a[3];
        if (HEAVY) {
            if (__any_sync(0xffffffffu, all != 0xffffffffu)) {
                /* four static rounds, one per word of the lane: the lanes whose word k has
                 * a candidate byte append it (slot from a ballot prefix); 32 pending
                 * entries are drained at once */
                /* the word before the lane's: the left neighbour's last, lane 0: lane 31's
                 * of the previous step (kept in a register, no corpus read) */
                const u32 pw = __shfl_sync(0xffffffffu, lane == 31 ? prevW : v.w, (lane + 31) & 31);
                const u32 wv[5] = {pw, v.x, v.y, v.z, v.w};
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const u32 m = ~a[k];
                    const u32 bal = __ballot_sync(0xffffffffu, m != 0);
                    if (bal) {
                        if (m) {
                            const u32 slot = qn + __popc(bal & ((1u << lane) - 1));
                            sts128(qAddr + slot * 16, chunk * 16 + 4 * k, m, wv[k], wv[k + 1]);
                        }
                        qn += __popc(bal);
                        if (qn >= 32) {
                            __syncwarp();
                            qn -= 32;
                            drainPairWords(p, bitmapAddr, qAddr, qn, 32, lane, stats);
                            __syncwarp();
                        }
                    }
                }
            }
            prevW = v.w;
            return;
        }
        const u32 bal = __ballot_sync(0xffffffffu, all != 0xffffffffu);
        if (bal) {
            if (all != 0xffffffffu) {
                const u32 e = qn + __popc(bal & ((1u << lane) - 1));
                sts128(qAddr + e * 16, ~a[0], ~a[1], ~a[2], ~a[3]);
                sts32(qAddr + PairQueue::CHUNK + e * 4, chunk);
            }
            qn += __popc(bal);
            if (qn >= 32) {
                __syncwarp();
                qn -= 32;
                drainPair(p, bitmapAddr, qAddr, qn, 32, lane, stats);
                __syncwarp();
            }
        }
    };
    /* Register pipeline two steps deep (cur = step 0 and nxt = step 1 are in flight since
     * before the barrier): with SB = 0 the first thing a step does is hand lane 31 the
     * next step's first word, so a load issued only one step ahead would be waited for at
     * once (long-scoreboard stalls of a full L2 round trip per step).  The load issued in
     * step s fetches step s + 2; it needs no bounds check while that whole step is
     * readable for every lane -- everywhere but at the very end of the corpus. */
    const u64 readableSteps = (p.readableEnd - runStart) >> 9;
    const u32 nFast = readableSteps >= (u64)nsteps + 2 ? nsteps : (readableSteps > 2 ? (u32)readableSteps - 2 : 0);
    /* main loop: four steps per iteration (loads at immediate offsets, no register
     * moves between steps) and ONE L2 prefetch, at its end, of the next iteration's
     * 2 KiB pfDist steps ahead (the first iteration's went out before the barrier) */
#pragma unroll 1
    for (; step + 4 <= nFast; step += 4, ptr += 2048) {
        const uint4 n2 = ldCs128(ptr + 1024);
        compute(cur, nxt.x, step * 32 + lane);
        const uint4 n3 = ldCs128(ptr + 1536);
        compute(nxt, n2.x, step * 32 + 32 + lane);
        cur = ldCs128(ptr + 2048);
        compute(n2, n3.x, step * 32 + 64 + lane);
        nxt = ldCs128(ptr + 2560);
        compute(n3, cur.x, step * 32 + 96 + lane);
        prefetchAhead(ptr + 2048);
    }
#pragma unroll 1
    for (; step < nsteps; step++, ptr += 512) {
        const uint4 n2 = load(ptr + 1024, step >= nFast);
        compute(cur, nxt.x, step * 32 + lane);
        cur = nxt;
        nxt = n2;
    }
    if (qn) {
        __syncwarp();
        if (HEAVY) {
            drainPairWords(p, bitmapAddr, qAddr, 0, qn, lane, stats);
        } else {
            drainPair(p, bitmapAddr, qAddr, 0, qn, lane, stats);
        }
    }
    if (stats[0]) {
        atomicAdd(p.counters + CTR_CANDIDATES, stats[0]);
    }
    if (stats[1]) {
        atomicAdd(p.counters + CTR_PREFILTER_PASS, stats[1]);
    }
}

/* ---- class 4-gram variant (FK_GRAM4): sets whose two-byte evidence saturates ----------
 *
 * With tens of thousands of literals every pair of letters occurs in every bucket and
 * the pair filter above passes any four letters (~6 % of printable text).  What still
 * separates such a set from the text is the JOINT last four bytes, so the first stage
 * becomes an exact membership test of the class 4-gram: every byte maps to one of 32
 * classes (per-lane rows as above, conflict free), the classes of the four bytes ending
 * at a position form a 20-bit index into a 1 Mbit bitmap in shared memory (128 KiB;
 * word = the three older classes, bit = the newest), one random 4-byte lookup per
 * position.  No buckets: a set bit is a candidate for every bucket, the second-level
 * bitmap in L2 (raw 4-byte key) and the hash confirm sort that out.
 *
 *   class row b (256 B): [E = 4 * c(b)] x 32 lanes | 128 B unused
 *   byte address of position e's word = E[e-3] + 33 * E[e-2] + 1025 * E[e-1]   (two IMADs)
 *   bit = E[e] >> 2
 *
 * The word index c[e-3] + 33 c[e-2] + 1025 c[e-1] instead of the plain bit fields
 * c[e-3] | c[e-2] << 5 | c[e-1] << 10: the bank of a lookup is then (c[e-3] + c[e-2] +
 * c[e-1]) mod 32, not c[e-3] alone -- with the plain fields every lane whose byte e-3 is
 * no letter (class 0: half of printable text) hits bank 0 at a different address, 11
 * wavefronts per lookup against ~3.5 now. */
struct GramQueue {
    static constexpr u32 SLOTS = 64;                      /* < 32 pending + <= 32 appended per round */
    static constexpr u32 RUN_START = 16 * SLOTS;          /* entry = {word offset in the run, 4-bit candidate map,
                                                           * the word before, the word}: the bytes travel along */
    static constexpr u32 WARP_BYTES = RUN_START + 16;
};
enum { GRAM_CLASS_BYTES = 256 * 256, GRAM_BITMAP_BYTES = 4 * (31 * (1 + 33 + 1025) + 1 + 63) / 64 * 64 };

/* 32 queue entries, one word with candidates per lane (1.02 candidates on average): the
 * exact raw 4-byte keys against the second-level table in L2 -- one BYTE per slot, the
 * buckets whose literals own a key hashing there -- all probes of the warp in flight
 * together (a drain costs ONE L2 round trip), and the survivors, with those buckets, to
 * the candidate list through one reservation. */
__device__ HSB_NOINLINE void drainGram(const ScanParams &p, u32 qAddr, u32 first, u32 count, u32 lane,
                                       u32 *stats) {
    const uint2 rs = lds64(qAddr + GramQueue::RUN_START);
    uint4 e = make_uint4(0, 0, 0, 0);
    if (lane < count) {
        e = lds128(qAddr + (first + lane) * 16);
    }
    u32 bk[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        bk[q] = 0;
        if ((e.y >> q) & 1) {
            bk[q] = 0xffu;
            if (p.bitmap2Shift) {
                const u32 key = __funnelshift_rc(e.z, e.w, 8 * (q + 1));
                const u32 h2 = (key * 0x85EBCA6Bu) >> p.bitmap2Shift;
                bk[q] = __ldg(reinterpret_cast<const u8 *>(p.bitmap2) + h2);
            }
        }
    }
    stats[0] += __popc(e.y & 0xfu);
    stats[1] += (bk[0] != 0) + (bk[1] != 0) + (bk[2] != 0) + (bk[3] != 0);
    appendWordCandidates(p, (((u64)rs.y << 32) | rs.x) + e.x, bk, lane);
}

template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1) scanKernelGram(const HSB_GRID_CONSTANT ScanParams p) {
    HSB_DYNAMIC_SMEM(smem);
    const u32 lane = threadIdx.x & 31;
    const u32 warp = threadIdx.x >> 5;
    const u32 nwarps = blockDim.x >> 5;
    {
        /* p.table = 256 class words; p.bitmap = the 128 KiB class 4-gram bitmap */
        const u32 *g = reinterpret_cast<const u32 *>(p.table);
        u32 *s = reinterpret_cast<u32 *>(smem);
        for (u32 i = threadIdx.x; i < 256 * 64; i += blockDim.x) {
            s[i] = ((i >> 5) & 1) ? 0u : __ldg(g + (i >> 6));
        }
        const uint4 *bm = reinterpret_cast<const uint4 *>(p.bitmap);
        uint4 *sb = reinterpret_cast<uint4 *>(smem + GRAM_CLASS_BYTES);
        for (u32 i = threadIdx.x; i < GRAM_BITMAP_BYTES / 16; i += blockDim.x) {
            sb[i] = __ldg(bm + i);
        }
    }
    __syncthreads();
    const u32 clsAddr = smemAddr(smem);
    const u32 gramAddr = clsAddr + GRAM_CLASS_BYTES;
    const u32 laneOff = lane * 4;
    const u32 qAddr = gramAddr + GRAM_BITMAP_BYTES + warp * GramQueue::WARP_BYTES;

    const u32 gwarp = blockIdx.x * nwarps + warp;
    const u32 totalWarps = gridDim.x * nwarps;
    const u32 qq = p.ntiles / totalWarps, rem = p.ntiles % totalWarps;
    const u32 myCount = qq + (gwarp < rem ? 1u : 0u);
    const u32 myFirst = p.tileFirst + gwarp * qq + min(gwarp, rem);
    if (myCount == 0) {
        return;
    }
    const u64 runStart = (u64)myFirst * p.tileBytes;
    u64 runEnd = runStart + (u64)myCount * p.tileBytes;
    if (runEnd > p.corpusBytes) {
        runEnd = p.corpusBytes;
    }
    const u32 nsteps = (u32)((runEnd - runStart + 511) >> 9);
    const u8 *ptr = p.corpus + runStart + lane * 16;
    const u8 *const endPtr = p.corpus + p.readableEnd;
    if (lane == 0) {
        sts64(qAddr + GramQueue::RUN_START, (u32)runStart, (u32)(runStart >> 32));
    }
    u32 stats[3] = {0, 0, 0};
    u32 qn = 0;
    auto load = [&](const u8 *src, bool guard) -> uint4 {
        uint4 r = make_uint4(0, 0, 0, 0);
        if (!guard || src + 16 <= endPtr) {
            r = ldCs128(src);
        }
        return r;
    };
    auto cls = [&](u32 w, int r) -> u32 { return lds32(clsAddr + __byte_perm(w, laneOff, 0x5504 + (r << 4))); };
    const size_t pfBytes = (size_t)p.pfDist * 512 + lane * 48;

    /* carryPack: E of the three bytes before the lane's chunk, one per byte lane (E < 128);
     * lane 0 inherits lane 31's of the previous step.  Entering a run: the bytes before it;
     * at the very start of the corpus the class of byte 0x00 stands in (a literal cannot
     * begin before position 0: the block lookup in confirm rejects such candidates). */
    u32 carryPack;
    u32 prevW = 0; /* the last word of the previous step (own lane's; lane 31's is the one used) */
    if (runStart != 0) {
        const u32 hw = __ldg(reinterpret_cast<const u32 *>(p.corpus + runStart - 4));
        carryPack = cls(hw, 1) | (cls(hw, 2) << 8) | (cls(hw, 3) << 16);
        prevW = hw;
    } else {
        const u32 z = cls(0, 0);
        carryPack = z | (z << 8) | (z << 16);
    }
    auto compute = [&](const uint4 cur, const u32 chunk) {
        const u32 w[4] = {cur.x, cur.y, cur.z, cur.w};
        u32 E[19]; /* E[3 + j] = 4 * class of the lane's byte j; E[0..2] = the three bytes before */
#pragma unroll
        for (int k = 0; k < 4; k++) {
#pragma unroll
            for (int r = 0; r < 4; r++) {
                E[3 + 4 * k + r] = cls(w[k], r);
            }
        }
        const u32 myPack = E[16] | (E[17] << 8) | (E[18] << 16);
        const u32 recv = __shfl_sync(0xffffffffu, myPack, (lane + 31) & 31);
        const u32 prev = lane == 0 ? carryPack : recv;
        carryPack = recv; /* lane 0: lane 31's, for the next step */
        E[0] = prev & 0xffu;
        E[1] = (prev >> 8) & 0xffu;
        E[2] = prev >> 16;
        u32 cm = 0;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const u32 addr = E[j] + 33u * E[j + 1] + 1025u * E[j + 2];
            const u32 word = lds32(gramAddr + addr);
            const u32 t = __funnelshift_r(word, 0, E[j + 3] >> 2); /* bit c(byte j) of the word */
            cm = __funnelshift_r(cm, t, 1);
        }
        cm >>= 16;
        if (__any_sync(0xffffffffu, cm != 0)) {
            /* four static rounds, one per word of the lane: the lanes whose word k holds a
             * candidate append it with its bytes; 32 pending entries are drained at once */
            /* the word before the lane's: the left neighbour's last, lane 0: lane 31's of
             * the previous step (kept in a register, no corpus read) */
            const u32 pw = __shfl_sync(0xffffffffu, lane == 31 ? prevW : cur.w, (lane + 31) & 31);
            const u32 wv[5] = {pw, cur.x, cur.y, cur.z, cur.w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const u32 m = (cm >> (4 * k)) & 0xfu;
                const u32 bal = __ballot_sync(0xffffffffu, m != 0);
                if (bal) {
                    if (m) {
                        const u32 slot = qn + __popc(bal & ((1u << lane) - 1));
                        sts128(qAddr + slot * 16, chunk * 16 + 4 * k, m, wv[k], wv[k + 1]);
                    }
                    qn += __popc(bal);
                    if (qn >= 32) {
                        __syncwarp();
                        qn -= 32;
                        drainGram(p, qAddr, qn, 32, lane, stats);
                        __syncwarp();
                    }
                }
            }
        }
        prevW = cur.w;
    };
    const u64 readableSteps = (p.readableEnd - runStart) >> 9;
    const u32 nFast = readableSteps >= (u64)nsteps + 2 ? nsteps : (readableSteps > 2 ? (u32)readableSteps - 2 : 0);
    uint4 cur = load(ptr, true);
    uint4 nxt = load(ptr + 512, true);
    u32 step = 0;
#pragma unroll 1
    for (; step + 4 <= nFast; step += 4, ptr += 2048) {
        if ((lane & 1) == 0) {
            const u8 *pf = ptr + pfBytes;
            if (pf < endPtr) {
                prefetchL2(pf);
            }
        }
        const uint4 n2 = ldCs128(ptr + 1024);
        compute(cur, step * 32 + lane);
        const uint4 n3 = ldCs128(ptr + 1536);
        compute(nxt, step * 32 + 32 + lane);
        cur = ldCs128(ptr + 2048);
        compute(n2, step * 32 + 64 + lane);
        nxt = ldCs128(ptr + 2560);
        compute(n3, step * 32 + 96 + lane);
    }
#pragma unroll 1
    for (; step < nsteps; step++, ptr += 512) {
        const uint4 n2 = load(ptr + 1024, step >= nFast);
        compute(cur, step * 32 + lane);
        cur = nxt;
        nxt = n2;
    }
    if (qn) {
        __syncwarp();
        drainGram(p, qAddr, 0, qn, lane, stats);
    }
    if (stats[0]) {
        atomicAdd(p.counters + CTR_CANDIDATES, stats[0]);
    }
    if (stats[1]) {
        atomicAdd(p.counters + CTR_PREFILTER_PASS, stats[1]);
    }
}

cudaError_t launchGram(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream) {
    void (*kern)(const ScanParams) = cfg.warps <= 24 ? scanKernelGram<768> : scanKernelGram<896>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smemBytes);
    if (e != cudaSuccess) {
        return e;
    }
    HSB_LAUNCH(kern, cfg.grid, cfg.warps * 32, cfg.smemBytes, stream, p);
    return cudaGetLastError();
}

/* Second kernel of every scan: one thread per candidate of the list the scan
 * kernel filled -- hash confirm, block lookup, literal program, record. */
template <int CONF> __device__ __forceinline__ void confirmList(const ScanParams &p) {
    const u32 total = p.counters[CTR_CANDQ];
    const u32 n = total < p.outCap ? total : p.outCap;
    if (total > p.outCap && blockIdx.x == 0 && threadIdx.x == 0) {
        /* the list overflowed: make the scan report more records than the ring
         * holds, which sends the caller down its grow-and-rescan path */
        atomicMax(p.counters + CTR_MATCHES, total);
    }
    const DevCand *list = reinterpret_cast<const DevCand *>(p.out + p.outCap);
    u32 nconf = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(list + i));
        const u64 g = ((u64)raw.y << 32) | raw.x;
        u32 buckets = raw.z;
        if (p.bucketFold) {
            buckets |= buckets << 8;
        }
        const u64 confVal = confValAt(p, g);
        if (p.confirmKind == CK_NOODLE) {
            if (buckets & 1) {
                confirmNoodle<CONF>(p, g, confVal, &nconf);
            }
        } else {
            while (buckets) {
                const u32 bucket = __ffs(buckets) - 1;
                buckets &= buckets - 1;
                confirmFdr<CONF>(p, bucket, g, confVal, &nconf);
            }
        }
    }
    if (nconf) {
        atomicAdd(p.counters + CTR_CONFIRMED, nconf);
    }
}

__global__ void __launch_bounds__(256) confirmKernel(const HSB_GRID_CONSTANT ScanParams p) {
    confirmList<CONF_PLAIN>(p);
}

/* the confirm kernel of a stream-set mask pass over rows (p.mask.rows.sorted set): each match sets the bit of the
 * batch row that holds its last byte, not of its block (a group) */
__global__ void __launch_bounds__(256) confirmRowsMaskKernel(const HSB_GRID_CONSTANT ScanParams p) {
    confirmList<CONF_ROWS_MASK>(p);
}

/* the confirm kernel of a first-match pass (p.mask.first set): each match lowers its block's entry, and a candidate
 * that ends after the entry is dropped before its program runs */
__global__ void __launch_bounds__(256) confirmFirstKernel(const HSB_GRID_CONSTANT ScanParams p) {
    confirmList<CONF_FIRST>(p);
}

cudaError_t launchWide(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream) {
    /* builds for 768 threads (80 registers), 896 (72) and 1024 (64, still no spills) */
    void (*kern)(const ScanParams) = cfg.warps <= 24   ? scanKernelWide<768>
                                     : cfg.warps <= 28 ? scanKernelWide<896>
                                                       : scanKernelWide<1024>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smemBytes);
    if (e != cudaSuccess) {
        return e;
    }
    HSB_LAUNCH(kern, cfg.grid, cfg.warps * 32, cfg.smemBytes, stream, p);
    return cudaGetLastError();
}

template <int SB> cudaError_t launchPair(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream) {
    /* heavy: the candidate path with one queue entry per word with candidates */
    void (*kern)(const ScanParams) =
        cfg.heavy ? (cfg.warps <= 24 ? scanKernelPair<SB, 768, 1> : scanKernelPair<SB, 896, 1>)
                  : (cfg.warps <= 24 ? scanKernelPair<SB, 768, 0> : scanKernelPair<SB, 896, 0>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smemBytes);
    if (e != cudaSuccess) {
        return e;
    }
    HSB_LAUNCH(kern, cfg.grid, cfg.warps * 32, cfg.smemBytes, stream, p);
    return cudaGetLastError();
}

} // namespace

size_t scanSmemBytes(int kind, u32 tableBytes, u32 bitmapBytes, int queueWarps) {
    if (kind == FK_GRAM4) { /* class rows + 1 Mbit class 4-gram bitmap + queues */
        return (size_t)GRAM_CLASS_BYTES + GRAM_BITMAP_BYTES + (size_t)queueWarps * GramQueue::WARP_BYTES;
    }
    if (kind == FK_PAIR32) { /* class rows (with the bitmap in their upper halves) + pair table + queues */
        return (size_t)PAIR_CLASS_BYTES + tableBytes + (size_t)queueWarps * PairQueue::WARP_BYTES;
    }
    /* FK_BYTE32: lane-replicated byte table + bitmap + queues */
    return (size_t)BYTE_TABLE_BYTES + bitmapBytes + (size_t)queueWarps * WideQueue::WARP_BYTES;
}

namespace {
__global__ void publishCountKernel(const ScanParams p) {
    const u32 r = threadIdx.x;
    if (r < p.nPeers) {
        DevMatch h;
        h.id = p.counters[CTR_MATCHES]; /* slot 0 = {count, 0, 0} */
        h.block = 0;
        h.to = 0;
        const size_t slot = (size_t)p.myRank * (p.peerCap + 1);
        *reinterpret_cast<uint4 *>(p.peers[r] + slot) = *reinterpret_cast<const uint4 *>(&h);
    }
}
} // namespace

namespace {
template <u32 FILL> __global__ void maskClearKernel(u32 *bits, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        bits[i] = FILL;
    }
}

/* the verdict hs_b200_scan_corpus_finish reaches from the same counters (finishScan) */
__global__ void maskStatusKernel(const u32 *counters, u32 outCap, u32 *status) {
    *status = counters[CTR_ERROR] || (counters[CTR_STREAM] & STREAM_BAD_LENGTH) || counters[CTR_MATCHES] > outCap;
}
} // namespace

cudaError_t launchMaskClear(u32 *bits, u64 n, int smCount, cudaStream_t stream, bool ones) {
    if (!n) {
        return cudaSuccess;
    }
    const u64 blocks = std::min<u64>((n + 255) / 256, (u64)std::max(1, smCount) * 8);
    if (ones) {
        HSB_LAUNCH(maskClearKernel<0xffffffffu>, (unsigned)blocks, 256, 0, stream, bits, n);
    } else {
        HSB_LAUNCH(maskClearKernel<0u>, (unsigned)blocks, 256, 0, stream, bits, n);
    }
    return cudaGetLastError();
}

cudaError_t launchMaskStatus(const u32 *counters, u32 outCap, u32 *status, cudaStream_t stream) {
    HSB_LAUNCH(maskStatusKernel, 1, 1, 0, stream, counters, outCap, status);
    return cudaGetLastError();
}

namespace {
__global__ void streamAssembleKernel(u8 *corpus, const u8 *hist, u32 nstreams, u32 pitch, const u32 *srcLens,
                                     u32 *lens, StreamMark *mark, u32 epoch) {
    const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nstreams) {
        return;
    }
    /* header = 16 bytes: zeros, then the hl history bytes right-aligned */
    const uint2 h = *reinterpret_cast<const uint2 *>(hist + (size_t)b * 8);
    const u32 hl = h.y >> 24;
    const u64 hv = (((u64)h.y << 32) | h.x) & 0x00ffffffffffffffULL; /* bytes 0..6 */
    u64 hi = 0;
    if (hl) {
        hi = hv << (8 * (8 - hl)); /* last history byte lands in byte 7 */
    }
    uint4 out;
    out.x = 0;
    out.y = 0;
    out.z = (u32)hi;
    out.w = (u32)(hi >> 32);
    *reinterpret_cast<uint4 *>(corpus + (size_t)b * pitch) = out;
    if (srcLens) {
        /* the scan reads the lengths from here: a bad one must not let a block reach past the buffer */
        u32 l = srcLens[b];
        if (l > pitch - 16) {
            l = 0;
            mark->bad = epoch + 1;
        }
        lens[b] = l;
    }
}

__global__ void streamAdvanceKernel(const u8 *corpus, u8 *hist, u64 *offsets, const u32 *lens, u32 uniformLen,
                                    u32 nstreams, u32 pitch, u32 histReq, u32 *counters, u32 outCap,
                                    StreamMark *mark, u32 epoch) {
    const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (!streamPassCommits(counters, outCap, mark, epoch, b == 0)) {
        return;
    }
    if (b >= nstreams) {
        return;
    }
    const u32 hl = hist[(size_t)b * 8 + 7];
    const u32 wl = uniformLen ? uniformLen : lens[b];
    if (wl == 0) {
        return;
    }
    /* maintainHistoryBuffer (src/runtime.c:478-508): keep the last histReq bytes */
    const u32 total = hl + wl;
    const u32 keep = total < histReq ? total : histReq;
    const u8 *end = corpus + (size_t)b * pitch + 16 + wl;
    u64 v = 0;
    for (u32 i = 0; i < keep; i++) {
        v |= (u64)end[(int)i - (int)keep] << (8 * i);
    }
    v |= (u64)keep << 56;
    *reinterpret_cast<uint2 *>(hist + (size_t)b * 8) = make_uint2((u32)v, (u32)(v >> 32));
    offsets[b] += wl;
}

__global__ void streamResetKernel(u8 *hist, u64 *offsets, const u32 *idx, u32 count, u32 nstreams,
                                  const StreamMark *mark, u32 epoch) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    /* a reset behind a pass that did not commit commits nothing either: the caller enqueues it again with the
     * passes */
    if (i >= count || mark->marked == epoch + 1) {
        return;
    }
    const u32 b = idx ? idx[i] : i;
    if (b >= nstreams) {
        return;
    }
    *reinterpret_cast<uint2 *>(hist + (size_t)b * 8) = make_uint2(0, 0);
    offsets[b] = 0;
}
} // namespace

cudaError_t launchStreamAssemble(u8 *corpus, const u8 *hist, u32 nstreams, u32 pitch, const u32 *srcLens,
                                 u32 *lens, StreamMark *mark, u32 epoch, cudaStream_t stream) {
    if (nstreams) {
        HSB_LAUNCH(streamAssembleKernel, (nstreams + 255) / 256, 256, 0, stream, corpus, hist, nstreams, pitch,
                   srcLens, lens, mark, epoch);
    }
    return cudaGetLastError();
}

cudaError_t launchStreamAdvance(const u8 *corpus, u8 *hist, u64 *offsets, const u32 *lens, u32 uniformLen,
                                u32 nstreams, u32 pitch, u32 histReq, u32 *counters, u32 outCap, StreamMark *mark,
                                u32 epoch, cudaStream_t stream) {
    if (nstreams) {
        HSB_LAUNCH(streamAdvanceKernel, (nstreams + 255) / 256, 256, 0, stream, corpus, hist, offsets, lens,
                   uniformLen, nstreams, pitch, histReq, counters, outCap, mark, epoch);
    }
    return cudaGetLastError();
}

cudaError_t launchStreamReset(u8 *hist, u64 *offsets, const u32 *idx, u32 count, u32 nstreams,
                              const StreamMark *mark, u32 epoch, cudaStream_t stream) {
    if (count) {
        HSB_LAUNCH(streamResetKernel, (count + 255) / 256, 256, 0, stream, hist, offsets, idx, count, nstreams,
                   mark, epoch);
    }
    return cudaGetLastError();
}

cudaError_t launchConfirm(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream) {
    if (p.mask.rows.sorted) {
        HSB_LAUNCH(confirmRowsMaskKernel, cfg.grid * 2, 256, 0, stream, p);
        return cudaGetLastError();
    }
    if (p.mask.first) {
        HSB_LAUNCH(confirmFirstKernel, cfg.grid * 2, 256, 0, stream, p);
        return cudaGetLastError();
    }
    HSB_LAUNCH(confirmKernel, cfg.grid * 2, 256, 0, stream, p);
    return cudaGetLastError();
}

cudaError_t launchPublishCount(const ScanParams &p, cudaStream_t stream) {
    HSB_LAUNCH(publishCountKernel, 1, 32, 0, stream, p);
    return cudaGetLastError();
}

cudaError_t launchScan(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream) {
    if (cfg.warps > (cfg.kind == FK_BYTE32 ? 32 : 28)) {
        return cudaErrorInvalidValue;
    }
    if (cfg.kind == FK_GRAM4) {
        return launchGram(cfg, p, stream);
    }
    if (cfg.kind == FK_PAIR32) {
        return cfg.slotBase ? launchPair<1>(cfg, p, stream) : launchPair<0>(cfg, p, stream);
    }
    if (cfg.kind == FK_BYTE32 && !(p.tileBytes & 1023)) {
        return launchWide(cfg, p, stream);
    }
    return cudaErrorInvalidValue;
}

} // namespace hsb
