/*
 * order_kernels.h -- the report rules of ReportRules::deliver (host/db_walk.cpp) on the device:
 * raw match records in HBM -> delivered matches in HBM, in (block, to, id) order, with no host
 * synchronisation (hs_b200_order_matches_async / hs_b200_order_records_async).
 *
 *   resolve   padding slots dropped, ENGINE_RECORD stripped, an engine's record replaced by the
 *             reports its program raises (CHECK_BOUNDS, offset_adjust); literal records kept.
 *             Counted per tile first, then scattered in input order.
 *   sort      stable LSD radix sort, 8-bit digits, of the key (block, to, id rank) packed into
 *             only as many bits as the largest block, the largest `to` and the largest rank need
 *             (up to 128 bits: every pass reads its digit from the three fields).  The number of
 *             passes is decided on the device; passes beyond it return at once.
 *   dedupe    a record equal to its predecessor goes; for an exhaustible id, only the first
 *             record of each (block, id) stays (a hash table keyed by (block, rank) keeps the
 *             lowest position).
 *   compact   the kept records, ids restored, into out[0, cap); their count into *count.
 *
 * Every kernel works in tiles of ORDER_TILE records (ORDER_ITEMS rounds of ORDER_THREADS), so the
 * grids are sized by the capacities the host knows and the counts are read on the device.  No CUB
 * or Thrust, and only the intrinsics the SIMT emulator of tests/emu models: the same code runs there.
 *
 * Included once, by api_device.cu (the entry points that enqueue it): the kernels compile in that
 * translation unit, in the product build and in the emulated one alike.
 */
#ifndef HSB200_ORDER_KERNELS_H
#define HSB200_ORDER_KERNELS_H

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "../host/db_walk.h"
#include "kernels.h"
#include "resolve.h"

namespace hsb {

namespace {

const u32 FULL = 0xffffffffu;
const u64 EX_EMPTY = ~0ull;

/* (once per ordering, by one thread) */
__device__ u32 bitsOf(u64 v) {
    u32 b = 0;
    for (; v; v >>= 1) {
        b++;
    }
    return b;
}

/* compare-and-swap of a hash-table key */
__device__ __forceinline__ u64 casKey(u64 *p, u64 expect, u64 key) {
#ifdef HSB_HOST_EMU /* the SIMT emulator of tests/emu runs one thread at a time between its barriers */
    const u64 old = *p;
    if (old == expect) {
        *p = key;
    }
    return old;
#else
    return atomicCAS((unsigned long long *)p, (unsigned long long)expect, (unsigned long long)key);
#endif
}

__device__ __forceinline__ u32 tilesOf(u32 n) { return (n + ORDER_TILE - 1) / ORDER_TILE; }

/* exclusive prefix of v over the block (warps * 32 threads, at most 32 warps) in thread order; *total
 * receives the block's sum.  sm: 33 words of shared memory. */
__device__ u32 blockExclusive(u32 v, u32 *sm, u32 *total) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    u32 x = v;
    for (u32 o = 1; o < 32; o <<= 1) {
        const u32 y = __shfl_up_sync(FULL, x, o);
        if (lane >= o) {
            x += y;
        }
    }
    if (lane == 31) {
        sm[warp] = x;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 run = 0;
        for (u32 w = 0; w < nwarps; w++) {
            const u32 t = sm[w];
            sm[w] = run;
            run += t;
        }
        sm[32] = run;
    }
    __syncthreads();
    const u32 r = sm[warp] + x - v;
    *total = sm[32];
    __syncthreads();
    return r;
}

/* index of program `off` in the table, or -1 */
__device__ int findProgram(const OrderParams &p, u32 off) { return indexOf(p.progOff, p.nProg, off); }

/* dense rank of report id `id`, or -1 */
__device__ int rankOf(const OrderParams &p, u32 id) { return indexOf(p.ids, p.nIds, id); }

/* What one raw record becomes (ReportRules::deliver): *prog = -1 and 1 record as it is (a literal's), or
 * the program whose reports replace it (0 records for a padding slot or a program not in the table). */
struct Resolved {
    DevMatch r;
    int prog;
    u32 count;
};

__device__ Resolved resolveOne(const OrderParams &p, DevMatch r) {
    Resolved x;
    x.prog = -1;
    x.count = 1;
    if (p.shape == SHAPE_PURE_LITERAL) {
        x.r = r;
        return x;
    }
    if (p.shape == SHAPE_LITERALS_OUTFIX) {
        if (!(r.to & ENGINE_RECORD)) {
            x.r = r;
            return x;
        }
        r.to &= ~ENGINE_RECORD;
    }
    x.r = r;
    x.count = 0;
    if (r.id == 0xffffffffu) {
        return x;
    }
    x.prog = findProgram(p, r.id);
    x.count = programReports(p.progStart, p.reps, x.prog, r.to, [](const OrderRep &) {});
    return x;
}

__global__ void orderSetupKernel(const OrderParams p) {
    OrderState *st = p.st;
    if (threadIdx.x == 0) {
        u32 n = p.inN;
        st->overflow = 0;
        if (p.inCount) {
            n = *p.inCount;
            if (n > p.inCap) {
                st->overflow = 1;
                n = 0;
            }
        }
        st->n = n;
        st->m = p.shape == SHAPE_PURE_LITERAL ? n : 0;
        st->kept = 0;
        st->maxTo = 0;
        st->maxBlock = 0;
        st->maxId = 0;
        st->unknownIds = 0;
        st->passes = 0;
        st->idBits = st->toBits = st->blockBits = 0;
    }
    for (u32 i = threadIdx.x; i < ORDER_MAX_PASSES * 256; i += blockDim.x) {
        p.binTotal[i] = 0;
    }
}

/* per tile: the number of records its input records resolve to */
__global__ void __launch_bounds__(ORDER_THREADS) resolveCountKernel(const OrderParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    const u32 n = p.st->n, base = blockIdx.x * ORDER_TILE;
    if (base >= n) {
        return;
    }
    u32 c = 0;
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        if (i < n) {
            c += resolveOne(p, p.in[i]).count;
        }
    }
    u32 total;
    blockExclusive(c, sm, &total);
    if (threadIdx.x == 0) {
        p.tileSum[blockIdx.x] = total;
    }
}

/* exclusive scan of the per-tile sums of `which` (0: the resolve counts of st->n records, 1: the kept
 * records of st->m) in place; the total goes to st->m / st->kept, and for 1 the delivered count to
 * *p.count (HS_B200_ORDER_RING_OVERFLOW after a ring overflow) */
__global__ void tileScanKernel(const OrderParams p, u32 which) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    OrderState *st = p.st;
    const u32 ntiles = tilesOf(which == 0 ? st->n : st->m);
    u32 carry = 0;
    for (u32 b = 0; b < ntiles; b += blockDim.x) {
        const u32 t = b + threadIdx.x;
        const u32 v = t < ntiles ? p.tileSum[t] : 0;
        u32 total;
        const u32 ex = blockExclusive(v, sm, &total);
        if (t < ntiles) {
            p.tileSum[t] = carry + ex;
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        if (which == 0) {
            st->m = carry;
        } else {
            st->kept = carry;
            *p.count = st->overflow ? ~0ull : (unsigned long long)carry;
        }
    }
}

__device__ __forceinline__ void warpMax(u64 &v) {
    for (u32 o = 16; o; o >>= 1) {
        const u64 y = __shfl_sync(FULL, v, (threadIdx.x & 31) ^ o);
        v = y > v ? y : v;
    }
}

/* write the resolved records of the tile into buf[0] in input order; the largest block, `to` and id */
__global__ void __launch_bounds__(ORDER_THREADS) resolveScatterKernel(const OrderParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    OrderState *st = p.st;
    const u32 n = st->n, base = blockIdx.x * ORDER_TILE;
    if (base >= n) {
        return;
    }
    const bool pure = p.shape == SHAPE_PURE_LITERAL;
    u32 run = pure ? base : p.tileSum[blockIdx.x];
    u64 maxBlock = 0, maxTo = 0, maxId = 0;
    u32 unknown = 0;
    DevMatch *dst = p.buf[0];
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        Resolved x;
        x.count = 0;
        x.prog = -1;
        if (i < n) {
            x = resolveOne(p, p.in[i]);
        }
        u32 total;
        u32 pos = run + blockExclusive(x.count, sm, &total);
        run += total;
        auto emit = [&](const DevMatch &o) {
            dst[pos++] = o;
            maxBlock = o.block > maxBlock ? o.block : maxBlock;
            maxTo = o.to > maxTo ? o.to : maxTo;
            maxId = o.id > maxId ? o.id : maxId;
            unknown |= rankOf(p, o.id) < 0;
        };
        if (x.count && x.prog < 0) {
            emit(x.r);
        } else if (x.count) {
            programReports(p.progStart, p.reps, x.prog, x.r.to, [&](const OrderRep &rp) {
                DevMatch o = x.r;
                o.id = rp.onmatch;
                o.to = (u64)((long long)x.r.to + rp.adjust) | (rp.logical ? LKEY_RECORD : 0);
                emit(o);
            });
        }
    }
    warpMax(maxBlock);
    warpMax(maxTo);
    warpMax(maxId);
    unknown = __ballot_sync(FULL, unknown != 0);
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&st->maxBlock, (u32)maxBlock);
        atomicMax((unsigned long long *)&st->maxTo, (unsigned long long)maxTo);
        atomicMax(&st->maxId, (u32)maxId);
        if (unknown) {
            atomicMax(&st->unknownIds, 1u);
        }
    }
}

/* the key's field widths and pass count; ids -> dense ranks when every id is in the table */
__global__ void __launch_bounds__(ORDER_THREADS) rankKernel(const OrderParams p) {
    OrderState *st = p.st;
    const u32 m = st->m, base = blockIdx.x * ORDER_TILE;
    const bool raw = st->unknownIds != 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        st->idBits = raw ? bitsOf(st->maxId) : bitsOf(p.nIds ? p.nIds - 1 : 0);
        st->toBits = bitsOf(st->maxTo);
        st->blockBits = bitsOf(st->maxBlock);
        st->passes = (st->idBits + st->toBits + st->blockBits + 7) / 8;
    }
    if (raw || base >= m) {
        return;
    }
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        if (i < m) {
            p.buf[0][i].id = (u32)rankOf(p, p.buf[0][i].id);
        }
    }
}

/* bits [lo, lo + 8) of the key (block : to : id), fields of the given widths from the low end */
struct KeyLayout {
    u32 idBits, toBits;
    __device__ static u32 part(u64 v, u32 start, u32 width, u32 lo) {
        if (width == 0 || start + width <= lo || start >= lo + 8) {
            return 0;
        }
        return (u32)(start >= lo ? v << (start - lo) : v >> (lo - start)) & 0xff;
    }
    __device__ u32 digit(const DevMatch &r, u32 pass) const {
        const u32 lo = pass * 8;
        return part(r.id, 0, idBits, lo) | part(r.to, idBits, toBits, lo) | part(r.block, idBits + toBits, 32, lo);
    }
};

__device__ __forceinline__ KeyLayout keyOf(const OrderState *st) {
    KeyLayout k;
    k.idBits = st->idBits;
    k.toBits = st->toBits;
    return k;
}

/* pass `pass`: per tile, the count of every digit value (hist[d][tile]) and their totals */
__global__ void __launch_bounds__(ORDER_THREADS) histKernel(const OrderParams p, u32 pass) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *h = reinterpret_cast<u32 *>(smem);
    const OrderState *st = p.st;
    const u32 m = st->m, base = blockIdx.x * ORDER_TILE;
    if (pass >= st->passes || base >= m) {
        return;
    }
    const KeyLayout key = keyOf(st);
    const DevMatch *src = p.buf[pass & 1];
    h[threadIdx.x] = 0;
    __syncthreads();
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        if (i < m) {
            atomicAdd(&h[key.digit(src[i], pass)], 1u);
        }
    }
    __syncthreads();
    const u32 c = h[threadIdx.x];
    p.hist[(size_t)threadIdx.x * p.tileCap + blockIdx.x] = c;
    if (c) {
        atomicAdd(&p.binTotal[pass * 256 + threadIdx.x], c);
    }
}

/* pass `pass`, one CTA per digit value d: hist[d][t] becomes the position of tile t's first record of
 * digit d (the records of smaller digits, then those of d in earlier tiles) */
__global__ void __launch_bounds__(ORDER_THREADS) histScanKernel(const OrderParams p, u32 pass) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    const OrderState *st = p.st;
    if (pass >= st->passes) {
        return;
    }
    const u32 d = blockIdx.x, ntiles = tilesOf(st->m);
    u32 total;
    blockExclusive(threadIdx.x < d ? p.binTotal[pass * 256 + threadIdx.x] : 0, sm, &total);
    u32 carry = total;
    u32 *row = p.hist + (size_t)d * p.tileCap;
    for (u32 b = 0; b < ntiles; b += blockDim.x) {
        const u32 t = b + threadIdx.x;
        const u32 v = t < ntiles ? row[t] : 0;
        const u32 ex = blockExclusive(v, sm, &total);
        if (t < ntiles) {
            row[t] = carry + ex;
        }
        carry += total;
    }
}

/* pass `pass`: move the tile's records from buf[pass & 1] to their places in buf[~pass & 1], keeping
 * the order of equal digits (a round at a time: within a warp by the lanes that share the digit,
 * across warps by the warps' counts) */
__global__ void __launch_bounds__(ORDER_THREADS) radixScatterKernel(const OrderParams p, u32 pass) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *binBase = reinterpret_cast<u32 *>(smem);            /* [256] */
    u32 *warpCnt = binBase + 256;                            /* [warps][256] */
    const OrderState *st = p.st;
    const u32 m = st->m, base = blockIdx.x * ORDER_TILE;
    if (pass >= st->passes || base >= m) {
        return;
    }
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = ORDER_THREADS / 32;
    const KeyLayout key = keyOf(st);
    const DevMatch *src = p.buf[pass & 1];
    DevMatch *dst = p.buf[(pass + 1) & 1];
    binBase[threadIdx.x] = p.hist[(size_t)threadIdx.x * p.tileCap + blockIdx.x];
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        for (u32 w = 0; w < nwarps; w++) {
            warpCnt[w * 256 + threadIdx.x] = 0;
        }
        __syncthreads();
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        const bool valid = i < m;
        DevMatch r;
        u32 d = 0;
        if (valid) {
            r = src[i];
            d = key.digit(r, pass);
        }
        /* lanes holding the same digit: AND of the ballots of every digit bit, agreeing */
        u32 peers = __ballot_sync(FULL, valid);
        for (u32 b = 0; b < 8; b++) {
            const u32 bit = (d >> b) & 1;
            const u32 set = __ballot_sync(FULL, bit);
            peers &= bit ? set : ~set;
        }
        const u32 below = __popc(peers & ((1u << lane) - 1));
        if (valid && below == 0) {
            warpCnt[warp * 256 + d] = (u32)__popc(peers);
        }
        __syncthreads();
        {   /* thread d: the warps' first positions of digit d, and the next round's base */
            u32 run = binBase[threadIdx.x];
            for (u32 w = 0; w < nwarps; w++) {
                const u32 c = warpCnt[w * 256 + threadIdx.x];
                warpCnt[w * 256 + threadIdx.x] = run;
                run += c;
            }
            binBase[threadIdx.x] = run;
        }
        __syncthreads();
        if (valid) {
            dst[warpCnt[warp * 256 + d] + below] = r;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ u64 exHash(u64 key) {
    key ^= key >> 33;
    key *= 0xff51afd7ed558ccdull;
    key ^= key >> 33;
    return key;
}

/* the sorted records after the last pass */
__device__ __forceinline__ const DevMatch *sorted(const OrderParams &p) { return p.buf[p.st->passes & 1]; }

/* exhaustible id of a sorted record: its (block, rank) key, or EX_EMPTY */
__device__ __forceinline__ u64 exKeyOf(const OrderParams &p, const DevMatch &r) {
    const int rank = p.st->unknownIds ? rankOf(p, r.id) : (int)r.id;
    if (rank < 0 || !__ldg(p.idEx + rank)) {
        return EX_EMPTY;
    }
    return ((u64)r.block << 32) | (u32)rank;
}

/* the lowest sorted position of every exhaustible (block, id) */
__global__ void __launch_bounds__(ORDER_THREADS) exInsertKernel(const OrderParams p) {
    const u32 m = p.st->m, base = blockIdx.x * ORDER_TILE;
    if (base >= m) {
        return;
    }
    const DevMatch *s = sorted(p);
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        if (i >= m) {
            continue;
        }
        const u64 key = exKeyOf(p, s[i]);
        if (key == EX_EMPTY) {
            continue;
        }
        for (u32 slot = (u32)exHash(key) & (p.exSlots - 1);; slot = (slot + 1) & (p.exSlots - 1)) {
            const u64 prev = casKey(&p.exKey[slot], EX_EMPTY, key);
            if (prev == EX_EMPTY || prev == key) {
                atomicMin(&p.exFirst[slot], i);
                break;
            }
        }
    }
}

/* is sorted record i delivered: not equal to its predecessor, and the first of its (block, id) if the
 * id is exhaustible */
__device__ bool keep(const OrderParams &p, const DevMatch *s, u32 i) {
    const DevMatch r = s[i];
    if (i > 0) {
        const DevMatch q = s[i - 1];
        if (q.block == r.block && q.to == r.to && q.id == r.id) {
            return false;
        }
    }
    if (!p.anyEx) {
        return true;
    }
    const u64 key = exKeyOf(p, r);
    if (key == EX_EMPTY) {
        return true;
    }
    for (u32 slot = (u32)exHash(key) & (p.exSlots - 1);; slot = (slot + 1) & (p.exSlots - 1)) {
        if (p.exKey[slot] == key) {
            return p.exFirst[slot] == i;
        }
    }
}

__global__ void __launch_bounds__(ORDER_THREADS) keepCountKernel(const OrderParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    const u32 m = p.st->m, base = blockIdx.x * ORDER_TILE;
    if (base >= m) {
        return;
    }
    const DevMatch *s = sorted(p);
    u32 c = 0;
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        c += i < m && keep(p, s, i);
    }
    u32 total;
    blockExclusive(c, sm, &total);
    if (threadIdx.x == 0) {
        p.tileSum[blockIdx.x] = total;
    }
}

/* the kept records, ids restored from their ranks, into out[0, outCap) */
__global__ void __launch_bounds__(ORDER_THREADS) compactKernel(const OrderParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    const u32 m = p.st->m, base = blockIdx.x * ORDER_TILE;
    if (base >= m) {
        return;
    }
    const DevMatch *s = sorted(p);
    const bool raw = p.st->unknownIds != 0;
    u64 run = p.tileSum[blockIdx.x];
    for (u32 k = 0; k < ORDER_ITEMS; k++) {
        const u32 i = base + k * ORDER_THREADS + threadIdx.x;
        const bool kept = i < m && keep(p, s, i);
        u32 total;
        const u64 pos = run + blockExclusive(kept, sm, &total);
        run += total;
        if (kept && pos < p.outCap) {
            DevMatch r = s[i];
            if (!raw) {
                r.id = __ldg(p.ids + r.id);
            }
            p.out[pos] = r;
        }
    }
}

} // namespace

cudaError_t launchOrder(const OrderParams &p, u32 maxPasses, cudaStream_t stream, unsigned *launches) {
    const size_t scanSmem = 33 * sizeof(u32);
    const u32 inTiles = (std::max(p.inCap, p.inN) + ORDER_TILE - 1) / ORDER_TILE;
    const u32 bufTiles = (p.bufCap + ORDER_TILE - 1) / ORDER_TILE;
    unsigned n = 0;
    cudaError_t e = cudaSuccess;
    auto check = [&]() {
        n++;
        if (e == cudaSuccess) {
            e = cudaGetLastError();
        }
    };
    HSB_LAUNCH(orderSetupKernel, 1, ORDER_THREADS, 0, stream, p);
    check();
    if (inTiles) {
        if (p.shape != SHAPE_PURE_LITERAL) {
            HSB_LAUNCH(resolveCountKernel, inTiles, ORDER_THREADS, scanSmem, stream, p);
            check();
            HSB_LAUNCH(tileScanKernel, 1, 1024, scanSmem, stream, p, 0u);
            check();
        }
        HSB_LAUNCH(resolveScatterKernel, inTiles, ORDER_THREADS, scanSmem, stream, p);
        check();
    }
    if (bufTiles) {
        HSB_LAUNCH(rankKernel, bufTiles, ORDER_THREADS, 0, stream, p);
        check();
        for (u32 pass = 0; pass < maxPasses && pass < ORDER_MAX_PASSES; pass++) {
            HSB_LAUNCH(histKernel, bufTiles, ORDER_THREADS, 256 * sizeof(u32), stream, p, pass);
            check();
            HSB_LAUNCH(histScanKernel, 256, ORDER_THREADS, scanSmem, stream, p, pass);
            check();
            HSB_LAUNCH(radixScatterKernel, bufTiles, ORDER_THREADS, (256 + 256 * ORDER_THREADS / 32) * sizeof(u32),
                       stream, p, pass);
            check();
        }
        if (p.anyEx) {
            HSB_LAUNCH(exInsertKernel, bufTiles, ORDER_THREADS, 0, stream, p);
            check();
        }
        HSB_LAUNCH(keepCountKernel, bufTiles, ORDER_THREADS, scanSmem, stream, p);
        check();
    }
    HSB_LAUNCH(tileScanKernel, 1, 1024, scanSmem, stream, p, 1u);
    check();
    if (bufTiles) {
        HSB_LAUNCH(compactKernel, bufTiles, ORDER_THREADS, scanSmem, stream, p);
        check();
    }
    *launches = n;
    return e;
}

} // namespace hsb
#endif
