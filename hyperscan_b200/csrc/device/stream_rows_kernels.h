/*
 * stream_rows_kernels.h -- stream-set passes over rows (hs_b200_streams_scan_rows_async) on the device: a batch of
 * rows in device memory, each tagged with the stream it is written to, in arrival order, becomes one block per
 * distinct stream of the batch (a group): the stream's look-behind, then its rows in row order, concatenated byte
 * for byte, so that a match may span rows.  The scan kernels read it as an ordinary block-table corpus; the records
 * are then mapped back to rows and stream offsets, and the streams of the batch advance.  The host knows only the
 * row count, the chars' size and the set's stream count.
 *
 *   sort      (stream, row) pairs, stable LSD radix sort by the stream, 8-bit digits, as many passes as the set's
 *             stream count needs: per tile the count of every digit, one warp per digit value scans the tiles'
 *             counts, and the scatter keeps the order of equal digits (order_kernels.h's scheme).  A stream id at
 *             or above nstreams fails the batch.
 *   groups    over the sorted rows: each row's length (a bad row fails the batch) and whether it starts a group;
 *             tile sums, one CTA scans them, then every sorted row gets its group and the bytes before it
 *             (posOf), and every group its first row, stream and first position.
 *   blocks    per group: look-behind (read from the set's state when the pass runs, so that passes enqueued back
 *             to back see each other's commits) plus its rows' bytes, padded to 16 (16 for an empty block); tile
 *             sums, one CTA scans them and takes the verdict (a bad batch marks the pass bad before the scan: every
 *             block is empty); then every group's block goes to the table, its look-behind and its pad into the
 *             corpus.  The table's entries past the last group are empty blocks 16 bytes apart behind it; the slack
 *             up to zeroEnd gets zeros.
 *   copy      a warp per row: the 16-byte words wholly inside the row's destination are assembled from two aligned
 *             loads (rows_kernels.h), the partial words at its two ends are written byte by byte (they are shared
 *             with the neighbouring rows).  Nothing outside [chars, chars + charsBytes) is read.
 *   rewrite   (after the scan, when the pass may commit) a record that ends in the look-behind goes (an earlier pass
 *             delivered it); the others get block = the row holding their last byte (a binary search over the
 *             group's rows, streamRowAt: an empty row holds no byte) and to = their stream offset.  The kept
 *             records are gathered in the ring's second half, then copied back with their count.  A mask pass
 *             (hs_b200_streams_scan_rows_mask_async) writes no records and skips this step: its confirm kernel
 *             drops the same ends and maps each match to its row with the same search as it sets the bit.
 *   advance   streamPassCommits' verdict; per group, the last histReq bytes of its block become the stream's
 *             look-behind and its rows' bytes are added to the stream's offset.
 *
 * No CUB or Thrust, and only the intrinsics the SIMT emulator of tests/emu models.  Included once, by api_device.cu,
 * after order_kernels.h and rows_kernels.h (whose blockExclusive, rowsExclusive, loadInside and bytesFrom it uses).
 */
#ifndef HSB200_STREAM_ROWS_KERNELS_H
#define HSB200_STREAM_ROWS_KERNELS_H

#include <cuda_runtime.h>

#include "kernels.h"

namespace hsb {

namespace {

__device__ __forceinline__ u32 srTiles(u32 n) { return (u32)(((u64)n + ROWS_TILE - 1) / ROWS_TILE); }

/* the (stream, row) pairs after the last radix pass */
__device__ __forceinline__ const uint2 *srSorted(const StreamRowsParams &p) { return p.pairs[p.passes & 1]; }

__device__ __forceinline__ u32 srDigit(uint2 e, u32 pass) { return (e.x >> (8 * pass)) & 0xff; }

/* row r's length; a row that decreases, ends past charsBytes or holds 4 GiB or more is empty and sets *bad */
__device__ __forceinline__ u32 srRowLen(const StreamRowsParams &p, u32 r, u32 *bad) {
    const u64 lo = p.offsets[r], hi = p.offsets[r + 1];
    if (hi < lo || hi > p.charsBytes || hi - lo > 0xffffffffull) {
        *bad = 1;
        return 0;
    }
    return (u32)(hi - lo);
}

__device__ __forceinline__ u64 srGroupBytes(const StreamRowsParams &p, u32 g) { return p.gPos[g + 1] - p.gPos[g]; }

/* the look-behind bytes stream s holds */
__device__ __forceinline__ u32 srHl(const StreamRowsParams &p, u32 s) { return p.lookBehind[(size_t)s * 8 + 7]; }

/* ---- sort ---- */

__global__ void __launch_bounds__(ROWS_THREADS) srInitKernel(const StreamRowsParams p) {
    u32 bad = 0;
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 i = (u64)blockIdx.x * ROWS_TILE + k * ROWS_THREADS + threadIdx.x;
        if (i < p.nrows) {
            u32 s = p.ids[i];
            if (s >= p.nstreams) { /* the batch fails; the row stays inside the set until then */
                bad = 1;
                s = 0;
            }
            p.pairs[0][i] = make_uint2(s, (u32)i);
        }
    }
    if (bad) {
        p.head->bad = 1;
    }
}

/* pass `pass`: per tile, the count of every digit value (tileDigits[d][tile]) and their totals */
__global__ void __launch_bounds__(ROWS_THREADS) srDigitKernel(const StreamRowsParams p, u32 pass) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *h = reinterpret_cast<u32 *>(smem);
    const uint2 *src = p.pairs[pass & 1];
    const u32 tiles = srTiles(p.nrows);
    h[threadIdx.x] = 0;
    __syncthreads();
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 i = (u64)blockIdx.x * ROWS_TILE + k * ROWS_THREADS + threadIdx.x;
        if (i < p.nrows) {
            atomicAdd(&h[srDigit(src[i], pass)], 1u);
        }
    }
    __syncthreads();
    const u32 c = h[threadIdx.x];
    p.tileDigits[(size_t)threadIdx.x * tiles + blockIdx.x] = c;
    if (c) {
        atomicAdd(&p.head->digits[pass * 256 + threadIdx.x], c);
    }
}

/* pass `pass`, one warp per digit value d: tileDigits[d][t] becomes the position of tile t's first pair of digit d */
__global__ void __launch_bounds__(32) srDigitScanKernel(const StreamRowsParams p, u32 pass) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    const u32 d = blockIdx.x, tiles = srTiles(p.nrows);
    u32 below = 0; /* the pairs of smaller digits */
    for (u32 j = threadIdx.x; j < d; j += blockDim.x) {
        below += p.head->digits[pass * 256 + j];
    }
    u32 total;
    blockExclusive(below, sm, &total);
    u32 carry = total;
    u32 *row = p.tileDigits + (size_t)d * tiles;
    for (u32 b = 0; b < tiles; b += blockDim.x) {
        const u32 t = b + threadIdx.x;
        const u32 v = t < tiles ? row[t] : 0u;
        const u32 ex = blockExclusive(v, sm, &total);
        if (t < tiles) {
            row[t] = carry + ex;
        }
        carry += total;
    }
}

/* pass `pass`: the tile's pairs from pairs[pass & 1] to their places in pairs[~pass & 1], equal digits in order (a
 * round at a time: within a warp by the lanes that share the digit, across warps by the warps' counts) */
__global__ void __launch_bounds__(ROWS_THREADS) srScatterKernel(const StreamRowsParams p, u32 pass) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *binBase = reinterpret_cast<u32 *>(smem); /* [256] */
    u32 *warpCnt = binBase + 256;                 /* [warps][256] */
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = ROWS_THREADS / 32;
    const uint2 *src = p.pairs[pass & 1];
    uint2 *dst = p.pairs[(pass + 1) & 1];
    binBase[threadIdx.x] = p.tileDigits[(size_t)threadIdx.x * srTiles(p.nrows) + blockIdx.x];
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        for (u32 w = 0; w < nwarps; w++) {
            warpCnt[w * 256 + threadIdx.x] = 0;
        }
        __syncthreads();
        const u64 i = (u64)blockIdx.x * ROWS_TILE + k * ROWS_THREADS + threadIdx.x;
        const bool valid = i < p.nrows;
        uint2 e = make_uint2(0, 0);
        u32 d = 0;
        if (valid) {
            e = src[i];
            d = srDigit(e, pass);
        }
        u32 peers = __ballot_sync(0xffffffffu, valid);
        for (u32 b = 0; b < 8; b++) {
            const u32 bit = (d >> b) & 1;
            const u32 set = __ballot_sync(0xffffffffu, bit);
            peers &= bit ? set : ~set;
        }
        const u32 below = __popc(peers & ((1u << lane) - 1));
        if (valid && below == 0) {
            warpCnt[warp * 256 + d] = (u32)__popc(peers);
        }
        __syncthreads();
        {
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
            dst[warpCnt[warp * 256 + d] + below] = e;
        }
        __syncthreads();
    }
}

/* ---- groups ---- */

/* per tile of sorted rows: their bytes and the groups that start in it */
__global__ void __launch_bounds__(ROWS_THREADS) srRowTileKernel(const StreamRowsParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    const uint2 *sorted = srSorted(p);
    const u64 first = (u64)blockIdx.x * ROWS_TILE + (u64)threadIdx.x * ROWS_ITEMS;
    u64 bytes = 0, starts = 0;
    u32 bad = 0;
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 i = first + k;
        if (i < p.nrows) {
            const uint2 e = sorted[i];
            bytes += srRowLen(p, e.y, &bad);
            starts += i == 0 || sorted[i - 1].x != e.x;
        }
    }
    u64 total, totalStarts;
    rowsExclusive(bytes, sm, &total);
    rowsExclusive(starts, sm, &totalStarts);
    if (bad) {
        p.head->bad = 1;
    }
    if (threadIdx.x == 0) {
        p.tileA[blockIdx.x] = total;
        p.tileB[blockIdx.x] = totalStarts;
    }
}

/* one CTA: exclusive scans of the tiles' bytes and group starts in place; the group count, and the end entries */
__global__ void __launch_bounds__(ROWS_THREADS) srRowScanKernel(const StreamRowsParams p, u32 tiles) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    u64 carryA = 0, carryB = 0;
    for (u32 b = 0; b < tiles; b += blockDim.x) {
        const u32 t = b + threadIdx.x;
        u64 totA, totB;
        const u64 exA = rowsExclusive(t < tiles ? p.tileA[t] : 0, sm, &totA);
        const u64 exB = rowsExclusive(t < tiles ? p.tileB[t] : 0, sm, &totB);
        if (t < tiles) {
            p.tileA[t] = carryA + exA;
            p.tileB[t] = carryB + exB;
        }
        carryA += totA;
        carryB += totB;
    }
    if (threadIdx.x == 0) {
        p.head->groups = (u32)carryB;
        p.gFirst[carryB] = p.nrows;
        p.gPos[carryB] = carryA;
    }
}

/* every sorted row's group and position; every group's first row, stream and position */
__global__ void __launch_bounds__(ROWS_THREADS) srRowWriteKernel(const StreamRowsParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    const uint2 *sorted = srSorted(p);
    const u64 first = (u64)blockIdx.x * ROWS_TILE + (u64)threadIdx.x * ROWS_ITEMS;
    u64 bytes = 0, starts = 0;
    u32 bad = 0;
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 i = first + k;
        if (i < p.nrows) {
            const uint2 e = sorted[i];
            bytes += srRowLen(p, e.y, &bad);
            starts += i == 0 || sorted[i - 1].x != e.x;
        }
    }
    u64 total;
    u64 at = p.tileA[blockIdx.x] + rowsExclusive(bytes, sm, &total);
    u32 g = (u32)(p.tileB[blockIdx.x] + rowsExclusive(starts, sm, &total)); /* groups started before */
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 i = first + k;
        if (i >= p.nrows) {
            break;
        }
        const uint2 e = sorted[i];
        if (i == 0 || sorted[i - 1].x != e.x) {
            p.gFirst[g] = (u32)i;
            p.gPos[g] = at;
            p.gStream[g] = e.x;
            g++;
        }
        p.groupOf[i] = g - 1;
        p.posOf[i] = at;
        at += srRowLen(p, e.y, &bad);
    }
}

/* ---- blocks ---- */

/* group g's block: look-behind plus its rows' bytes (*len), and its padded size */
__device__ __forceinline__ u64 srBlockPad(const StreamRowsParams &p, u32 g, u64 *len, u32 *hl) {
    *hl = srHl(p, p.gStream[g]);
    *len = *hl + srGroupBytes(p, g);
    return *len ? HSB_ROUNDUP(*len, 16) : 16;
}

/* per tile of groups: their blocks' padded sizes; a block past 32 bits fails the batch */
__global__ void __launch_bounds__(ROWS_THREADS) srGroupTileKernel(const StreamRowsParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    const u32 groups = p.head->groups;
    const u64 first = (u64)blockIdx.x * ROWS_TILE + (u64)threadIdx.x * ROWS_ITEMS;
    u64 pad = 0;
    u32 bad = 0;
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 g = first + k;
        if (g < groups) {
            u64 len;
            u32 hl;
            pad += srBlockPad(p, (u32)g, &len, &hl);
            bad |= len > 0xffffffffull;
        }
    }
    u64 total;
    rowsExclusive(pad, sm, &total);
    if (bad) {
        p.head->bad = 1;
    }
    if (threadIdx.x == 0) {
        p.tileA[blockIdx.x] = total;
    }
}

/* one CTA: exclusive scan of the tiles' padded sizes in place, the packed end, and the verdict: a bad batch marks
 * the pass bad (streamPassCommits then marks the set) and leaves every block empty */
__global__ void __launch_bounds__(ROWS_THREADS) srGroupScanKernel(const StreamRowsParams p, u32 tiles) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    u64 carry = 0;
    for (u32 b = 0; b < tiles; b += blockDim.x) {
        const u32 t = b + threadIdx.x;
        u64 total;
        const u64 ex = rowsExclusive(t < tiles ? p.tileA[t] : 0, sm, &total);
        if (t < tiles) {
            p.tileA[t] = carry + ex;
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        const bool bad = p.head->bad != 0;
        p.head->packedEnd = bad ? 0 : carry;
        if (bad) {
            p.mark->bad = p.epoch + 1;
        }
    }
}

/* every group's block into the table, its look-behind and pad into the corpus; empty entries past the last group;
 * zeros from the packed end to zeroEnd */
__global__ void __launch_bounds__(ROWS_THREADS) srGroupWriteKernel(const StreamRowsParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    const u32 groups = p.head->groups;
    const bool bad = p.head->bad != 0;
    const u64 end = p.head->packedEnd;
    const u64 first = (u64)blockIdx.x * ROWS_TILE + (u64)threadIdx.x * ROWS_ITEMS;
    u64 pad = 0;
    for (u32 k = 0; k < ROWS_ITEMS && !bad; k++) {
        const u64 g = first + k;
        if (g < groups) {
            u64 len;
            u32 hl;
            pad += srBlockPad(p, (u32)g, &len, &hl);
        }
    }
    u64 total;
    u64 at = p.tileA[blockIdx.x] + rowsExclusive(pad, sm, &total);
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 g = first + k;
        if (g >= p.nrows) {
            break;
        }
        if (bad || g >= groups) {
            p.blockOff[g] = bad ? 16 * g : end + 16 * (g - groups);
            p.blockLen[g] = 0;
            continue;
        }
        u64 len;
        u32 hl;
        const u64 next = at + srBlockPad(p, (u32)g, &len, &hl);
        const u32 s = p.gStream[g];
        p.blockOff[g] = at;
        p.blockLen[g] = (u32)len;
        p.gHl[g] = hl;
        p.gBase[g] = p.streamOffset[s] - hl;
        for (u32 j = 0; j < hl; j++) {
            p.corpus[at + j] = p.lookBehind[(size_t)s * 8 + j];
        }
        for (u64 q = at + len; q < next; q++) {
            p.corpus[q] = 0;
        }
        at = next;
    }
    const u64 threads = (u64)gridDim.x * blockDim.x;
    for (u64 q = end + 16 * ((u64)blockIdx.x * blockDim.x + threadIdx.x); q < p.zeroEnd; q += 16 * threads) {
        *reinterpret_cast<uint4 *>(p.corpus + q) = make_uint4(0, 0, 0, 0);
    }
}

/* a warp per sorted row: its bytes to their place in its group's block */
__global__ void __launch_bounds__(ROWS_THREADS) srCopyKernel(const StreamRowsParams p) {
    if (p.head->bad) {
        return;
    }
    const u32 lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
    const u64 warps = (u64)gridDim.x * wpc;
    const uint2 *sorted = srSorted(p);
    const uintptr_t lo = (uintptr_t)p.chars, hi = lo + p.charsBytes;
    for (u64 k = (u64)blockIdx.x * wpc + (threadIdx.x >> 5); k < p.nrows; k += warps) {
        const u32 r = sorted[k].y, g = p.groupOf[k];
        const u64 from = p.offsets[r], end = p.offsets[r + 1]; /* checked: the batch is good */
        const u64 dst = p.blockOff[g] + p.gHl[g] + (p.posOf[k] - p.gPos[g]), dstEnd = dst + (end - from);
        for (u64 w = (dst & ~15ull) + lane * 16; w < dstEnd; w += 512) {
            if (w >= dst && w + 16 <= dstEnd) {
                const uintptr_t src = lo + (uintptr_t)(from + (w - dst)), a = src & ~(uintptr_t)15;
                const u32 sh = (u32)(src & 15);
                const uint4 x = loadInside(a, lo, hi);
                const uint4 y = sh ? loadInside(a + 16, lo, hi) : make_uint4(0, 0, 0, 0);
                *reinterpret_cast<uint4 *>(p.corpus + w) = bytesFrom(x, y, sh);
            } else { /* a word shared with the neighbouring rows, the look-behind or the pad */
                const u64 q0 = w > dst ? w : dst, q1 = w + 16 < dstEnd ? w + 16 : dstEnd;
                for (u64 q = q0; q < q1; q++) {
                    p.corpus[q] = p.chars[from + (q - dst)];
                }
            }
        }
    }
}

/* ---- after the scan ---- */

/* when the pass may commit: every record that ends past its block's look-behind, mapped to its row and stream
 * offset, into the ring's second half */
__global__ void __launch_bounds__(ROWS_THREADS) srRewriteKernel(const StreamRowsParams p) {
    if (!streamPassCommits(p.counters, p.outCap, p.mark, p.epoch, false)) {
        return;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        p.head->applied = 1;
    }
    const u32 n = p.counters[CTR_MATCHES];
    const uint2 *sorted = srSorted(p);
    const u64 threads = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += threads) {
        DevMatch m = p.out[i];
        const u32 g = m.block, hl = p.gHl[g];
        if (m.to <= hl) {
            continue;
        }
        m.block = sorted[streamRowAt(p.gFirst, p.posOf, g, p.gPos[g] + (m.to - 1 - hl))].y;
        m.to += p.gBase[g];
        p.out[p.outCap + atomicAdd(&p.head->kept, 1u)] = m;
    }
}

/* the kept records back to the front of the ring, and their count */
__global__ void __launch_bounds__(ROWS_THREADS) srCompactKernel(const StreamRowsParams p) {
    if (!p.head->applied) {
        return;
    }
    const u32 n = p.head->kept;
    const u64 threads = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += threads) {
        p.out[i] = p.out[p.outCap + i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        p.counters[CTR_MATCHES] = n;
    }
}

/* per group, when the pass may commit: maintainHistoryBuffer (src/runtime.c:478-508) over its block, and the
 * stream's offset */
__global__ void __launch_bounds__(ROWS_THREADS) srAdvanceKernel(const StreamRowsParams p) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (!streamPassCommits(p.counters, p.outCap, p.mark, p.epoch, g == 0) || g >= p.head->groups) {
        return;
    }
    const u64 bytes = srGroupBytes(p, (u32)g);
    if (!bytes) {
        return;
    }
    const u32 s = p.gStream[g];
    const u64 total = p.gHl[g] + bytes;
    const u32 keep = total < p.histReq ? (u32)total : p.histReq;
    const u8 *end = p.corpus + p.blockOff[g] + total;
    u64 v = 0;
    for (u32 i = 0; i < keep; i++) {
        v |= (u64)end[(int)i - (int)keep] << (8 * i);
    }
    v |= (u64)keep << 56;
    *reinterpret_cast<uint2 *>(p.lookBehind + (size_t)s * 8) = make_uint2((u32)v, (u32)(v >> 32));
    p.streamOffset[s] += bytes;
}

/* a batch of no rows: nothing to scan, but the pass still takes the set's verdict, so that a set marked or bad in
 * this epoch keeps its pass from committing and reporting success */
__global__ void srVerdictKernel(u32 *counters, u32 outCap, StreamMark *mark, u32 epoch) {
    streamPassCommits(counters, outCap, mark, epoch, true);
}

} // namespace

cudaError_t launchStreamVerdict(u32 *counters, u32 outCap, StreamMark *mark, u32 epoch, cudaStream_t stream) {
    HSB_LAUNCH(srVerdictKernel, 1, 1, 0, stream, counters, outCap, mark, epoch);
    return cudaGetLastError();
}

cudaError_t launchStreamRowsPlan(const StreamRowsParams &p, int smCount, cudaStream_t stream, unsigned *launches) {
    *launches = 0;
    if (!p.nrows) {
        return cudaSuccess;
    }
    const u32 tiles = (u32)(((u64)p.nrows + ROWS_TILE - 1) / ROWS_TILE);
    const size_t sm32 = 33 * sizeof(u32), sm64 = 33 * sizeof(u64);
    unsigned n = 0;
    HSB_LAUNCH(srInitKernel, tiles, ROWS_THREADS, 0, stream, p);
    n++;
    for (u32 pass = 0; pass < p.passes; pass++) {
        HSB_LAUNCH(srDigitKernel, tiles, ROWS_THREADS, 256 * sizeof(u32), stream, p, pass);
        HSB_LAUNCH(srDigitScanKernel, 256, 32, sm32, stream, p, pass);
        HSB_LAUNCH(srScatterKernel, tiles, ROWS_THREADS, (256 + 256 * ROWS_THREADS / 32) * sizeof(u32), stream, p,
                   pass);
        n += 3;
    }
    HSB_LAUNCH(srRowTileKernel, tiles, ROWS_THREADS, sm64, stream, p);
    HSB_LAUNCH(srRowScanKernel, 1, ROWS_THREADS, sm64, stream, p, tiles);
    HSB_LAUNCH(srRowWriteKernel, tiles, ROWS_THREADS, sm64, stream, p);
    HSB_LAUNCH(srGroupTileKernel, tiles, ROWS_THREADS, sm64, stream, p);
    HSB_LAUNCH(srGroupScanKernel, 1, ROWS_THREADS, sm64, stream, p, tiles);
    HSB_LAUNCH(srGroupWriteKernel, tiles, ROWS_THREADS, sm64, stream, p);
    const u64 wpc = ROWS_THREADS / 32;
    const u64 grid = std::min<u64>(((u64)p.nrows + wpc - 1) / wpc, (u64)smCount * 16);
    HSB_LAUNCH(srCopyKernel, (unsigned)grid, ROWS_THREADS, 0, stream, p);
    *launches = n + 7;
    return cudaGetLastError();
}

cudaError_t launchStreamRowsCommit(const StreamRowsParams &p, bool mask, int smCount, cudaStream_t stream,
                                   unsigned *launches) {
    *launches = 0;
    if (!p.nrows) {
        return cudaSuccess;
    }
    if (!mask) { /* a mask pass set its rows' bits in the scan: it has no records to rewrite */
        const u64 grid = std::min<u64>(((u64)p.outCap + ROWS_THREADS - 1) / ROWS_THREADS, (u64)smCount * 8);
        HSB_LAUNCH(srRewriteKernel, (unsigned)grid, ROWS_THREADS, 0, stream, p);
        HSB_LAUNCH(srCompactKernel, (unsigned)grid, ROWS_THREADS, 0, stream, p);
        *launches = 2;
    }
    HSB_LAUNCH(srAdvanceKernel, (unsigned)(((u64)p.nrows + ROWS_THREADS - 1) / ROWS_THREADS), ROWS_THREADS, 0, stream,
               p);
    *launches += 1;
    return cudaGetLastError();
}

StreamRowsMap streamRowsMap(const StreamRowsParams &p) {
    StreamRowsMap m;
    m.sorted = p.pairs[p.passes & 1]; /* srSorted */
    m.posOf = p.posOf;
    m.gPos = p.gPos;
    m.gFirst = p.gFirst;
    m.gHl = p.gHl;
    return m;
}

} // namespace hsb
#endif
