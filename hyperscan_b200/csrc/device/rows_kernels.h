/*
 * rows_kernels.h -- row scans (hs_b200_scan_rows_async) on the device: a column of rows in device memory -- chars
 * plus an offsets array, every row at any byte -- becomes the packed corpus the scan kernels read (ScanParams:
 * blocks 16-byte aligned, zeros between them and after the last) with its block table, and, for engine runs that
 * cut rows into segments, the segment plan.  The host knows only the row count and the chars' size.
 *
 *   plan      per tile of ROWS_TILE rows: check the offsets and sum the rows' padded sizes (the length rounded up
 *             to 16, and 16 for an empty row); one CTA scans the tile sums and takes the verdict; then every row's
 *             packed start and length go to the block table.  A bad table (an offset below the one before, an end
 *             past charsBytes, a row of 4 GiB or more) leaves every row empty and fails the pass: CTR_STREAM gets
 *             STREAM_BAD_LENGTH and the record count is raised above the ring before the scan runs, the protocol
 *             of the stream sets' bad lengths.
 *   repack    a warp per ROWS_SPAN bytes of the packed corpus, 512 bytes a step: the lanes load the table entries
 *             of the 32 rows from the step's first on (blocks start at least 16 bytes apart, so a step crosses at
 *             most 31 row starts), each lane finds the row of its 16 bytes among them by shuffles, loads the two
 *             aligned 16-byte words that hold them, shifts in registers and stores 16 bytes.  Pads and the slack
 *             up to the host's bound get zeros.  A word that reaches outside [chars, chars + charsBytes) is read
 *             byte by byte, inside only.
 *   segments  (engine runs that cut rows, launchEngine) one CTA numbers every row's segments and writes the cut
 *             list; a grid-stride kernel writes the segment table.  Entries past the real end, in lists sized by
 *             the host's bound, are empty first segments of row 0 and cuts of no segments at segment 0, which
 *             every pass of launchDfaSegments walks as nothing.
 *
 * No CUB or Thrust, and only the intrinsics the SIMT emulator of tests/emu models.  Included once, by
 * api_device.cu, after order_kernels.h (whose blockExclusive it uses).
 */
#ifndef HSB200_ROWS_KERNELS_H
#define HSB200_ROWS_KERNELS_H

#include <cuda_runtime.h>

#include "kernels.h"

namespace hsb {

namespace {

__device__ __forceinline__ u64 shflUp64(u64 v, u32 d) {
    const u32 lo = __shfl_up_sync(0xffffffffu, (u32)v, d), hi = __shfl_up_sync(0xffffffffu, (u32)(v >> 32), d);
    return ((u64)hi << 32) | lo;
}

/* exclusive prefix of v over the block (at most 32 warps) in thread order; *total the block's sum.  sm: 33 words. */
__device__ u64 rowsExclusive(u64 v, u64 *sm, u64 *total) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    u64 x = v;
    for (u32 o = 1; o < 32; o <<= 1) {
        const u64 y = shflUp64(x, o);
        if (lane >= o) {
            x += y;
        }
    }
    if (lane == 31) {
        sm[warp] = x;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        u64 run = 0;
        for (u32 w = 0; w < nwarps; w++) {
            const u64 t = sm[w];
            sm[w] = run;
            run += t;
        }
        sm[32] = run;
    }
    __syncthreads();
    const u64 r = sm[warp] + x - v;
    *total = sm[32];
    __syncthreads();
    return r;
}

/* row i: its length and padded size, or bad */
struct RowFacts {
    u64 pad;
    u32 len;
    u32 bad;
};

__device__ __forceinline__ RowFacts rowFacts(const RowsParams &p, u64 i) {
    const u64 lo = p.offsets[i], hi = p.offsets[i + 1];
    RowFacts f;
    f.bad = hi < lo || hi > p.charsBytes || hi - lo > 0xffffffffull;
    f.len = f.bad ? 0u : (u32)(hi - lo);
    f.pad = f.len ? HSB_ROUNDUP((u64)f.len, 16) : 16;
    return f;
}

/* per tile: the sum of its rows' padded sizes, and whether one of them is bad */
__global__ void __launch_bounds__(ROWS_THREADS) rowsTileKernel(const RowsParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    const u64 first = (u64)blockIdx.x * ROWS_TILE + (u64)threadIdx.x * ROWS_ITEMS;
    u64 pad = 0;
    u32 bad = 0;
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        if (first + k < p.nrows) {
            const RowFacts f = rowFacts(p, first + k);
            pad += f.pad;
            bad |= f.bad;
        }
    }
    u64 total, anyBad;
    rowsExclusive(pad, sm, &total);
    rowsExclusive(bad, sm, &anyBad);
    if (threadIdx.x == 0) {
        p.tilePad[blockIdx.x] = total;
        p.tileBad[blockIdx.x] = (u32)anyBad;
    }
}

/* exclusive scan of the tile sums in place, and the verdict; a bad table fails the pass before the scan runs */
__global__ void __launch_bounds__(ROWS_THREADS) rowsScanKernel(const RowsParams p, u32 ntiles) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    u64 carry = 0;
    u32 bad = 0;
    for (u32 b = 0; b < ntiles; b += blockDim.x) {
        const u32 t = b + threadIdx.x;
        const u64 v = t < ntiles ? p.tilePad[t] : 0;
        bad |= t < ntiles ? p.tileBad[t] : 0u;
        u64 total;
        const u64 ex = rowsExclusive(v, sm, &total);
        if (t < ntiles) {
            p.tilePad[t] = carry + ex;
        }
        carry += total;
    }
    u64 anyBad;
    rowsExclusive(bad, sm, &anyBad);
    if (threadIdx.x == 0) {
        *p.bad = (u32)anyBad;
        if (anyBad) {
            p.counters[CTR_STREAM] |= STREAM_BAD_LENGTH;
            /* a multiple of eight: the engine lanes reserve record slots eight at a time */
            p.counters[CTR_MATCHES] = (u32)HSB_ROUNDUP((u64)p.outCap + 1, 8);
        }
    }
}

/* every row's packed start and length into the block table (a bad table: empty rows 16 bytes apart) */
__global__ void __launch_bounds__(ROWS_THREADS) rowsTableKernel(const RowsParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u64 *sm = reinterpret_cast<u64 *>(smem);
    const bool bad = *p.bad != 0;
    const u64 first = (u64)blockIdx.x * ROWS_TILE + (u64)threadIdx.x * ROWS_ITEMS;
    u64 local = 0;
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        if (first + k < p.nrows) {
            local += rowFacts(p, first + k).pad;
        }
    }
    u64 total;
    u64 at = p.tilePad[blockIdx.x] + rowsExclusive(local, sm, &total);
    for (u32 k = 0; k < ROWS_ITEMS; k++) {
        const u64 i = first + k;
        if (i >= p.nrows) {
            break;
        }
        if (bad) {
            p.blockOff[i] = 16 * i;
            p.blockLen[i] = 0;
        } else {
            const RowFacts f = rowFacts(p, i);
            p.blockOff[i] = at;
            p.blockLen[i] = f.len;
            at += f.pad;
        }
    }
}

/* byte b of v |= x */
__device__ __forceinline__ void orByte(uint4 &v, u32 b, u32 x) {
    const u32 s = 8 * (b & 3);
    if (b < 4) {
        v.x |= x << s;
    } else if (b < 8) {
        v.y |= x << s;
    } else if (b < 12) {
        v.z |= x << s;
    } else {
        v.w |= x << s;
    }
}

/* the 16-byte aligned word at w, of which only the bytes inside [lo, hi) are read (the others are 0) */
__device__ __forceinline__ uint4 loadInside(uintptr_t w, uintptr_t lo, uintptr_t hi) {
    if (w >= lo && w + 16 <= hi) {
        return *reinterpret_cast<const uint4 *>(w);
    }
    uint4 v = make_uint4(0, 0, 0, 0);
    for (u32 b = 0; b < 16; b++) {
        if (w + b >= lo && w + b < hi) {
            orByte(v, b, *reinterpret_cast<const u8 *>(w + b));
        }
    }
    return v;
}

/* bytes [sh, sh + 16) of the 32 bytes a ++ b */
__device__ __forceinline__ uint4 bytesFrom(uint4 a, uint4 b, u32 sh) {
    u32 w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x, w5 = b.y, w6 = b.z, w7 = b.w;
    if (sh & 8) {
        w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; w5 = w7;
    }
    if (sh & 4) {
        w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5;
    }
    const u32 s = 8 * (sh & 3);
    return make_uint4(__funnelshift_r(w0, w1, s), __funnelshift_r(w1, w2, s), __funnelshift_r(w2, w3, s),
                      __funnelshift_r(w3, w4, s));
}

__device__ __forceinline__ u32 firstBytes(u32 w, int n) { return n >= 4 ? w : n <= 0 ? 0u : w & ((1u << (8 * n)) - 1); }

__global__ void __launch_bounds__(ROWS_THREADS) rowsRepackKernel(const RowsParams p) {
    const u32 lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
    const u64 spans = (p.zeroEnd + ROWS_SPAN - 1) / ROWS_SPAN, warps = (u64)gridDim.x * wpc;
    const bool bad = *p.bad != 0;
    const uintptr_t lo = (uintptr_t)p.chars, hi = lo + p.charsBytes;
    for (u64 sp = (u64)blockIdx.x * wpc + (threadIdx.x >> 5); sp < spans; sp += warps) {
        const u64 base = sp * ROWS_SPAN;
        u32 r0 = 0, rh = p.nrows; /* the row of `base`: the last one that starts at or before it */
        while (rh - r0 > 1) {
            const u32 mid = r0 + ((rh - r0) >> 1);
            if (p.blockOff[mid] <= base) {
                r0 = mid;
            } else {
                rh = mid;
            }
        }
        for (u32 step = 0; step < ROWS_SPAN / 512; step++) {
            const u64 q = base + step * 512 + lane * 16;
            /* lane j holds row r0 + j, and the row of q is among them: r0 starts at or before the step, and a
             * step crosses at most 31 more row starts; each lane finds its row in the lanes' registers */
            const u32 mine = r0 + lane;
            const bool have = mine < p.nrows;
            const u64 start = have ? p.blockOff[mine] : ~0ull, from = have ? p.offsets[mine] : 0;
            const u32 rowLen = have ? p.blockLen[mine] : 0u;
            u32 j = 0;
            for (u32 d = 16; d; d >>= 1) {
                if (__shfl_sync(0xffffffffu, start, j + d) <= q) {
                    j += d;
                }
            }
            const u64 o = q - __shfl_sync(0xffffffffu, start, j), at = __shfl_sync(0xffffffffu, from, j);
            const u32 len = __shfl_sync(0xffffffffu, rowLen, j);
            uint4 v = make_uint4(0, 0, 0, 0);
            if (!bad && o < len) {
                const int n = len - o < 16 ? (int)(len - o) : 16;
                const uintptr_t src = lo + (uintptr_t)at + (uintptr_t)o, w = src & ~(uintptr_t)15;
                const u32 sh = (u32)(src & 15);
                const uint4 a = loadInside(w, lo, hi);
                const uint4 b = sh + n > 16 ? loadInside(w + 16, lo, hi) : make_uint4(0, 0, 0, 0);
                v = bytesFrom(a, b, sh);
                v.x = firstBytes(v.x, n);
                v.y = firstBytes(v.y, n - 4);
                v.z = firstBytes(v.z, n - 8);
                v.w = firstBytes(v.w, n - 12);
            }
            if (q < p.zeroEnd) {
                *reinterpret_cast<uint4 *>(p.corpus + q) = v;
            }
            r0 += __shfl_sync(0xffffffffu, j, 31);
        }
    }
}

/* the segments of every row, numbered in row order (segFirst), and the cut list; unused cuts: {0, 0} */
__global__ void rowsSegCountKernel(const RowSegParams p) {
    HSB_DYNAMIC_SMEM(smem);
    u32 *sm = reinterpret_cast<u32 *>(smem);
    u32 carry = 0, cutCarry = 0;
    for (u64 b = 0; b < p.nrows; b += blockDim.x) {
        const u64 i = b + threadIdx.x;
        const u32 len = i < p.nrows ? p.blockLen[i] : 0u;
        const bool cut = i < p.nrows && len > p.cutAbove;
        const u32 n = i >= p.nrows ? 0u : cut ? (u32)(((u64)len + p.segLen - 1) / p.segLen) : 1u;
        u32 total, cutTotal;
        const u32 ex = blockExclusive(n, sm, &total);
        const u32 exCut = blockExclusive(cut ? 1u : 0u, sm, &cutTotal);
        if (i < p.nrows) {
            p.segFirst[i] = carry + ex;
            if (cut) {
                p.cuts[cutCarry + exCut] = make_uint2(carry + ex, n);
            }
        }
        carry += total;
        cutCarry += cutTotal;
    }
    if (threadIdx.x == 0) {
        p.segFirst[p.nrows] = carry;
    }
    for (u32 j = cutCarry + threadIdx.x; j < p.cutCap; j += blockDim.x) {
        p.cuts[j] = make_uint2(0, 0);
    }
}

/* the segment table: segment j of the row whose numbers hold it; unused entries: empty first segments of row 0 */
__global__ void __launch_bounds__(ROWS_THREADS) rowsSegWriteKernel(const RowSegParams p) {
    const u32 total = p.segFirst[p.nrows];
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < p.segCap; j += (u64)gridDim.x * blockDim.x) {
        DfaSeg sg = {0, 0, 0, SEG_FIRST};
        if (j < total) {
            u32 r = 0, e = p.nrows;
            while (e - r > 1) {
                const u32 mid = r + ((e - r) >> 1);
                if (p.segFirst[mid] <= j) {
                    r = mid;
                } else {
                    e = mid;
                }
            }
            const u32 k = (u32)j - p.segFirst[r], n = p.segFirst[r + 1] - p.segFirst[r], len = p.blockLen[r];
            const u32 start = k * p.segLen;
            sg.block = r;
            sg.start = n == 1 ? 0u : start;
            sg.len = n == 1 ? len : min(p.segLen, len - start);
            sg.flags = (k == 0 ? (u32)SEG_FIRST : 0u) | (k == n - 1 ? (u32)SEG_LAST : 0u);
        }
        p.segs[j] = sg;
    }
}

} // namespace

cudaError_t launchRowPlan(const RowsParams &p, int smCount, cudaStream_t stream, unsigned *launches) {
    *launches = 0;
    if (!p.nrows) {
        return cudaSuccess;
    }
    const u32 ntiles = (u32)(((u64)p.nrows + ROWS_TILE - 1) / ROWS_TILE);
    const size_t smem = 33 * sizeof(u64);
    HSB_LAUNCH(rowsTileKernel, ntiles, ROWS_THREADS, smem, stream, p);
    HSB_LAUNCH(rowsScanKernel, 1, ROWS_THREADS, smem, stream, p, ntiles);
    HSB_LAUNCH(rowsTableKernel, ntiles, ROWS_THREADS, smem, stream, p);
    const u64 spans = (p.zeroEnd + ROWS_SPAN - 1) / ROWS_SPAN, wpc = ROWS_THREADS / 32;
    const u64 grid = std::min<u64>((spans + wpc - 1) / wpc, (u64)smCount * 16);
    HSB_LAUNCH(rowsRepackKernel, (unsigned)grid, ROWS_THREADS, 0, stream, p);
    *launches = 4;
    return cudaGetLastError();
}

cudaError_t launchRowSegments(const RowSegParams &p, int smCount, cudaStream_t stream, unsigned *launches) {
    *launches = 0;
    if (!p.nrows) {
        return cudaSuccess;
    }
    HSB_LAUNCH(rowsSegCountKernel, 1, 1024, 33 * sizeof(u32), stream, p);
    const u64 grid = std::min<u64>(((u64)p.segCap + ROWS_THREADS - 1) / ROWS_THREADS, (u64)smCount * 8);
    HSB_LAUNCH(rowsSegWriteKernel, (unsigned)grid, ROWS_THREADS, 0, stream, p);
    *launches = 2;
    return cudaGetLastError();
}

} // namespace hsb
#endif
