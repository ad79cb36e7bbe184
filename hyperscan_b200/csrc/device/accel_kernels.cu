/*
 * accel_kernels.cu -- the "skip to the next interesting byte" primitives of the
 * reference (src/nfa/accel.h:46-121, run_accel src/nfa/accel.c:35) as one
 * sm_90a kernel: first position in [0, len) whose byte (pair) is in the class.
 *
 *   vermicelli        src/nfa/vermicelli.h:43-110    byte == c  (nocase: & 0xdf)
 *   double vermicelli src/nfa/vermicelli.h:172-246   c1 at p, c2 at p+1; a
 *                     lone c1 in the last byte is a (partial) hit
 *   shufti            src/nfa/shufti.c:104-150       lo[c & 15] & hi[c >> 4] != 0
 *   truffle           src/nfa/truffle.c:40-118       (c < 0x80 ? m1 : m2)[c & 15]
 *                                                    & (1 << ((c >> 4) & 7)) != 0
 *
 * The 16-entry nibble tables (the reference's pshufb operands) live in four
 * registers each and are indexed with PRMT byte permutes, four input bytes per
 * instruction; each thread classifies 16 bytes from one coalesced uint4 load
 * and the block reduces "first hit" with a ballot + one atomicMin.
 *
 * In the reference these run inside hwlmExec / the NFA engines to skip ahead
 * (src/hwlm/hwlm.c:48-101); on the GPU the literal path does not need a skip
 * (every byte is streamed once at full bandwidth), so they are exported as
 * stand-alone entry points for parity and for the DFA/NFA engines to come.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace hsb {

namespace {

/* PRMT in its default mode: selector nibble bit 3 replicates the selected
 * byte's sign bit (the __byte_perm intrinsic only honours bits 2:0). */
__device__ __forceinline__ u32 prmt(u32 a, u32 b, u32 sel) {
#ifdef HSB_HOST_EMU /* SIMT emulator of tests/emu (test infrastructure) */
    return hsb_emu_prmt(a, b, sel);
#else
    u32 d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
#endif
}

/* 16-entry x 8-bit table lookup for the four nibble indices packed one per
 * byte in idx (0..15), t[0..3] = entries 0-3, 4-7, 8-11, 12-15. */
__device__ __forceinline__ u32 nibbleLookup(const u32 t[4], u32 idx) {
    u32 x = idx & 0x07070707u;                            /* index within an 8-entry half */
    x |= x >> 4;                                          /* byte0 = i0|i1<<4, byte2 = i2|i3<<4 */
    const u32 sel = __byte_perm(x, 0, 0x4420);            /* selector nibbles i0,i1,i2,i3 */
    const u32 hiMask = prmt(idx << 4, 0, 0xba98);         /* 0xff where idx >= 8 (sign replicate) */
    const u32 lo8 = __byte_perm(t[0], t[1], sel);
    const u32 hi8 = __byte_perm(t[2], t[3], sel);
    return (lo8 & ~hiMask) | (hi8 & hiMask);
}

struct AccelParams {
    u32 type;
    u32 t0[4], t1[4]; /* shufti lo/hi, truffle mask1/mask2 */
    u32 c1x4, c2x4, casex4;
};

/* 0xff in each byte lane where a == b */
__device__ __forceinline__ u32 eq4(u32 a, u32 b) { return __vcmpeq4(a, b); }
/* 0xff in each byte lane that is non-zero */
__device__ __forceinline__ u32 nz4(u32 a) { return ~__vcmpeq4(a, 0); }

__global__ void __launch_bounds__(256) accelFindKernel(AccelParams p, const u8 *buf, u64 len,
                                                       unsigned long long *result) {
    const u64 chunks = (len + 15) / 16;
    for (u64 ch = (u64)blockIdx.x * blockDim.x + threadIdx.x;; ch += (u64)gridDim.x * blockDim.x) {
        /* whole warps leave together (ballot below): one lane reads the best
         * position found so far and broadcasts it, so that every lane of the
         * warp takes the same decision whatever the other warps publish meanwhile */
        const u64 warpFirst = ch - (threadIdx.x & 31);
        u64 best = 0;
        if ((threadIdx.x & 31) == 0) {
            best = *(volatile unsigned long long *)result;
        }
        best = __shfl_sync(0xffffffffu, best, 0);
        if (warpFirst >= chunks || warpFirst * 16 >= best) {
            return;
        }
        u32 w[5] = {0, 0, 0, 0, 0};
        if (ch < chunks) {
            const u64 base = ch * 16;
            if (base + 20 <= len) {
                const uint4 v = *reinterpret_cast<const uint4 *>(buf + base);
                w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
                w[4] = *reinterpret_cast<const u32 *>(buf + base + 16);
            } else {
                for (int i = 0; i < 20; i++) {
                    if (base + i < len) {
                        w[i >> 2] |= (u32)buf[base + i] << (8 * (i & 3));
                    }
                }
            }
        }
        u32 hit = 0; /* bit i = byte i of the 16 is a hit */
#pragma unroll
        for (int k = 0; k < 4; k++) {
            u32 m;
            if (p.type == ACCEL_SHUFTI) {
                const u32 lo = nibbleLookup(p.t0, w[k] & 0x0f0f0f0fu);
                const u32 hi = nibbleLookup(p.t1, (w[k] >> 4) & 0x0f0f0f0fu);
                m = nz4(lo & hi);
            } else if (p.type == ACCEL_TRUFFLE) {
                const u32 lo = w[k] & 0x0f0f0f0fu;
                const u32 a = nibbleLookup(p.t0, lo), b = nibbleLookup(p.t1, lo);
                const u32 top = prmt(w[k], 0, 0xba98); /* 0xff where byte >= 0x80 */
                const u32 sel = (a & ~top) | (b & top);
                /* bit (c >> 4) & 7 of each byte */
                const u32 sh = (w[k] >> 4) & 0x07070707u;
                u32 bits = 0;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    bits |= (1u << ((sh >> (8 * i)) & 7)) << (8 * i);
                }
                m = nz4(sel & bits);
            } else {
                m = eq4(w[k] & p.casex4, p.c1x4);
                if (p.type == ACCEL_DVERM || p.type == ACCEL_DVERM_NOCASE) {
                    const u32 nxt = __funnelshift_r(w[k], w[k + 1], 8);
                    m &= eq4(nxt & p.casex4, p.c2x4);
                }
            }
            /* one bit per byte lane */
            hit |= ((m & 0x00000080u) >> 7 | (m & 0x00008000u) >> 14 | (m & 0x00800000u) >> 21 |
                    (m & 0x80000000u) >> 28)
                   << (4 * k);
        }
        u64 pos = ~0ull;
        if (ch < chunks) {
            const u64 base = ch * 16;
            u32 valid = hit;
            const bool dbl = p.type == ACCEL_DVERM || p.type == ACCEL_DVERM_NOCASE;
            if (base + 16 > len) {
                valid &= (1u << (len - base)) - 1;
            }
            if (dbl && base + 16 >= len) {
                /* the pair must lie inside the buffer ... */
                const u32 last = (u32)(len - 1 - base);
                valid &= ~(1u << last);
                /* ... but a lone c1 in the last byte is a partial hit */
                const u32 lb = (w[last >> 2] >> (8 * (last & 3))) & 0xff;
                if ((lb & (p.casex4 & 0xff)) == (p.c1x4 & 0xff)) {
                    valid |= 1u << last;
                }
            }
            if (valid) {
                pos = base + (__ffs(valid) - 1);
            }
        }
        /* first hit of the warp -> one atomic */
        const u32 any = __ballot_sync(0xffffffffu, pos != ~0ull);
        if (any) {
            const int src = __ffs(any) - 1;
            const u64 first = __shfl_sync(0xffffffffu, pos, src);
            if ((threadIdx.x & 31) == 0) {
                atomicMin(result, (unsigned long long)first);
            }
            return; /* later chunks of this warp are further right */
        }
    }
}

} // namespace

cudaError_t launchAccelFind(int type, const u8 *params, const u8 *d_buf, u64 len, u64 *d_result,
                            cudaStream_t stream) {
    AccelParams p;
    memset(&p, 0, sizeof(p));
    p.type = (u32)type;
    p.casex4 = 0xffffffffu;
    switch (type) {
    case ACCEL_VERM_NOCASE:
    case ACCEL_DVERM_NOCASE:
        p.casex4 = 0xdfdfdfdfu;
        /* fallthrough */
    case ACCEL_VERM:
    case ACCEL_DVERM:
        p.c1x4 = (params[0] & (p.casex4 & 0xff)) * 0x01010101u;
        p.c2x4 = (params[1] & (p.casex4 & 0xff)) * 0x01010101u;
        break;
    case ACCEL_SHUFTI:
    case ACCEL_TRUFFLE:
        memcpy(p.t0, params, 16);
        memcpy(p.t1, params + 16, 16);
        break;
    default:
        return cudaErrorInvalidValue;
    }
    const unsigned long long init = len;
    cudaError_t e = cudaMemcpyAsync(d_result, &init, 8, cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) {
        return e;
    }
    if (len == 0) {
        return cudaSuccess;
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const u64 chunks = (len + 15) / 16;
    const u64 blocks = (chunks + 255) / 256;
    const int grid = (int)(blocks < (u64)sms * 8 ? blocks : (u64)sms * 8);
    HSB_LAUNCH(accelFindKernel, grid, 256, 0, stream, p, d_buf, len, (unsigned long long *)d_result);
    return cudaGetLastError();
}

} // namespace hsb
