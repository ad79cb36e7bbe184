/*
 * simt_emu.h -- TEST INFRASTRUCTURE (like oracle/): a single-threaded SIMT
 * emulator that lets the kernels of hyperscan_b200/csrc/device/*.cu run on a
 * CPU, compiled as plain C++ (-DHSB_HOST_EMU), so that the kernel LOGIC
 * (filter indexing, carries, queues, confirm, programs, block lookup) is covered
 * by `pytest -m "not gpu"` and new variants can be debugged without GPU time.
 *
 * It is NOT a scan path of the product: the emulated library is built by
 * tests/emu/build_emu.py into tests/emu/_build/, is loaded only by tests/, and
 * libhs_b200.so contains none of it.  It says nothing about performance and
 * does not model PTX-level behaviour (memory ordering, bank conflicts, TMA).
 *
 * Model: every CUDA thread of a block is a fiber (ucontext); fibers run one at
 * a time and switch only inside warp / block synchronising intrinsics
 * (__shfl*_sync, __ballot_sync, __any_sync, __syncwarp, __syncthreads), which
 * complete when all live lanes of the warp (threads of the block) have arrived.
 * Blocks of a grid run one after another.
 */
#ifndef HSB_SIMT_EMU_H
#define HSB_SIMT_EMU_H

#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <functional>

struct dim3 {
    unsigned x, y, z;
    dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { uint2 v = {x, y}; return v; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 v = {x, y, z, w}; return v; }

namespace hsb_emu {

struct ThreadCtx {
    dim3 tid, bid, bdim, gdim;
};
extern ThreadCtx *g_cur;              /* the running fiber */
uint8_t *dynamicSmem();               /* base of the block's dynamic shared memory */

enum Op { OP_SHFL_IDX, OP_SHFL_UP, OP_SHFL_DOWN, OP_BALLOT, OP_SYNCWARP };
uint32_t warpCollective(Op op, uint32_t value, uint32_t aux);
void blockBarrier();

/* run `body` once per thread of every block (threadIdx etc. set up) */
void launch(dim3 grid, dim3 block, size_t smemBytes, const std::function<void()> &body);

} // namespace hsb_emu

#define threadIdx (hsb_emu::g_cur->tid)
#define blockIdx (hsb_emu::g_cur->bid)
#define blockDim (hsb_emu::g_cur->bdim)
#define gridDim (hsb_emu::g_cur->gdim)

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
/* (__noinline__ is spelled HSB_NOINLINE in the sources: libstdc++ uses the bare word as an attribute) */
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

/* ---- warp / block intrinsics ---------------------------------------------- */
static inline uint32_t __shfl_sync(unsigned, uint32_t v, unsigned src) {
    return hsb_emu::warpCollective(hsb_emu::OP_SHFL_IDX, v, src);
}
static inline uint64_t __shfl_sync(unsigned m, uint64_t v, unsigned src) {
    const uint32_t lo = __shfl_sync(m, (uint32_t)v, src), hi = __shfl_sync(m, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}
static inline uint64_t __shfl_sync(unsigned m, unsigned long long v, unsigned src) {
    return __shfl_sync(m, (uint64_t)v, src);
}
static inline uint32_t __shfl_up_sync(unsigned, uint32_t v, unsigned d) {
    return hsb_emu::warpCollective(hsb_emu::OP_SHFL_UP, v, d);
}
static inline uint32_t __shfl_down_sync(unsigned, uint32_t v, unsigned d) {
    return hsb_emu::warpCollective(hsb_emu::OP_SHFL_DOWN, v, d);
}
static inline uint32_t __ballot_sync(unsigned, int pred) {
    return hsb_emu::warpCollective(hsb_emu::OP_BALLOT, pred ? 1u : 0u, 0);
}
static inline int __any_sync(unsigned, int pred) {
    return hsb_emu::warpCollective(hsb_emu::OP_BALLOT, pred ? 1u : 0u, 0) != 0;
}
static inline void __syncwarp(unsigned = 0xffffffffu) { hsb_emu::warpCollective(hsb_emu::OP_SYNCWARP, 0, 0); }
static inline void __syncthreads() { hsb_emu::blockBarrier(); }

/* ---- scalar intrinsics ------------------------------------------------------- */
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline int __ffs(uint32_t v) { return __builtin_ffs((int)v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t s) {
    const uint64_t v = ((uint64_t)hi << 32) | lo;
    return (uint32_t)((v << (s & 31)) >> 32);
}
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) {
    const uint64_t v = ((uint64_t)hi << 32) | lo;
    return (uint32_t)(v >> (s & 31));
}
static inline uint32_t __funnelshift_rc(uint32_t lo, uint32_t hi, uint32_t s) { /* shift clamped to 32 */
    const uint64_t v = ((uint64_t)hi << 32) | lo;
    return (uint32_t)(v >> (s > 32 ? 32 : s));
}
static inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
/* PRMT, default mode, selector nibble bit 3 = replicate the byte's sign */
static inline uint32_t hsb_emu_prmt(uint32_t a, uint32_t b, uint32_t sel) {
    const uint64_t ab = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t s = (sel >> (4 * i)) & 0xf;
        uint32_t byte = (uint32_t)(ab >> (8 * (s & 7))) & 0xff;
        if (s & 8) {
            byte = (byte & 0x80) ? 0xff : 0x00;
        }
        r |= byte << (8 * i);
    }
    return r;
}
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
    return hsb_emu_prmt(a, b, sel & 0x7777); /* the intrinsic honours selector bits 2:0 only */
}
static inline uint32_t __vcmpeq4(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        if (((a >> (8 * i)) & 0xff) == ((b >> (8 * i)) & 0xff)) {
            r |= 0xffu << (8 * i);
        }
    }
    return r;
}
template <class T> static inline T __ldg(const T *p) { return *p; }
using std::max;
using std::min;

template <class T> static inline T atomicAdd(T *p, T v) { const T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicExch(T *p, T v) { const T o = *p; *p = v; return o; }
template <class T> static inline T atomicMin(T *p, T v) { const T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicMax(T *p, T v) { const T o = *p; if (v > o) *p = v; return o; }

#endif
