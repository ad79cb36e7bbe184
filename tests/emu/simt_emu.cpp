/* simt_emu.cpp -- fiber scheduler of the SIMT emulator (see simt_emu.h; test infrastructure). */
#include "simt_emu.h"

#include <stdio.h>
#include <stdlib.h>
#include <ucontext.h>

#include <vector>

namespace hsb_emu {

namespace {

const size_t STACK_BYTES = 256 * 1024;

struct Fiber {
    ucontext_t ctx;
    ThreadCtx tc;
    char *stack = nullptr;
    bool done = false;
    unsigned warp = 0, lane = 0;
};

struct WarpState {
    uint32_t live = 0;     /* lanes that have not left the kernel */
    uint32_t arrived = 0;
    uint32_t gen = 0;
    Op op = OP_SYNCWARP;
    uint32_t val[32], aux[32], out[32];
};

struct BlockState {
    std::vector<Fiber> fibers;
    std::vector<WarpState> warps;
    uint8_t *smem = nullptr;
    unsigned liveThreads = 0, barArrived = 0, barGen = 0;
    const std::function<void()> *body = nullptr;
    unsigned progress = 0; /* bumped whenever any fiber gets past a wait */
};

BlockState *g_blk = nullptr;
Fiber *g_fiber = nullptr;
ucontext_t g_main;

void yield() { swapcontext(&g_fiber->ctx, &g_main); }

[[noreturn]] void die(const char *what) {
    fprintf(stderr, "simt_emu: %s\n", what);
    abort();
}

void leave(Fiber *f) {
    f->done = true;
    BlockState *b = g_blk;
    WarpState &w = b->warps[f->warp];
    w.live &= ~(1u << f->lane);
    b->liveThreads--;
    b->progress++;
    if (w.arrived && w.arrived == w.live) {
        die("a lane left the kernel while the rest of its warp waits in a warp-synchronous intrinsic");
    }
    if (b->barArrived && b->barArrived == b->liveThreads) {
        die("a thread left the kernel while the rest of its block waits in __syncthreads");
    }
}

void trampoline() {
    Fiber *f = g_fiber;
    (*g_blk->body)();
    leave(f);
    swapcontext(&f->ctx, &g_main);
}

} // namespace

ThreadCtx *g_cur = nullptr;

uint8_t *dynamicSmem() { return g_blk->smem; }

uint32_t warpCollective(Op op, uint32_t value, uint32_t aux) {
    Fiber *f = g_fiber;
    WarpState &w = g_blk->warps[f->warp];
    if (w.arrived && w.op != op) {
        die("lanes of one warp are in different warp-synchronous intrinsics (divergent collective)");
    }
    w.op = op;
    w.val[f->lane] = value;
    w.aux[f->lane] = aux;
    w.arrived |= 1u << f->lane;
    const uint32_t myGen = w.gen;
    if (w.arrived == w.live) {
        uint32_t ballot = 0;
        for (unsigned l = 0; l < 32; l++) {
            if (((w.live >> l) & 1) && w.val[l]) {
                ballot |= 1u << l;
            }
        }
        for (unsigned l = 0; l < 32; l++) {
            if (!((w.live >> l) & 1)) {
                continue;
            }
            switch (op) {
            case OP_SHFL_IDX: w.out[l] = w.val[w.aux[l] & 31]; break;
            case OP_SHFL_UP: w.out[l] = l >= w.aux[l] ? w.val[l - w.aux[l]] : w.val[l]; break;
            case OP_SHFL_DOWN: w.out[l] = l + w.aux[l] < 32 ? w.val[l + w.aux[l]] : w.val[l]; break;
            case OP_BALLOT: w.out[l] = ballot; break;
            case OP_SYNCWARP: w.out[l] = 0; break;
            }
        }
        w.arrived = 0;
        w.gen++;
        g_blk->progress++;
    } else {
        while (w.gen == myGen) {
            yield();
        }
    }
    return w.out[f->lane];
}

void blockBarrier() {
    BlockState *b = g_blk;
    const unsigned myGen = b->barGen;
    if (++b->barArrived == b->liveThreads) {
        b->barArrived = 0;
        b->barGen++;
        b->progress++;
    } else {
        while (b->barGen == myGen) {
            yield();
        }
    }
}

void launch(dim3 grid, dim3 block, size_t smemBytes, const std::function<void()> &body) {
    if (block.y != 1 || block.z != 1 || grid.y != 1 || grid.z != 1 || block.x == 0 || block.x > 1024) {
        die("only 1-D launches of up to 1024 threads are modelled");
    }
    if (g_blk) {
        die("nested launch");
    }
    static const bool trace = getenv("HSB_EMU_TRACE") != nullptr;
    if (trace) {
        fprintf(stderr, "simt_emu: launch grid %u block %u smem %zu\n", grid.x, block.x, smemBytes);
    }
    const unsigned nthreads = block.x, nwarps = (nthreads + 31) / 32;
    BlockState b;
    b.fibers.resize(nthreads);
    b.warps.resize(nwarps);
    b.body = &body;
    /* fiber stacks: one lazily mapped arena reused by every launch */
    static char *arena = nullptr;
    static size_t arenaBytes = 0;
    if ((size_t)nthreads * STACK_BYTES > arenaBytes) {
        free(arena);
        arenaBytes = (size_t)nthreads * STACK_BYTES;
        arena = (char *)malloc(arenaBytes);
        if (!arena) {
            die("out of memory for fiber stacks");
        }
    }
    /* poison-free but deterministic shared memory */
    /* sized to the launch's request (+ alignment slack) so that a sanitizer build sees
     * accesses past the end of the window */
    std::vector<uint8_t> smem(smemBytes + 128, 0xcd);
    uint8_t *base = smem.data();
    base += (128 - ((uintptr_t)base & 127)) & 127;
    b.smem = base;
    g_blk = &b;
    for (unsigned bx = 0; bx < grid.x; bx++) {
        memset(smem.data(), 0xcd, smem.size());
        b.liveThreads = nthreads;
        b.barArrived = 0;
        for (unsigned w = 0; w < nwarps; w++) {
            const unsigned lanes = std::min(32u, nthreads - w * 32);
            b.warps[w].live = lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1);
            b.warps[w].arrived = 0;
        }
        for (unsigned t = 0; t < nthreads; t++) {
            Fiber &f = b.fibers[t];
            f.done = false;
            f.warp = t / 32;
            f.lane = t % 32;
            f.tc.tid = dim3(t);
            f.tc.bid = dim3(bx);
            f.tc.bdim = block;
            f.tc.gdim = grid;
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = arena + (size_t)t * STACK_BYTES;
            f.ctx.uc_stack.ss_size = STACK_BYTES;
            f.ctx.uc_link = &g_main;
            makecontext(&f.ctx, trampoline, 0);
        }
        for (;;) {
            const unsigned before = b.progress;
            bool allDone = true;
            for (unsigned t = 0; t < nthreads; t++) {
                Fiber &f = b.fibers[t];
                if (f.done) {
                    continue;
                }
                allDone = false;
                g_fiber = &f;
                g_cur = &f.tc;
                swapcontext(&g_main, &f.ctx);
            }
            if (allDone) {
                break;
            }
            if (b.progress == before) {
                die("deadlock: no thread of the block can make progress");
            }
        }
    }
    g_blk = nullptr;
    g_fiber = nullptr;
    g_cur = nullptr;
}

} // namespace hsb_emu
