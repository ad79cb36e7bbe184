/*
 * api_device.cu -- device half of the C ABI: scratch, corpus handles and the
 * scan entry points (include/hs_b200.h).  The thin host shim around the
 * sm_90a kernels in scan_kernels.cu:
 *
 *   hs_alloc_scratch / hs_clone_scratch / hs_scratch_size / hs_free_scratch
 *        src/scratch.c:244-460 -- here a scratch owns a CUDA stream, the
 *        match-record ring in HBM and the device images of the databases it
 *        was allocated for.
 *   hs_scan   src/runtime.c:316-475 -- argument checks and early-outs follow
 *        the reference; the body is "copy block to HBM, launch, read records
 *        back, replay callbacks in offset order".
 *   hs_b200_* the batched / device-resident forms of the same (hsbench scans
 *        a set of blocks: tools/hsbench/main.cpp:503-527).
 *
 * There is no CPU scan path in this library: without a usable CUDA device
 * hs_alloc_scratch fails with HS_ARCH_ERROR.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <new>
#include <unordered_set>
#include <vector>

#include "../host/api_internal.h"
#include "../host/db_walk.h"
#include "../host/pair_table.h"
#include "kernels.h"
#include "order_kernels.h"
#include "rows_kernels.h"
#include "stream_rows_kernels.h"

using namespace hsb;

namespace {

const u32 SCRATCH_MAGIC = 0x544F4259; /* src/scratch.h:48 */
const size_t FRONT_PAD = 256;         /* readable bytes before corpus position 0 */

std::atomic<unsigned long long> g_launches{0};

/* runtime tunables (hs_b200_set_runtime_option / HSB200_* environment): the scan
 * geometry, and two switches that force either side of a choice the library
 * otherwise makes from the database */
struct RuntimeOpts {
    int warps = 0;           /* per CTA; 0 = 28 (896 threads x 72 registers) */
    int tileBytes = 1024;
    int pfDist = -1;         /* L2 prefetch distance (kernels.h ScanParams.pfDist); -1 = per kernel: 2 steps
                              * (1 KiB) for the pair kernel, 4 for the others.  On an H100 SXM (700 W) 4 against 8
                              * took 17 % off the Teddy-48 and noodle kernels and left 5 000 / 50 000 literals
                              * unchanged (1 GiB, tools/sweep.py); the pair kernel at 2 steps against 4 took 2-6 %
                              * off 96 (fat Teddy), 200 and 1 000 literals (DESIGN.md section 3.3); on a card
                              * limited to 400 W, whose clock is power-bound, 4 and 8 are level */
    int gram = 1;            /* FDR sets: 1 = class 4-gram first stage (FK_GRAM4) for sets that would fill the
                              * pair kernel's 32 KiB bitmap beyond 10 % (all literals >= 4 bytes), 2 = whenever
                              * possible, 0 = never */
    int heavy = 1;           /* FK_PAIR32 candidate path: 1 (and 2) = per-word entries, 0 = per-lane entries */
    int dfaIlp = 1;          /* DFA kernels: blocks walked by one lane at a time; 2 = two interleaved state chains
                              * per lane (half the warps for the same block count) */
    int engineSegment = 0;   /* engine runs: 0 = cut long blocks into segments when the blocks leave most resident
                              * lanes idle (planSegments), N > 0 = cut every block longer than N into N-byte
                              * segments, -1 = never cut */
    int chunkMB = 128;       /* host->device pipeline granularity */
    int initialRing = 1 << 20;
};
RuntimeOpts g_opts;
bool g_optsInit = false;

void initOpts() {
    if (g_optsInit) {
        return;
    }
    g_optsInit = true;
    struct { const char *env; int *v; } e[] = {
        {"HSB200_WARPS", &g_opts.warps},       {"HSB200_TILE", &g_opts.tileBytes},
        {"HSB200_CHUNK_MB", &g_opts.chunkMB},  {"HSB200_RING", &g_opts.initialRing},
        {"HSB200_PF_DIST", &g_opts.pfDist},    {"HSB200_HEAVY", &g_opts.heavy},
        {"HSB200_GRAM", &g_opts.gram},         {"HSB200_DFA_ILP", &g_opts.dfaIlp},
        {"HSB200_ENGINE_SEGMENT", &g_opts.engineSegment}};
    for (auto &x : e) {
        const char *s = getenv(x.env);
        if (s && *s) {
            *x.v = atoi(s);
        }
    }
}

/* Memory of the segmented engine runs (launchEngine): in device memory the plan, the first open segment of each
 * block and the per-segment states, grown on demand; the plan's host image in pinned memory, so that its copy
 * does not wait for the stream; and what the runs did, for hs_b200_engine_segment_stats. */
struct SegArea {
    u8 *d = nullptr;
    size_t bytes = 0;
    u8 *h = nullptr;                       /* pinned: the plan being copied */
    size_t hBytes = 0;
    cudaEvent_t copied = nullptr;          /* recorded after the last copy out of h */
    std::vector<u8> plan;                  /* the plan now in d (empty: none) */
    unsigned long long *d_stats = nullptr; /* SEGSTAT_COUNT counters */
    unsigned long long runs = 0, segments = 0;
    SegArea() = default;
    SegArea(const SegArea &) = delete;
    SegArea &operator=(const SegArea &) = delete;
    ~SegArea() {
        if (copied) {
            cudaEventSynchronize(copied);
            cudaEventDestroy(copied);
        }
        cudaFreeHost(h);
        cudaFree(d);
        cudaFree(d_stats);
    }
};

/* ---- device image of one database --------------------------------------- */

struct DevImage {
    const hs_database_t *db = nullptr;   /* identity of the database the image was built from (a key: never
                                          * dereferenced -- the application may have freed it) */
    std::vector<u8> dbCopy;
    u32 dbCopyShift = 0;              /* its bytes (header + bytecode, bytecode offset preserved), so that
                                          * hs_clone_scratch can rebuild the image without the original */
    u32 crc = 0, length = 0;
    u8 *d_bc = nullptr;
    u8 *d_table = nullptr;
    u32 tableBytes = 0;
    u8 *d_bitmap = nullptr;
    u32 bitmapBytes = 0, bitmapShift = 0, keyBytes = 0;
    u32 pairBytes = 0, bitmapBits = 0; /* FK_PAIR32 layout (kernels.h) */
    u32 bucketFold = 0;
    /* the outfix engines (bytecode offset, NFA.length) in queue order: one alone (FK_OUTFIX) or beside the
     * literal matcher, or several alone (FK_OUTFIX); empty: none */
    std::vector<std::pair<u32, u32>> engines;
    /* what launchDfa needs to run them over a corpus: the one engine's parameters, or for several engines
     * one fused launch per engine kind over the descriptors at d_engines */
    std::vector<DfaParams> engineRuns;
    DfaEngine *d_engines = nullptr;
    u8 *d_bitmap2 = nullptr; /* second level (HBM / L2) for large literal sets */
    u32 bitmap2Shift = 0;
    int kind = FK_BYTE32;
    int slotBase = 0;
    u32 confOff = 0, engineOff = 0;
    u32 confirmKind = CK_FDR;
    u64 groups = 0;
    u32 minWidth = 0;
    ReportRules rules;                   /* how its records are delivered (borrows dbCopy) */
    /* the same rules as device tables, for hs_b200_order_*_async (order_kernels.h): OrderParams'
     * table fields; orderStatus != HS_SUCCESS when an engine program cannot be laid out */
    hs_error_t orderStatus = HS_SUCCESS;
    u8 *d_rules = nullptr;
    OrderParams orderTables;
    u32 maxFanout = 1;
    s32 maxAdjust = 0;
    size_t deviceBytes = 0;
};

/* A scratch (and a corpus / stream set) is bound to the CUDA device that was current
 * when it was created: its streams, events, record ring and database images live
 * there.  The reference lets any thread use any scratch, and a fresh thread's current
 * device is 0, so every entry point that touches one switches to its device for the
 * duration of the call and restores the caller's. */
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) {
            switched = cudaSetDevice(dev) == cudaSuccess;
        }
    }
    ~DeviceGuard() {
        if (switched) {
            cudaSetDevice(prev);
        }
    }
    DeviceGuard(const DeviceGuard &) = delete;
    DeviceGuard &operator=(const DeviceGuard &) = delete;
};

#define CUDA_TRY(expr)                                                                     \
    do {                                                                                   \
        cudaError_t e__ = (expr);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            return e__ == cudaErrorMemoryAllocation ? HS_NOMEM : HS_UNKNOWN_ERROR;         \
        }                                                                                  \
    } while (0)

/* Keys of the prefilter bitmaps: every literal's last m <= 4 bytes with the
 * don't-care bits of LitInfo.msk enumerated.  false = cannot be keyed usefully. */
bool tailKeys(const std::vector<LitTail> &tails, u32 *keyBytes, std::vector<u32> *keys) {
    if (tails.empty()) {
        return false;
    }
    u32 m = 4;
    for (const LitTail &t : tails) {
        m = std::min(m, t.size);
    }
    if (m < 2) {
        return false; /* single-byte literals: the first stage is already exact */
    }
    for (const LitTail &t : tails) {
        const u32 v = (u32)(t.v >> 32) >> (8 * (4 - m));
        const u32 care = (u32)(t.msk >> 32) >> (8 * (4 - m));
        const u32 full = m == 4 ? 0xffffffffu : (1u << (8 * m)) - 1;
        const u32 dc = ~care & full;
        if (__builtin_popcount(dc) > 10) {
            return false; /* too loose to enumerate */
        }
        u32 sub = 0;
        do {
            keys->push_back((v & care) | sub);
            sub = (sub - dc) & dc;
        } while (sub);
    }
    *keyBytes = m;
    return true;
}

/* Second level of the prefilter bitmaps, in HBM / L2 and probed only by the first
 * level's survivors: ~1024 bits per key, at least 2^lg bits, <= 64 MB.  Returns
 * its shift (32 - log2(bits)). */
u32 buildLevel2(const std::vector<u32> &keys, u32 lg, std::vector<u8> *level2) {
    while (lg < 29 && (1ull << lg) < (u64)keys.size() * 1024) {
        lg++;
    }
    level2->assign((size_t)1 << (lg - 3), 0);
    for (u32 k : keys) {
        const u32 h = (k * 0x85EBCA6Bu) >> (32 - lg);
        (*level2)[h >> 3] |= (u8)(1u << (h & 7));
    }
    return 32 - lg;
}

/* Second-stage prefilter of the wide kernel: a bitmap over a hash of each literal's
 * last keyBytes bytes (tailKeys).  A clear bit proves no literal ends at a candidate
 * position, so the hash confirm in HBM/L2 is only reached by ~1% of the first stage's
 * false positives.  Returns an empty vector when the set cannot be keyed usefully. */
std::vector<u8> buildBitmap(const std::vector<LitTail> &tails, u32 *keyBytes, u32 *shift,
                            std::vector<u8> *level2, u32 *shift2) {
    std::vector<u32> keys;
    u32 m = 0;
    if (!tailKeys(tails, &m, &keys)) {
        return std::vector<u8>();
    }
    u32 lg = 13; /* 8 Kbit .. 512 Kbit (64 KB), ~256 bits per key when possible */
    while (lg < 19 && (1ull << lg) < (u64)keys.size() * 256) {
        lg++;
    }
    std::vector<u8> bm((size_t)1 << (lg - 3), 0);
    for (u32 k : keys) {
        const u32 h = (k * 0x9E3779B1u) >> (32 - lg);
        bm[h >> 3] |= (u8)(1u << (h & 7));
    }
    *keyBytes = m;
    *shift = 32 - lg;
    if (keys.size() * 32 > ((size_t)1 << lg)) {
        *shift2 = buildLevel2(keys, lg + 1, level2); /* the first level is more than ~3 % full */
    }
    return bm;
}

/* FK_PAIR32 bitmaps: first level of `bits` bits (index = mulhi(key * K, bits)) in
 * shared memory, second level in HBM / L2 when the first is more than ~3 % full. */
void buildPairBitmaps(const std::vector<u32> &keys, u32 bits, std::vector<u8> *level1,
                      std::vector<u8> *level2, u32 *shift2) {
    level1->assign((size_t)(bits + 31) / 32 * 4, 0);
    for (u32 k : keys) {
        const u32 h = (u32)(((u64)(k * 0x9E3779B1u) * bits) >> 32);
        (*level1)[h >> 3] |= (u8)(1u << (h & 7));
    }
    *shift2 = keys.size() * 32 > bits ? buildLevel2(keys, 20, level2) : 0;
}

/* FK_GRAM4 tables: a byte -> class map (<= 32 classes) and the 1 Mbit bitmap of the class
 * 4-grams that some literal's last four bytes can produce (caseless letters through
 * LitInfo.msk).  Bytes no tail uses share class 0; if more than 31 byte values are in
 * use, the two cases of a letter share a class first (a case-sensitive literal then also
 * admits the other case at the first stage -- the exact 4-byte bitmap in L2 and the
 * confirm sort that out), then the rarest byte values are folded together. */
bool buildGramTables(const std::vector<LitTail> &tails, std::vector<u8> *classWords, std::vector<u8> *bitmap) {
    u32 count[256] = {0};
    for (const LitTail &t : tails) {
        if (t.size < 4) {
            return false; /* needs four known bytes per literal */
        }
        for (u32 p = 0; p < 4; p++) {
            const u8 c = (u8)(t.v >> (8 * (7 - p))), m = (u8)(t.msk >> (8 * (7 - p)));
            for (u32 b = 0; b < 256; b++) {
                if ((b & m) == c) {
                    count[b]++;
                }
            }
        }
    }
    u32 cls[256];
    std::vector<std::vector<u32>> groups; /* groups[i] = byte values of class i + 1 */
    for (u32 b = 0; b < 256; b++) {
        if (count[b]) {
            groups.push_back({b});
        }
    }
    auto weight = [&](const std::vector<u32> &g) {
        u64 w = 0;
        for (u32 b : g) {
            w += count[b];
        }
        return w;
    };
    if (groups.size() > 31) { /* fold the cases of letters */
        std::vector<std::vector<u32>> folded;
        std::vector<bool> done(256, false);
        for (const auto &g : groups) {
            const u32 b = g[0];
            if (done[b]) {
                continue;
            }
            done[b] = true;
            std::vector<u32> ng = {b};
            const bool alpha = (b >= 'a' && b <= 'z') || (b >= 'A' && b <= 'Z');
            if (alpha && count[b ^ 0x20]) {
                ng.push_back(b ^ 0x20);
                done[b ^ 0x20] = true;
            }
            folded.push_back(ng);
        }
        groups.swap(folded);
    }
    while (groups.size() > 31) { /* fold the two rarest groups */
        size_t a = 0, b = 1;
        if (weight(groups[b]) < weight(groups[a])) {
            std::swap(a, b);
        }
        for (size_t i = 2; i < groups.size(); i++) {
            if (weight(groups[i]) < weight(groups[a])) {
                b = a;
                a = i;
            } else if (weight(groups[i]) < weight(groups[b])) {
                b = i;
            }
        }
        groups[std::min(a, b)].insert(groups[std::min(a, b)].end(), groups[std::max(a, b)].begin(),
                                      groups[std::max(a, b)].end());
        groups.erase(groups.begin() + (long)std::max(a, b));
    }
    for (u32 b = 0; b < 256; b++) {
        cls[b] = 0;
    }
    for (size_t i = 0; i < groups.size(); i++) {
        for (u32 b : groups[i]) {
            cls[b] = (u32)i + 1;
        }
    }
    classWords->resize(256 * 4);
    for (u32 b = 0; b < 256; b++) {
        const u32 e = cls[b] * 4;
        memcpy(classWords->data() + 4 * b, &e, 4);
    }
    /* word index c[e-3] + 33 c[e-2] + 1025 c[e-1] (kernels.h FK_GRAM4): sized like the kernel's window */
    bitmap->assign((size_t)scanSmemBytes(FK_GRAM4, 0, 0, 0) - 65536, 0);
    for (const LitTail &t : tails) {
        /* classes each of the last four bytes can take: [0] = byte e-3 ... [3] = byte e */
        u32 opts[4] = {0, 0, 0, 0}; /* bitmask over classes */
        for (u32 p = 0; p < 4; p++) {
            const u8 c = (u8)(t.v >> (8 * (7 - p))), m = (u8)(t.msk >> (8 * (7 - p)));
            for (u32 b = 0; b < 256; b++) {
                if ((b & m) == c) {
                    opts[3 - p] |= 1u << cls[b];
                }
            }
        }
        for (u32 c3 = 0; c3 < 32; c3++) {
            if (!((opts[0] >> c3) & 1)) continue;
            for (u32 c2 = 0; c2 < 32; c2++) {
                if (!((opts[1] >> c2) & 1)) continue;
                for (u32 c1 = 0; c1 < 32; c1++) {
                    if (!((opts[2] >> c1) & 1)) continue;
                    const u32 word = c3 + 33 * c2 + 1025 * c1;
                    u32 w;
                    memcpy(&w, bitmap->data() + 4 * (size_t)word, 4);
                    w |= opts[3];
                    memcpy(bitmap->data() + 4 * (size_t)word, &w, 4);
                }
            }
        }
    }
    return true;
}

/* What launchDfa needs to know about a serialized engine (struct NFA + McClellan 8 / 16,
 * Sheng or LimEx-32 ... -512), checked against its length.  HS_ARCH_ERROR: an engine or a feature
 * (wide states, bounded repeats) the DFA / NFA kernels do not implement. */
hs_error_t engineParams(const void *nfa, size_t nfa_len, DfaParams *out) {
    if (!nfa || nfa_len < sizeof(NFA) + 64) {
        return HS_INVALID;
    }
    NFA hdr;
    memcpy(&hdr, nfa, sizeof(hdr));
    if (hdr.length > nfa_len) {
        return HS_INVALID;
    }
    DfaParams &p = *out;
    memset(&p, 0, sizeof(p));
    p.kind = hdr.type;
    p.ilp = g_opts.dfaIlp == 2 ? 2u : 1u;
    if (hdr.type == NFA_MCCLELLAN_8 || hdr.type == NFA_MCCLELLAN_16) {
        if (nfa_len < sizeof(NFA) + sizeof(McClellan)) {
            return HS_INVALID;
        }
        McClellan m;
        memcpy(&m, (const u8 *)nfa + sizeof(NFA), sizeof(m));
        if (m.has_wide) {
            return HS_ARCH_ERROR; /* wide states (mcclellan.c:168-225) are not built here */
        }
        const u32 rows = hdr.type == NFA_MCCLELLAN_16 ? m.sherman_limit : m.state_count;
        p.tableBytes = (rows << m.alphaShift) * (hdr.type == NFA_MCCLELLAN_16 ? 2u : 1u);
        p.states = m.state_count;
        if (hdr.type == NFA_MCCLELLAN_8 && (m.state_count == 0 || m.state_count > 256)) {
            return HS_INVALID;
        }
        if (sizeof(NFA) + sizeof(McClellan) + p.tableBytes > nfa_len) {
            return HS_INVALID;
        }
    } else if (hdr.type == NFA_SHENG) {
        if (nfa_len < sizeof(NFA) + sizeof(Sheng)) {
            return HS_INVALID;
        }
    } else if (hdr.type == NFA_LIMEX_32 || hdr.type == NFA_LIMEX_64 || hdr.type == NFA_LIMEX_128 ||
               hdr.type == NFA_LIMEX_256 || hdr.type == NFA_LIMEX_512) {
        /* (the 384-state model is not built: the emitter here never produces it) */
        size_t structSize, excSize, stateBytes, shiftCountAt;
        switch (hdr.type) {
#define HSB_LIMEX_MODEL(T, L, E, B)                                                     \
        case T:                                                                         \
            structSize = sizeof(L), excSize = sizeof(E), stateBytes = B, shiftCountAt = offsetof(L, shiftCount); \
            break;
            HSB_LIMEX_MODEL(NFA_LIMEX_32, LimExNFA32, NFAException32, 4)
            HSB_LIMEX_MODEL(NFA_LIMEX_64, LimExNFA64, NFAException64, 8)
            HSB_LIMEX_MODEL(NFA_LIMEX_128, LimExNFA128, NFAException128, 16)
            HSB_LIMEX_MODEL(NFA_LIMEX_256, LimExNFA256, NFAException256, 32)
        default:
            HSB_LIMEX_MODEL(NFA_LIMEX_512, LimExNFA512, NFAException512, 64)
#undef HSB_LIMEX_MODEL
        }
        if (nfa_len < sizeof(NFA) + structSize) {
            return HS_INVALID;
        }
        /* the count / offset fields precede the state-sized ones and sit at the same offsets in every model */
        LimExNFA32 lx;
        memcpy(&lx, (const u8 *)nfa + sizeof(NFA), offsetof(LimExNFA32, init));
        u32 shiftCount;
        memcpy(&shiftCount, (const u8 *)nfa + sizeof(NFA) + shiftCountAt, 4);
        if (lx.repeatCount) {
            return HS_ARCH_ERROR; /* bounded repeats (repeat control blocks, tug / pos triggers) are not built */
        }
        if (stateBytes > 8 && ((uintptr_t)nfa & 7)) {
            return HS_INVALID; /* the wide state sets are read as 64-bit words */
        }
        const size_t body = nfa_len - sizeof(NFA);
        if (shiftCount > 8 || lx.exceptionCount > 8 * stateBytes ||
            structSize + stateBytes * lx.reachSize > body ||
            (size_t)lx.exceptionOffset + (size_t)lx.exceptionCount * excSize > body ||
            (size_t)lx.acceptOffset + (size_t)lx.acceptCount * sizeof(NFAAccept) > body ||
            (size_t)lx.acceptEodOffset + (size_t)lx.acceptEodCount * sizeof(NFAAccept) > body) {
            return HS_INVALID;
        }
        p.states = hdr.nPositions;
        for (u32 i = 0; i < lx.exceptionCount; i++) {
            /* hasSquash sits right after the two state-sized masks and the two u32 of every model's exception */
            const u8 kind = *((const u8 *)nfa + sizeof(NFA) + lx.exceptionOffset + i * excSize + 2 * stateBytes + 8);
            p.squashes |= kind == LIMEX_SQUASH_CYCLIC || kind == LIMEX_SQUASH_REPORT;
        }
    } else {
        return HS_ARCH_ERROR; /* LimEx-384, McSheng, Gough, Castle, ...: not built */
    }
    return HS_SUCCESS;
}

void freeImage(DevImage *im) {
    if (!im) {
        return;
    }
    cudaFree(im->d_bc);
    cudaFree(im->d_table);
    cudaFree(im->d_bitmap);
    cudaFree(im->d_bitmap2);
    cudaFree(im->d_rules);
    cudaFree(im->d_engines);
    delete im;
}

/* The report rules of an image as device tables (DeviceRules, one allocation): program reports, program
 * offsets and starts, report ids and their exhaustible marks.  An engine program the tables cannot hold
 * leaves orderStatus set; only the device ordering refuses the database then. */
hs_error_t uploadOrderTables(DevImage *im) {
    DeviceRules dr;
    std::vector<EngineBytes> engines;
    for (const auto &e : im->engines) {
        engines.push_back({im->rules.bc + e.first, e.second});
    }
    im->orderStatus = buildDeviceRules(&im->rules, engines, &dr);
    if (im->orderStatus != HS_SUCCESS) {
        return HS_SUCCESS;
    }
    std::vector<OrderRep> reps(dr.reps.size());
    for (size_t i = 0; i < reps.size(); i++) {
        const ProgReport &r = dr.reps[i];
        reps[i] = {r.onmatch, r.offset_adjust, r.min_bound, r.max_bound, r.logical ? 1u : 0u, 0};
    }
    const size_t repBytes = reps.size() * sizeof(OrderRep), offBytes = dr.progOff.size() * 4,
                 startBytes = dr.progStart.size() * 4, idBytes = dr.ids.size() * 4, exBytes = dr.ids.size();
    const size_t total = repBytes + offBytes + startBytes + idBytes + exBytes;
    std::vector<u8> img(total + 1);
    size_t at = 0;
    auto put = [&](const void *src, size_t n) {
        if (n) {
            memcpy(img.data() + at, src, n);
        }
        at += n;
        return at - n;
    };
    const size_t oRep = put(reps.data(), repBytes), oOff = put(dr.progOff.data(), offBytes),
                 oStart = put(dr.progStart.data(), startBytes), oIds = put(dr.ids.data(), idBytes),
                 oEx = put(dr.idExhaustible.data(), exBytes);
    CUDA_TRY(cudaMalloc(&im->d_rules, img.size()));
    CUDA_TRY(cudaMemcpy(im->d_rules, img.data(), img.size(), cudaMemcpyHostToDevice));
    im->deviceBytes += img.size();
    OrderParams &t = im->orderTables;
    memset(&t, 0, sizeof(t));
    t.shape = (u32)im->rules.shape;
    t.reps = (const OrderRep *)(im->d_rules + oRep);
    t.progOff = (const u32 *)(im->d_rules + oOff);
    t.progStart = (const u32 *)(im->d_rules + oStart);
    t.nProg = (u32)dr.progOff.size();
    t.ids = (const u32 *)(im->d_rules + oIds);
    t.idEx = im->d_rules + oEx;
    t.nIds = (u32)dr.ids.size();
    t.anyEx = std::find(dr.idExhaustible.begin(), dr.idExhaustible.end(), 1) != dr.idExhaustible.end();
    im->maxFanout = std::max<u32>(1, dr.maxFanout);
    im->maxAdjust = dr.maxAdjust;
    return HS_SUCCESS;
}

/* Several engines: one launch per engine kind present instead of one per engine (DfaParams.engines), so
 * that a corpus too small to fill the GPU for one engine runs all of them side by side.  Replaces
 * im->engineRuns (one per engine, nfa set) with one run per kind, in the order the kinds first appear in
 * the queues, over descriptors uploaded to im->d_engines. */
hs_error_t fuseEngineRuns(DevImage *im) {
    std::vector<DfaEngine> descs;
    std::vector<DfaParams> runs;
    std::vector<size_t> firstDesc;
    std::vector<bool> done(im->engineRuns.size(), false);
    for (size_t q = 0; q < im->engineRuns.size(); q++) {
        if (done[q]) {
            continue;
        }
        DfaParams run = im->engineRuns[q];
        run.nfa = nullptr;
        run.tableBytes = run.states = run.squashes = 0;
        run.nengines = 0;
        firstDesc.push_back(descs.size());
        for (size_t j = q; j < im->engineRuns.size(); j++) {
            const DfaParams &e = im->engineRuns[j];
            if (e.kind != run.kind) {
                continue;
            }
            done[j] = true;
            descs.push_back({e.nfa, e.tableBytes, e.states, e.squashes, 0});
            run.tableBytes = std::max(run.tableBytes, e.tableBytes);
            run.states = std::max(run.states, e.states);
            run.nengines++;
        }
        runs.push_back(run);
    }
    CUDA_TRY(cudaMalloc(&im->d_engines, descs.size() * sizeof(DfaEngine)));
    CUDA_TRY(cudaMemcpy(im->d_engines, descs.data(), descs.size() * sizeof(DfaEngine), cudaMemcpyHostToDevice));
    im->deviceBytes += descs.size() * sizeof(DfaEngine);
    for (size_t i = 0; i < runs.size(); i++) {
        runs[i].engines = im->d_engines + firstDesc[i];
    }
    im->engineRuns.swap(runs);
    return HS_SUCCESS;
}

/* Derive the device image: a copy of the bytecode plus the first-stage table
 * in the form the shift-OR kernel consumes (DESIGN.md section 3). */
hs_error_t buildImage(const hs_database_t *db, DevImage **out) {
    initOpts();
    const DbHeader *h = (const DbHeader *)db;
    const RoseEngine *r = dbRose(db);
    const u8 *bc = (const u8 *)r;
    const DbShape shape = dbShape(db);
    if (shape == SHAPE_UNSUPPORTED || shape == SHAPE_MALFORMED) {
        return shape == SHAPE_MALFORMED ? HS_INVALID : HS_ARCH_ERROR;
    }
    std::unique_ptr<DevImage, void (*)(DevImage *)> im(new (std::nothrow) DevImage(), freeImage);
    if (!im) {
        return HS_NOMEM;
    }
    im->db = db;
    {
        /* same address modulo 64 as the original, so that every offset-derived alignment holds */
        const size_t total = sizeof(DbHeader) + h->length;
        im->dbCopy.resize(total + 128);
        const size_t want = (uintptr_t)db & 63, have = (uintptr_t)im->dbCopy.data() & 63;
        im->dbCopyShift = (u32)((want + 64 - have) & 63);
        memcpy(im->dbCopy.data() + im->dbCopyShift, db, std::min(total, (size_t)h->bytecode + h->length));
    }
    im->crc = h->crc32;
    im->length = h->length;
    im->groups = r->initialGroups & r->floating_group_mask;
    im->minWidth = r->minWidth;
    if (shape != SHAPE_PURE_LITERAL) {
        /* hs_scan -> soleOutfixBlockExec (src/runtime.c:245-280): ONE engine over the whole block,
         * its reports are report programs (roseReportAdaptor, src/rose/match.c:611-633).  The
         * engine runs on the DFA / NFA kernels (dfa_kernels.cu) straight from the bytecode copy;
         * the programs are resolved on the host when the records are delivered (ReportRules).  With
         * a literal matcher beside it (roseBlockExec's outfix), the engine's records are tagged so
         * that the host can tell them from the literals'.  Several outfixes without a literal matcher
         * (roseBlockExec over several outfix queues) all run over every block, into one record ring */
        std::vector<EngineBytes> engines;
        if (!outfixEngines(db, &engines)) {
            return HS_INVALID;
        }
        for (const EngineBytes &e : engines) {
            DfaParams dp;
            const hs_error_t er = engineParams(e.nfa, e.len, &dp);
            if (er != HS_SUCCESS) {
                return er;
            }
            dp.toTag = shape == SHAPE_LITERALS_OUTFIX ? ENGINE_RECORD : 0;
            im->engines.push_back({(u32)(e.nfa - bc), e.len});
            im->engineRuns.push_back(dp);
        }
    }
    /* a literal program that uses a state-carrying opcode of roseRunProgram_l that the device
     * interpreter does not implement (delayed literals, SOM, chained reports) is refused here
     * rather than mid-scan */
    std::vector<LitTail> tails;
    const hs_error_t er = loadReportRules((const hs_database_t *)(im->dbCopy.data() + im->dbCopyShift), &im->rules,
                                          &tails);
    if (er != HS_SUCCESS) {
        return er;
    }
    const HWLM *hw = (const HWLM *)(bc + r->fmatcherOffset);
    const u32 engOff = r->fmatcherOffset + HWLM_ENGINE_OFFSET;
    std::vector<u8> table, bitmap, bitmap2;
    /* FK_PAIR32 / FK_GRAM4 tables from the literals' tails (FDR sets, and fat Teddy with its 16
     * buckets folded onto 8 first-stage bits) */
    auto pairStage = [&](bool allowGram) {
        u32 minSize = 8;
        for (const LitTail &t : tails) {
            minSize = std::min(minSize, t.size);
        }
        im->kind = FK_PAIR32;
        im->slotBase = minSize >= 2 ? 1 : 0;
        /* shared memory: 64 KiB class rows (the 32 KiB prefilter bitmap in their upper
         * halves) + 32 x 32 classes (128 KiB pair table) + queues */
        std::vector<u32> keys;
        u32 kb = 0;
        const bool keyed = tailKeys(tails, &kb, &keys);
        std::vector<u8> gramBitmap;
        /* measured crossover (DESIGN.md section 3.7): 5 000 literals (12.5 k keys) scan
         * 10 % faster through the 4-gram kernel, 1 000 literals 38 % slower */
        const bool gramWorth = keys.size() >= 10000;
        if (allowGram && (g_opts.gram == 2 || (g_opts.gram == 1 && gramWorth)) && keyed && kb == 4 &&
            buildGramTables(tails, &table, &gramBitmap)) {
            /* the pair evidence saturates for such sets: exact class 4-gram membership
             * instead (FK_GRAM4), exact raw 4-byte keys in L2 behind it */
            im->kind = FK_GRAM4;
            im->keyBytes = 4;
            bitmap.swap(gramBitmap);
            /* second level in L2: one BYTE per slot = the buckets of the literals whose
             * raw 4-byte key hashes there (~64 slots per key, <= 64 MB), so that a
             * survivor reaches confirm with its real buckets, not all eight */
            u32 lg2 = 16;
            while (lg2 < 26 && (1ull << lg2) < (u64)keys.size() * 64) {
                lg2++;
            }
            bitmap2.assign((size_t)1 << lg2, 0);
            for (const LitTail &t : tails) {
                const u32 v = (u32)(t.v >> 32), care = (u32)(t.msk >> 32), dc = ~care;
                u32 sub = 0;
                do {
                    const u32 k = (v & care) | sub;
                    bitmap2[(k * 0x85EBCA6Bu) >> (32 - lg2)] |= (u8)(1u << (t.bucket & 7));
                    sub = (sub - dc) & dc;
                } while (sub);
            }
            im->bitmap2Shift = 32 - lg2;
            return;
        }
        PairTables pt;
        buildPairTables(tails, (u32)im->slotBase, &pt, 32, 32);
        im->pairBytes = pt.nClass1 * 4096;
        if (getenv("HSB200_TRACE")) {
            fprintf(stderr, "[hs_b200] class-pair tables: %u x %u classes, modelled %.4f candidates/byte, "
                            "%zu prefilter keys\n", pt.nClass0, pt.nClass1, pt.modelRate, keys.size());
        }
        table.resize(sizeof(pt.classWord) + sizeof(pt.pair));
        memcpy(table.data(), pt.classWord, sizeof(pt.classWord));
        memcpy(table.data() + sizeof(pt.classWord), pt.pair, sizeof(pt.pair));
        if (keyed) {
            im->keyBytes = kb;
            im->bitmapBits = 262144;
            buildPairBitmaps(keys, im->bitmapBits, &bitmap, &bitmap2, &im->bitmap2Shift);
        }
    };
    if (shape == SHAPE_SOLE_OUTFIX || shape == SHAPE_OUTFIXES) {
        im->kind = FK_OUTFIX;
        im->groups = 0;
    } else if (hw->type == HWLM_ENGINE_NOOD) {
        /* single literal: one bucket, slots = the last <= 4 bytes of msk/cmp
         * (first char in the low byte: src/hwlm/noodle_build.cpp:100-118) */
        NoodTable n;
        memcpy(&n, bc + engOff, sizeof(n));
        im->confirmKind = CK_NOODLE;
        im->engineOff = engOff;
        im->kind = FK_BYTE32;
        table.assign(256 * 4, 0);
        for (u32 b = 0; b < 256; b++) {
            u32 e = 0;
            for (u32 p = 0; p < 4; p++) {
                u8 v = 0xfe; /* buckets 1..7 never match */
                if (p < n.msk_len) {
                    const u32 i = n.msk_len - 1 - p;
                    const u8 m = (u8)(n.msk >> (8 * i)), c = (u8)(n.cmp >> (8 * i));
                    if ((b & m) != c) {
                        v |= 1;
                    }
                }
                e |= (u32)v << (8 * p);
            }
            memcpy(&table[b * 4], &e, 4);
        }
    } else {
        /* FDR or Teddy: loadReportRules refused any other matcher */
        FDR f;
        memcpy(&f, bc + engOff, sizeof(f));
        im->confirmKind = CK_FDR;
        im->confOff = engOff + f.confOffset;
        if (f.engineID == 0) {
            pairStage(true);
        } else if (teddyNumBuckets(f.engineID) == 16) {
            /* fat Teddy (49..96 literals): the class-pair kernel with 8 bucket bits that
             * carry buckets i and i + 8 (confirmKernel unfolds them) */
            pairStage(false);
            im->bucketFold = 1;
        } else {
            /* per-byte entry: slot m = lo_m[b & 15] | hi_m[b >> 4]
             * (src/fdr/teddy.c:918-969, teddy_compile.cpp:440-509) */
            const u32 nm = teddyNumMasks(f.engineID);
            const u8 *mb = bc + engOff + TEDDY_MASK_OFFSET;
            im->kind = FK_BYTE32;
            table.assign(256 * 4, 0);
            for (u32 b = 0; b < 256; b++) {
                u32 e = 0;
                for (u32 m = 0; m < nm; m++) {
                    e |= (u32)(u8)(mb[2 * m * 16 + (b & 15)] | mb[(2 * m + 1) * 16 + (b >> 4)]) << (8 * m);
                }
                memcpy(&table[b * 4], &e, 4);
            }
        }
    }
    if (im->kind == FK_BYTE32) {
        bitmap = buildBitmap(tails, &im->keyBytes, &im->bitmapShift, &bitmap2, &im->bitmap2Shift);
    }
    if (bitmap2.empty()) {
        im->bitmap2Shift = 0;
    }
    im->tableBytes = (u32)table.size();
    im->bitmapBytes = (u32)bitmap.size();
    cudaError_t e = cudaSuccess;
    auto upload = [&](u8 **d, const void *src, size_t bytes, size_t allocBytes) {
        if (e == cudaSuccess && bytes) {
            e = cudaMalloc(d, allocBytes);
            if (e == cudaSuccess) {
                e = cudaMemcpy(*d, src, bytes, cudaMemcpyHostToDevice);
            }
        }
    };
    upload(&im->d_bc, bc, h->length, HSB_ROUNDUP(h->length, 16));
    upload(&im->d_table, table.data(), table.size(), HSB_ROUNDUP(table.size(), 16));
    upload(&im->d_bitmap, bitmap.data(), bitmap.size(), bitmap.size());
    upload(&im->d_bitmap2, bitmap2.data(), bitmap2.size(), bitmap2.size());
    if (e != cudaSuccess) {
        return e == cudaErrorMemoryAllocation ? HS_NOMEM : HS_UNKNOWN_ERROR;
    }
    im->deviceBytes = HSB_ROUNDUP(h->length, 16) + HSB_ROUNDUP(table.size(), 16) + bitmap.size() + bitmap2.size();
    for (size_t q = 0; q < im->engines.size(); q++) {
        im->engineRuns[q].nfa = im->d_bc + im->engines[q].first;
    }
    if (shape == SHAPE_OUTFIXES) {
        const hs_error_t fused = fuseEngineRuns(im.get());
        if (fused != HS_SUCCESS) {
            return fused;
        }
    }
    const hs_error_t ordered = uploadOrderTables(im.get());
    if (ordered != HS_SUCCESS) {
        return ordered;
    }
    *out = im.release();
    return HS_SUCCESS;
}

} // namespace

/* ---- corpus handle --------------------------------------------------------- */

struct hs_b200_corpus {
    int device = 0;
    u8 *d_alloc = nullptr;   /* owned allocation (nullptr when wrapping) */
    u8 *d_data = nullptr;    /* corpus position 0 */
    u64 bytes = 0;           /* end of the last block */
    u64 readableEnd = 0;
    u64 *d_off = nullptr;
    u32 *d_len = nullptr;
    size_t nblocks = 0;
    u32 uniformPitch = 0;
    u32 uniformLen = 0;      /* all blocks equally long (and uniformPitch set): tables not needed */
    u64 payload = 0;         /* sum of block lengths */
    size_t capData = 0, capBlocks = 0; /* allocation sizes when reused */
    /* the pitched corpus of a stream set (kernels.h ScanParams.streamPitch) */
    u32 streamPitch = 0;
    const u8 *streamHist = nullptr;
    const u64 *streamOffset = nullptr;
    std::vector<u32> h_len;  /* block lengths, for the end-of-block evaluation of logical combinations */
    u32 maxLen = 0;          /* the longest block (resident corpora): bounds a match's end offset */
    /* a row scan's staging corpus (hs_b200_scan_rows_async): its block table is filled on the device, h_len is
     * empty, `bytes` is the host's bound and `payload` the size of the rows' chars, which bounds their sum */
    bool deviceTables = false;
};

/* ---- scratch ------------------------------------------------------------------ */

struct hs_scratch {
    u32 magic;
    u8 in_use;
    int device;
    void *alloc_base;        /* what g_scratch_alloc returned */
    cudaStream_t stream, copyStream;
    cudaEvent_t evStart, evStop;
    cudaEvent_t evDone;       /* counters of the pending scan have landed on the host */
    std::vector<cudaEvent_t> *chunkEvents;
    std::vector<DevImage *> *images;
    DevMatch *d_out;         /* 2 * outCap records: the ring, then the scan kernels' candidate list */
    u32 outCap;
    u32 *d_counters;
    u32 *h_counters;         /* pinned */
    hs_b200_corpus *inlineCorpus; /* staging for hs_scan / hs_b200_scan_blocks */
    const hs_b200_corpus *lastCorpus; /* of the last resident scan: its block lengths, for hs_b200_fetch_matches */
    u8 *h_stage, *h_stage2;  /* pinned pack buffers (unaligned host blocks), alternating */
    size_t h_stageCap, h_stage2Cap;
    cudaEvent_t evStage, evStage2;
    std::vector<u64> *tmpOff;
    /* fused exchange over peer memory (hs_b200_set_peer_exchange) */
    u32 nPeers, myRank, peerCap, blockBase;
    DevMatch *peers[MAX_PEERS];
    bool pending;
    u32 lastCount;
    /* of the last hs_b200_scan_corpus_async: bounds of its records' block and end offset, for the sort key
     * of hs_b200_order_matches_async */
    u64 lastBlocks, lastMaxLen;
    /* of the last scan, when it was a stream-set pass: its set's epoch (StreamMark), which finishScan advances
     * once it has seen the set marked; null otherwise */
    u32 *streamEpoch;
    /* temporaries of hs_b200_order_*_async (order_kernels.h), grown on demand */
    u8 *d_order;
    size_t orderBytes;
    /* of hs_b200_scan_rows_async and hs_b200_streams_scan_rows_async: the staging corpus, and the plan's temporaries
     * (rows_kernels.h, stream_rows_kernels.h), grown on demand */
    hs_b200_corpus *rowsCorpus;
    u8 *d_rows;
    size_t rowsBytes;
    SegArea *seg;            /* of the engine runs, created on first use */
    float lastMs;
    int smCount, maxSmem;
};

namespace {

hs_error_t validDb(const hs_database_t *db) { /* src/database.h:125-137 */
    const DbHeader *h = (const DbHeader *)db;
    if (!h || h->magic != DB_MAGIC) {
        return HS_INVALID;
    }
    if (h->version != DB_VERSION) {
        return HS_DB_VERSION_ERROR;
    }
    return HS_SUCCESS;
}

/* A database the scan entry points of `mode` accept: valid, bytecode 16-byte aligned */
hs_error_t checkDb(const hs_database_t *db, u32 mode) {
    hs_error_t r = validDb(db);
    if (r != HS_SUCCESS) {
        return r;
    }
    const RoseEngine *rose = dbRose(db);
    if ((uintptr_t)rose % 16) {
        return HS_INVALID;
    }
    return rose->mode == mode ? HS_SUCCESS : HS_DB_MODE_ERROR;
}

bool validScratch(const hs_scratch *s) { return s && (uintptr_t)s % 64 == 0 && s->magic == SCRATCH_MAGIC; }

hs_error_t dbIsValid(const hs_database_t *db) { /* src/database.c:326-350 */
    hs_error_t r = validDb(db);
    if (r != HS_SUCCESS) {
        return r;
    }
    const DbHeader *h = (const DbHeader *)db;
    const u64 known = PLATFORM_NOAVX2 | PLATFORM_NOAVX512 | PLATFORM_NOAVX512VBMI;
    if (h->platform & ~known) {
        return HS_DB_PLATFORM_ERROR;
    }
    if ((uintptr_t)dbRose(db) % 16) {
        return HS_INVALID;
    }
    if (crc32c(0, (const u8 *)dbRose(db), h->length) != h->crc32) {
        return HS_INVALID;
    }
    return HS_SUCCESS;
}

bool markInUse(hs_scratch *s) { /* src/scratch.h:249-271 */
    if (s->in_use) {
        return true;
    }
    s->in_use = 1;
    return false;
}
void unmarkInUse(hs_scratch *s) { s->in_use = 0; }

hs_error_t findImage(hs_scratch *s, const hs_database_t *db, DevImage **out) {
    const DbHeader *h = (const DbHeader *)db;
    for (DevImage *im : *s->images) {
        if (im->db == db && im->crc == h->crc32 && im->length == h->length) {
            *out = im;
            return HS_SUCCESS;
        }
    }
    DeviceGuard guard(s->device); /* the image is allocated on the scratch's device */
    DevImage *im = nullptr;
    hs_error_t r = buildImage(db, &im);
    if (r != HS_SUCCESS) {
        return r;
    }
    s->images->push_back(im);
    *out = im;
    return HS_SUCCESS;
}

hs_error_t growRing(hs_scratch *s, u32 cap) {
    if (cap <= s->outCap) {
        return HS_SUCCESS;
    }
    DeviceGuard guard(s->device);
    DevMatch *n = nullptr;
    CUDA_TRY(cudaMalloc(&n, (size_t)cap * sizeof(DevMatch) * 2));
    cudaFree(s->d_out);
    s->d_out = n;
    s->outCap = cap;
    return HS_SUCCESS;
}

/* After a scan that produced `count` records into a ring too small for them: grow it
 * with a quarter to spare, so that the rescan fits */
hs_error_t growRingFor(hs_scratch *s, u32 count) {
    return growRing(s, (u32)std::min<u64>((u64)count + count / 4 + 1024, 0xfffffff0ull));
}

void freeCorpus(hs_b200_corpus *c) {
    if (!c) {
        return;
    }
    cudaFree(c->d_alloc);
    cudaFree(c->d_off);
    cudaFree(c->d_len);
    delete c;
}

/* (Re)size a corpus handle's device buffers (grow-only). */
hs_error_t reserveCorpus(hs_b200_corpus *c, u64 dataBytes, size_t nblocks) {
    DeviceGuard guard(c->device);
    const size_t need = FRONT_PAD + HSB_ROUNDUP(dataBytes, 16) + 64;
    if (need > c->capData) {
        cudaFree(c->d_alloc);
        c->d_alloc = nullptr;
        c->capData = 0;
        const size_t cap = need + need / 8;
        CUDA_TRY(cudaMalloc(&c->d_alloc, cap));
        CUDA_TRY(cudaMemset(c->d_alloc, 0, FRONT_PAD));
        c->capData = cap;
    }
    c->d_data = c->d_alloc + FRONT_PAD;
    if (nblocks > c->capBlocks) {
        cudaFree(c->d_off);
        cudaFree(c->d_len);
        c->d_off = nullptr;
        c->d_len = nullptr;
        c->capBlocks = 0;
        const size_t cap = nblocks + nblocks / 8 + 16;
        CUDA_TRY(cudaMalloc(&c->d_off, cap * sizeof(u64)));
        CUDA_TRY(cudaMalloc(&c->d_len, cap * sizeof(u32)));
        c->capBlocks = cap;
    }
    return HS_SUCCESS;
}

u32 detectPitch(const u64 *off, const u32 *len, size_t n) {
    if (n == 0) {
        return 0;
    }
    if (n == 1) {
        return off[0] == 0 ? (u32)std::max<u64>(16, HSB_ROUNDUP((u64)len[0], 16)) : 0;
    }
    const u64 pitch = off[1] - off[0];
    if (off[0] != 0 || pitch == 0 || pitch > 0xffffffffu) {
        return 0;
    }
    for (size_t i = 0; i < n; i++) {
        if (off[i] != i * pitch || len[i] > pitch) {
            return 0;
        }
    }
    return (u32)pitch;
}

struct ScanPlan {
    LaunchCfg cfg;
    u32 tileBytes, pfDist;
};

hs_error_t planScan(const hs_scratch *s, const DevImage *im, ScanPlan *pl) {
    initOpts();
    memset(&pl->cfg, 0, sizeof(pl->cfg));
    if (im->kind == FK_OUTFIX) { /* one launch over all blocks once the corpus has arrived (launchRange) */
        pl->tileBytes = 1u << 20;
        pl->pfDist = 0;
        return HS_SUCCESS;
    }
    /* the wide kernel (FK_BYTE32) is built for 768, 896 and 1024 threads, the pair and
     * gram kernels for 768 and 896; as many warps as the shared memory has queues for */
    const bool wide = im->kind == FK_BYTE32;
    int warps = g_opts.warps > 0 ? std::min(wide ? 32 : 28, g_opts.warps) : 28;
    const u32 tableBytes = im->kind == FK_PAIR32 ? im->pairBytes : im->tableBytes;
    while (warps > 1 && scanSmemBytes(im->kind, tableBytes, im->bitmapBytes, warps) > (size_t)s->maxSmem) {
        warps--;
    }
    pl->cfg.smemBytes = scanSmemBytes(im->kind, tableBytes, im->bitmapBytes, warps);
    if (pl->cfg.smemBytes > (size_t)s->maxSmem) {
        return HS_NOMEM;
    }
    pl->cfg.kind = im->kind;
    pl->cfg.slotBase = im->slotBase;
    /* pair-kernel candidate path: one queue entry per word with candidates.  Its drain needs
     * no corpus read and reserves list slots once per warp, and it was level or faster on
     * every set measured, from 0.015 to 7 candidates per KiB (DESIGN.md section 3.3);
     * heavy=0 selects the per-lane entries */
    pl->cfg.heavy = im->kind == FK_PAIR32 && g_opts.heavy != 0;
    pl->cfg.grid = s->smCount;
    pl->cfg.warps = warps;
    pl->tileBytes = (u32)std::max(512, g_opts.tileBytes) & ~511u;
    if (wide) {
        pl->tileBytes = std::max(1024u, pl->tileBytes & ~1023u); /* a warp-iteration covers 1 KiB */
    }
    const int pfDist = g_opts.pfDist >= 0 ? g_opts.pfDist : im->kind == FK_PAIR32 ? 2 : 4;
    pl->pfDist = (u32)std::min(64, pfDist);
    return HS_SUCCESS;
}

void fillParams(const hs_scratch *s, const DevImage *im, const hs_b200_corpus *c,
                const ScanPlan &pl, ScanParams *p) {
    memset(p, 0, sizeof(*p));
    p->corpus = c->d_data;
    p->corpusBytes = c->bytes;
    p->readableEnd = c->readableEnd;
    p->tileBytes = pl.tileBytes;
    p->pfDist = pl.pfDist;
    p->blockOff = c->d_off;
    p->blockLen = c->d_len;
    p->nblocks = (u32)c->nblocks;
    p->uniformPitch = c->uniformPitch;
    p->uniformLen = c->uniformLen;
    p->streamPitch = c->streamPitch;
    p->streamHist = c->streamHist;
    p->streamOffset = c->streamOffset;
    p->bc = im->d_bc;
    p->table = im->d_table;
    p->tableBytes = im->tableBytes;
    p->bitmap = im->d_bitmap;
    p->bitmapBytes = im->bitmapBytes;
    p->pairBytes = im->pairBytes;
    p->bucketFold = im->bucketFold;
    p->bitmapBits = im->bitmapBits;
    p->bitmapShift = im->bitmapShift;
    p->keyBytes = im->keyBytes;
    p->bitmap2 = (const u32 *)im->d_bitmap2;
    p->bitmap2Shift = im->d_bitmap2 ? im->bitmap2Shift : 0;
    p->confOff = im->confOff;
    p->engineOff = im->engineOff;
    p->confirmKind = im->confirmKind;
    p->groups = im->groups;
    p->out = s->d_out;
    p->outCap = s->outCap;
    p->counters = s->d_counters;
    p->nPeers = s->nPeers;
    p->myRank = s->myRank;
    p->peerCap = s->peerCap;
    p->blockBase = s->blockBase;
    for (u32 r = 0; r < s->nPeers; r++) {
        p->peers[r] = s->peers[r];
    }
}

/* The segment plan of the default rule (engine_segment = 0; DESIGN.md section 10f): a run of `engines` engines has
 * engines x blocks lanes of work, and blocks are cut only when that would leave more than half of the lanes the
 * run keeps resident idle, and only blocks longer than twice the segment length.  That length is at least SEG_MIN
 * and otherwise as long as makes engines x segments about fill the resident lanes, so that the segment states
 * (engines x 2 x segments) stay bounded by the GPU, not by the engine count.  A segment's guess comes from
 * SEG_WARM bytes in front of it; SEG_ROUNDS parallel SEG_JOIN rounds precede the sequential SEG_SETTLE walk.  A
 * forced length (engine_segment = N > 0) whose segment area would pass SEG_FORCED_MAX fails the scan with
 * HS_NOMEM. */
enum : u32 { SEG_MIN = 4096, SEG_WARM = 256, SEG_ROUNDS = 2 };
static const size_t SEG_FORCED_MAX = (size_t)1 << 30;

/* The rule from the block count and the payload alone: may blocks of c be cut for a run of `engines` engines of
 * `kind`, and if so, into segments of *segLen bytes, the blocks longer than *cutAbove. */
bool segmentRule(const hs_b200_corpus *c, u32 kind, u64 engines, int smCount, u64 *segLen, u64 *cutAbove) {
    const int opt = g_opts.engineSegment;
    if (opt < 0 || c->nblocks == 0) {
        return false;
    }
    *segLen = *cutAbove = (u64)opt;
    if (opt == 0) {
        const u64 lanes = dfaResidentLanes(kind, smCount);
        if (engines * c->nblocks * 2 > lanes) {
            return false; /* the blocks alone keep half the resident lanes busy or more */
        }
        *segLen = std::max<u64>(SEG_MIN, HSB_ROUNDUP(c->payload * engines / lanes + 1, 16));
        *cutAbove = 2 * *segLen;
    }
    return true;
}

/* Cut the blocks of c for a run of `engines` engines of `kind`?  Fills the segment table (every block, in order: a
 * block not cut is one segment with both flags) and the cut blocks {first segment, segments}; false: one lane per
 * block. */
bool planSegments(const hs_b200_corpus *c, u32 kind, u64 engines, int smCount, std::vector<DfaSeg> *segs,
                  std::vector<uint2> *cuts) {
    u64 segLen = 0, cutAbove = 0;
    if (c->h_len.size() != c->nblocks || !segmentRule(c, kind, engines, smCount, &segLen, &cutAbove)) {
        return false;
    }
    if (*std::max_element(c->h_len.begin(), c->h_len.end()) <= cutAbove) {
        return false;
    }
    segs->clear();
    cuts->clear();
    for (size_t b = 0; b < c->nblocks; b++) {
        const u32 len = c->h_len[b];
        if (len <= cutAbove) {
            segs->push_back({(u32)b, 0, len, SEG_FIRST | SEG_LAST});
            continue;
        }
        const u32 n = (u32)((len + segLen - 1) / segLen);
        cuts->push_back(make_uint2((u32)segs->size(), n));
        for (u32 i = 0; i < n; i++) {
            const u32 start = (u32)(i * segLen);
            segs->push_back({(u32)b, start, (u32)std::min<u64>(segLen, len - start),
                             (i == 0 ? (u32)SEG_FIRST : 0u) | (i == n - 1 ? (u32)SEG_LAST : 0u)});
        }
    }
    return true;
}

/* Run an engine (dp from engineParams, dp.nfa its bytes in device memory), or a fused launch of several
 * (dp.engines), over every block of corpus c, into the record ring out[0, outCap) and its counters.  Long
 * blocks are cut into segments walked by lanes of their own (planSegments); `seg` holds their plan and states.
 * A corpus whose block lengths only the device knows (deviceTables) gets its plan from launchRowSegments, in
 * lists sized by the bound the payload sets: no block may be cut when the payload is no longer than cutAbove. */
cudaError_t launchEngine(DfaParams dp, const hs_b200_corpus *c, DevMatch *out, u32 outCap,
                         u32 *counters, int smCount, int maxSmem, SegArea *seg, cudaStream_t stream) {
    dp.corpus = c->d_data;
    dp.readableEnd = c->readableEnd;
    dp.blockOff = c->d_off;
    dp.blockLen = c->d_len;
    dp.nblocks = (u32)c->nblocks;
    dp.uniformPitch = c->uniformPitch;
    dp.uniformLen = c->uniformLen;
    dp.out = out;
    dp.outCap = outCap;
    dp.counters = counters;
    initOpts();
    std::vector<DfaSeg> segs;
    std::vector<uint2> cuts;
    const size_t engines = dp.engines ? dp.nengines : 1;
    u64 segLen = 0, cutAbove = 0, nsegs = 0, ncuts = 0;
    const bool devicePlan = c->deviceTables && segmentRule(c, dp.kind, engines, smCount, &segLen, &cutAbove) &&
                            c->payload > cutAbove;
    if (devicePlan) {
        nsegs = c->nblocks + c->payload / segLen + 1;
        ncuts = std::min<u64>(c->nblocks, c->payload / (cutAbove + 1));
        if (nsegs > 0xfffffff0ull) {
            return cudaErrorMemoryAllocation;
        }
    } else if (planSegments(c, dp.kind, engines, smCount, &segs, &cuts)) {
        nsegs = segs.size();
        ncuts = cuts.size();
    } else {
        const cudaError_t e = launchDfa(dp, smCount, maxSmem, stream);
        if (e == cudaSuccess) {
            g_launches++;
        }
        return e;
    }
    /* [segs][cuts][device plans: the first segment of every block][per engine, per block: first open segment]
     * [per engine: guess states, end states] */
    const size_t segBytes = HSB_ROUNDUP(nsegs * sizeof(DfaSeg), 256);
    const size_t cutBytes = HSB_ROUNDUP(ncuts * sizeof(uint2), 256);
    const size_t planBytes = segBytes + (devicePlan ? cutBytes + (c->nblocks + 1) * sizeof(u32) : ncuts * sizeof(uint2));
    const size_t openBytes = HSB_ROUNDUP(engines * c->nblocks * sizeof(u32), 256);
    const size_t statesAt = HSB_ROUNDUP(planBytes, 256) + openBytes;
    const size_t need = statesAt + engines * 2 * nsegs * dfaStateBytes(dp.kind);
    if (g_opts.engineSegment > 0 && need > SEG_FORCED_MAX) {
        return cudaErrorMemoryAllocation; /* a forced length too short for this corpus and engine count */
    }
    if (!seg->d_stats) {
        cudaError_t e = cudaMalloc(&seg->d_stats, SEGSTAT_COUNT * sizeof(unsigned long long));
        if (e == cudaSuccess) e = cudaMemset(seg->d_stats, 0, SEGSTAT_COUNT * sizeof(unsigned long long));
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&seg->copied, cudaEventDisableTiming);
        if (e != cudaSuccess) {
            return e;
        }
    }
    if (need > seg->bytes) {
        cudaFree(seg->d); /* (synchronises with any run still using it) */
        seg->d = nullptr;
        seg->bytes = 0;
        seg->plan.clear();
        const cudaError_t e = cudaMalloc(&seg->d, need + need / 4);
        if (e != cudaSuccess) {
            return e;
        }
        seg->bytes = need + need / 4;
    }
    cudaError_t e = cudaSuccess;
    if (devicePlan) {
        RowSegParams rp;
        rp.blockLen = c->d_len;
        rp.nrows = (u32)c->nblocks;
        rp.segLen = (u32)segLen;
        rp.cutAbove = (u32)std::min<u64>(cutAbove, 0xffffffffull);
        rp.segs = reinterpret_cast<DfaSeg *>(seg->d);
        rp.segCap = (u32)nsegs;
        rp.cuts = reinterpret_cast<uint2 *>(seg->d + segBytes);
        rp.cutCap = (u32)ncuts;
        rp.segFirst = reinterpret_cast<u32 *>(seg->d + segBytes + cutBytes);
        seg->plan.clear(); /* what is in device memory is no host plan's image */
        unsigned launched = 0;
        e = launchRowSegments(rp, smCount, stream, &launched);
        g_launches += launched;
        if (e != cudaSuccess) {
            return e;
        }
    }
    /* the plan's image; copied only when it differs from the one in device memory (a scan of the same corpus
     * again, or the next engine kind of the same scan, reuses it) */
    std::vector<u8> image;
    if (!devicePlan) {
        image.assign(planBytes, 0);
        memcpy(image.data(), segs.data(), segs.size() * sizeof(DfaSeg));
        memcpy(image.data() + segBytes, cuts.data(), cuts.size() * sizeof(uint2));
    }
    if (!devicePlan && image != seg->plan) {
        e = cudaEventSynchronize(seg->copied); /* the last copy out of the pinned buffer has been made */
        if (e == cudaSuccess && planBytes > seg->hBytes) {
            cudaFreeHost(seg->h);
            seg->h = nullptr;
            seg->hBytes = 0;
            e = cudaMallocHost(&seg->h, planBytes + planBytes / 4);
            if (e == cudaSuccess) {
                seg->hBytes = planBytes + planBytes / 4;
            }
        }
        if (e == cudaSuccess) {
            memcpy(seg->h, image.data(), planBytes);
            e = cudaMemcpyAsync(seg->d, seg->h, planBytes, cudaMemcpyHostToDevice, stream);
        }
        if (e == cudaSuccess) e = cudaEventRecord(seg->copied, stream);
        if (e != cudaSuccess) {
            seg->plan.clear();
            return e;
        }
        seg->plan.swap(image);
    }
    u32 *open = reinterpret_cast<u32 *>(seg->d + HSB_ROUNDUP(planBytes, 256));
    e = cudaMemsetAsync(open, 0xff, engines * c->nblocks * sizeof(u32), stream);
    if (e != cudaSuccess) {
        return e;
    }
    dp.segs = reinterpret_cast<const DfaSeg *>(seg->d);
    dp.nsegs = (u32)nsegs;
    dp.cuts = reinterpret_cast<const uint2 *>(seg->d + segBytes);
    dp.ncuts = (u32)ncuts;
    dp.warm = SEG_WARM;
    dp.segOpen = open;
    dp.segStates = seg->d + statesAt;
    dp.segStats = seg->d_stats;
    unsigned launches = 0;
    e = launchDfaSegments(dp, smCount, maxSmem, SEG_ROUNDS, stream, &launches);
    g_launches += launches;
    if (e == cudaSuccess) {
        seg->runs++;
        seg->segments += nsegs;
    }
    return e;
}

/* Launch over tiles [t0, t1) of the corpus on `stream`; t0 == 0 is the first range of a
 * scan, whose counters were all cleared just before.  mask != null: a mask or first-match pass. */
hs_error_t launchRange(hs_scratch *s, const DevImage *im, const hs_b200_corpus *c,
                       const ScanPlan &pl, u32 t0, u32 t1, cudaStream_t stream, const MaskOut *mask) {
    if (t1 <= t0) {
        return HS_SUCCESS;
    }
    if (im->kind != FK_OUTFIX) {
        ScanParams p;
        fillParams(s, im, c, pl, &p);
        if (mask) {
            p.mask = *mask;
        }
        p.tileFirst = t0;
        p.ntiles = t1 - t0;
        LaunchCfg cfg = pl.cfg;
        const u32 perCta = (u32)cfg.warps;
        cfg.grid = (int)std::min<u32>((u32)cfg.grid, (p.ntiles + perCta - 1) / perCta);
        if (t0 > 0) {
            CUDA_TRY(cudaMemsetAsync(s->d_counters + CTR_CANDQ, 0, sizeof(u32), stream));
        }
        CUDA_TRY(launchScan(cfg, p, stream));
        g_launches++;
        CUDA_TRY(launchConfirm(cfg, p, stream));
        g_launches++;
    }
    if (!im->engineRuns.empty()) {
        /* a block is one thread's walk from its first byte: after the last range of the corpus,
         * the engines run over every block, into the same record ring (whose count only ever grows by
         * whole groups of eight slots while no literal record is in it: the fused launches need no
         * alignSharedRing between them) */
        const u32 ntiles = (u32)((c->bytes + pl.tileBytes - 1) / pl.tileBytes);
        if (t1 >= ntiles) {
            for (DfaParams dp : im->engineRuns) {
                if (mask) {
                    dp.mask = *mask;
                }
                if (!s->seg) {
                    s->seg = new (std::nothrow) SegArea();
                    if (!s->seg) {
                        return HS_NOMEM;
                    }
                }
                CUDA_TRY(launchEngine(dp, c, s->d_out, s->outCap, s->d_counters, s->smCount, s->maxSmem, s->seg,
                                      stream));
            }
        }
    }
    return HS_SUCCESS;
}

hs_error_t finishScan(hs_scratch *s, u32 *count) {
    /* wait for THIS scan only: a later scan may already be queued behind it
     * on the same stream (double-buffered callers) */
    cudaError_t e = cudaEventSynchronize(s->evDone);
    s->pending = false;
    if (e != cudaSuccess) {
        return HS_UNKNOWN_ERROR;
    }
    cudaEventElapsedTime(&s->lastMs, s->evStart, s->evStop);
    const u32 stream = s->h_counters[CTR_STREAM];
    if (stream && s->streamEpoch) {
        /* a stream-set pass did not commit: the passes and resets enqueued from now on belong to the next epoch,
         * which the mark does not hold back (no device work: a reset enqueued before may still be pending) */
        *s->streamEpoch = *s->streamEpoch + 1 == 0xffffffffu ? 0 : *s->streamEpoch + 1;
    }
    if (s->h_counters[CTR_ERROR]) {
        return HS_UNKNOWN_ERROR;
    }
    if (stream & STREAM_BAD_LENGTH) {
        s->lastCount = 0;
        return HS_INVALID;
    }
    *count = s->h_counters[CTR_MATCHES];
    s->lastCount = *count;
    return HS_SUCCESS;
}

/* A corpus still on its way from the host, in nchunks pieces.  chunk(ci, &covered)
 * issues piece ci's copy, makes the scan stream wait for it, and returns how long a
 * prefix of the corpus is then on the device.  The scan launches the tiles of that
 * prefix before it asks for the next piece, so each copy (and the host-side packing
 * of the next piece) overlaps the kernels of the pieces before it. */
struct Upload {
    size_t nchunks;
    std::function<hs_error_t(size_t ci, u64 *covered)> chunk;
};

/* The device half of one stream-set pass over a pitched corpus (hs_b200_streams_*): the set's state and, for
 * writes whose lengths the caller keeps in device memory, those lengths. */
struct StreamPass {
    u8 *hist;
    u64 *offset;
    u32 *len;            /* the lengths the scan reads (the corpus's blockLen) */
    const u32 *srcLen;   /* != null: the caller's, checked and copied into len by the assemble kernel */
    u32 histReq;
    StreamMark *mark;
    u32 *epoch;          /* the set's epoch (host memory), read at enqueue time */
};

/* Enqueue a scan of the whole corpus on `stream`: reset the counters, launch the tile
 * ranges, read the counters back.  The only place a scan's stream sequence is issued.
 * For a stream-set pass (sp), the look-behind is written in front of every write first,
 * and the streams advance -- or the set is marked -- before the counters are read back.
 * For a row scan (rows), the row plan fills c's block table and packs the rows into it first.
 * For a stream-set pass over rows (srows), the rows are grouped by stream and packed into c first, and the records
 * are rewritten to rows and stream offsets and the streams advance -- or the set is marked -- after the scan; a mask
 * pass over rows has no records to rewrite (its confirm kernel maps every match to its row) and only advances.
 * For a mask pass (mask), the caller's mask is zeroed before the scan, which sets bits instead of writing records,
 * and *status (if given) receives the pass's verdict last, after a stream set's advance: a pass the set did not
 * commit has its record count raised above the ring by then (streamPassCommits).  A first-match pass (mask->first)
 * is the same sequence with its table filled with ones instead. */
/* the first kernel of a mask or first-match pass: every word of the caller's output written before the scan */
static cudaError_t clearOutput(const MaskOut &m, size_t nblocks, int smCount, cudaStream_t stream) {
    return m.first ? launchMaskClear(reinterpret_cast<u32 *>(m.first), 2 * (u64)nblocks, smCount, stream, true)
                   : launchMaskClear(m.bits, (u64)nblocks * m.words, smCount, stream);
}

hs_error_t enqueueScan(hs_scratch *s, const DevImage *im, const hs_b200_corpus *c,
                       cudaStream_t stream, const Upload *up = nullptr, const StreamPass *sp = nullptr,
                       const RowsParams *rows = nullptr, const MaskOut *mask = nullptr, u32 *status = nullptr,
                       const StreamRowsParams *srows = nullptr) {
    if (s->nPeers && (im->rules.shape == SHAPE_LITERALS_OUTFIX || im->rules.shape == SHAPE_OUTFIXES)) {
        /* the engine kernel stores no records into the peers' exchange buffers, and the count it
         * publishes would cover them: an exchange of both halves' records, or of several engines',
         * is not built */
        return HS_ARCH_ERROR;
    }
    ScanPlan pl;
    hs_error_t r = planScan(s, im, &pl);
    if (r != HS_SUCCESS) {
        return r;
    }
    CUDA_TRY(cudaMemsetAsync(s->d_counters, 0, CTR_COUNT * sizeof(u32), stream));
    if (mask) {
        CUDA_TRY(clearOutput(*mask, c->nblocks, s->smCount, stream));
        g_launches++;
    }
    if (sp) {
        CUDA_TRY(launchStreamAssemble(c->d_data, sp->hist, (u32)c->nblocks, c->streamPitch, sp->srcLen, sp->len,
                                      sp->mark, *sp->epoch, stream));
        g_launches++;
    }
    if (rows) {
        unsigned launched = 0;
        CUDA_TRY(launchRowPlan(*rows, s->smCount, stream, &launched));
        g_launches += launched;
    }
    if (srows) {
        unsigned launched = 0;
        CUDA_TRY(cudaMemsetAsync(srows->head, 0, sizeof(StreamRowsHead), stream));
        CUDA_TRY(launchStreamRowsPlan(*srows, s->smCount, stream, &launched));
        g_launches += launched;
    }
    CUDA_TRY(cudaEventRecord(s->evStart, stream));
    const u32 ntiles = (u32)((c->bytes + pl.tileBytes - 1) / pl.tileBytes);
    u32 tDone = 0;
    for (size_t ci = 0; up && ci < up->nchunks; ci++) {
        u64 covered = 0;
        r = up->chunk(ci, &covered);
        if (r != HS_SUCCESS) {
            return r;
        }
        /* tiles wholly inside the copied prefix (plus look-ahead) */
        const u32 tEnd = covered >= c->bytes ? ntiles : covered > 16 ? (u32)((covered - 16) / pl.tileBytes) : 0;
        r = launchRange(s, im, c, pl, tDone, tEnd, stream, mask);
        if (r != HS_SUCCESS) {
            return r;
        }
        tDone = std::max(tDone, tEnd);
    }
    r = launchRange(s, im, c, pl, tDone, ntiles, stream, mask);
    if (r != HS_SUCCESS) {
        return r;
    }
    CUDA_TRY(cudaEventRecord(s->evStop, stream));
    if (sp) {
        CUDA_TRY(launchStreamAdvance(c->d_data, sp->hist, sp->offset, sp->len, c->uniformLen, (u32)c->nblocks,
                                     c->streamPitch, sp->histReq, s->d_counters, s->outCap, sp->mark, *sp->epoch,
                                     stream));
        g_launches++;
    }
    if (srows) {
        unsigned launched = 0;
        CUDA_TRY(launchStreamRowsCommit(*srows, mask != nullptr, s->smCount, stream, &launched));
        g_launches += launched;
    }
    s->streamEpoch = sp ? sp->epoch : nullptr;
    if (status) {
        CUDA_TRY(launchMaskStatus(s->d_counters, s->outCap, status, stream));
        g_launches++;
    }
    if (s->nPeers) {
        ScanParams pp;
        fillParams(s, im, c, pl, &pp);
        CUDA_TRY(launchPublishCount(pp, stream));
        g_launches++;
    }
    CUDA_TRY(cudaMemcpyAsync(s->h_counters, s->d_counters, CTR_COUNT * sizeof(u32),
                             cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaEventRecord(s->evDone, stream));
    s->pending = true;
    return HS_SUCCESS;
}

double nowMs() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct ScanTimes {
    double enqueued = 0, waited = 0, read = 0; /* nowMs() after each step of the last pass */
};

/* Scan a corpus on the scratch's stream (uploading it through `up`, if given) and
 * read its records back: ordered, with the report rules applied (ReportRules::deliver), or
 * raw when !ordered.  When the record ring overflows, it grows and the corpus, resident
 * by then, is scanned again as one range.  A second pass finds the real record count;
 * a third may be needed, because the candidate list can overflow before the ring does.
 * A third overflow is an error.  A first pass that uploads the corpus in several chunks
 * runs one range per chunk, and each range reports a candidate-list overflow with its own
 * candidate count only, which is too small to size the ring for one range over the whole
 * corpus.  So that pass does not count: the rescans then run exactly as for a corpus
 * that was resident from the start. */
hs_error_t scanRecords(hs_scratch *s, DevImage *im, const hs_b200_corpus *c, const Upload *up,
                       bool ordered, std::vector<DevMatch> *matches, ScanTimes *times = nullptr,
                       const u32 *lengths = nullptr, const StreamPass *sp = nullptr) {
    ScanTimes unused;
    ScanTimes &t = times ? *times : unused;
    const int passes = up && up->nchunks > 1 ? 4 : 3;
    for (int attempt = 0; attempt < passes; attempt++) {
        hs_error_t r = enqueueScan(s, im, c, s->stream, attempt == 0 ? up : nullptr, sp);
        if (r != HS_SUCCESS) {
            return r;
        }
        t.enqueued = nowMs();
        u32 count = 0;
        r = finishScan(s, &count);
        t.waited = nowMs();
        if (r != HS_SUCCESS) {
            return r;
        }
        if (count > s->outCap) {
            r = growRingFor(s, count);
            if (r != HS_SUCCESS) {
                return r;
            }
            continue;
        }
        matches->resize(count);
        if (count) {
            CUDA_TRY(cudaMemcpyAsync(matches->data(), s->d_out, (size_t)count * sizeof(DevMatch),
                                     cudaMemcpyDeviceToHost, s->stream));
            CUDA_TRY(cudaStreamSynchronize(s->stream));
        }
        t.read = nowMs();
        return ordered ? im->rules.deliver(matches, lengths, c->nblocks) : HS_SUCCESS;
    }
    return HS_UNKNOWN_ERROR;
}

/* Lay host blocks out for a corpus handle.  Returns through *direct whether the
 * caller's buffer could be copied as it lies (all starts 16-byte aligned
 * relative to the first block, ascending, disjoint), and through *uniPitch and
 * *uniLen (or zeros) that it also holds equally long blocks at a fixed pitch. */
void layoutBlocks(const unsigned long long *offsets, const unsigned *lengths, size_t nblocks,
                  std::vector<u64> *packed, u64 *total, u64 *payload, bool *direct, u32 *uniPitch, u32 *uniLen) {
    *uniPitch = *uniLen = 0;
    /* fast path (hsbench-style corpora): equally long blocks at a fixed
     * 16-byte aligned pitch -- one tight pass, no packed table at all */
    if (nblocks >= 2 && lengths[0] && offsets[1] > offsets[0]) {
        const u64 base = offsets[0], pitch = offsets[1] - offsets[0];
        const u32 len0 = lengths[0];
        if (pitch % 16 == 0 && pitch <= 0xffffffffu && len0 <= pitch) {
            /* two simple loops the compiler vectorises */
            size_t bad = 0;
            u64 expect = base;
            for (size_t i = 0; i < nblocks; i++, expect += pitch) {
                bad += offsets[i] != expect;
            }
            for (size_t i = 0; i < nblocks; i++) {
                bad += lengths[i] != len0;
            }
            if (!bad) {
                packed->clear();
                *total = (nblocks - 1) * pitch + len0;
                *payload = (u64)nblocks * len0;
                *direct = true;
                *uniPitch = (u32)pitch;
                *uniLen = len0;
                return;
            }
        }
    }
    packed->resize(nblocks);
    bool ok = nblocks > 0;
    u64 pay = 0;
    const u64 base = nblocks ? offsets[0] : 0;
    u64 prevEnd = 0;
    for (size_t i = 0; i < nblocks; i++) {
        pay += lengths[i];
        if (ok) {
            if (offsets[i] < base || (offsets[i] - base) % 16 || offsets[i] - base < prevEnd) {
                ok = false;
            } else {
                (*packed)[i] = offsets[i] - base;
                prevEnd = offsets[i] - base + lengths[i];
            }
        }
    }
    if (!ok) {
        u64 pos = 0;
        for (size_t i = 0; i < nblocks; i++) {
            (*packed)[i] = pos;
            pos += HSB_ROUNDUP((u64)lengths[i], 16);
            if (lengths[i] == 0) {
                pos += 16; /* keep starts distinct */
            }
        }
        prevEnd = nblocks ? (*packed)[nblocks - 1] + lengths[nblocks - 1] : 0;
    }
    *total = prevEnd;
    *payload = pay;
    *direct = ok;
}

} // namespace

extern "C" {

hs_error_t hs_valid_platform(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        return HS_ARCH_ERROR;
    }
    /* the library carries sm_90a code only, which loads on compute capability 9.0 alone */
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, 0);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, 0);
    return major == 9 && minor == 0 ? HS_SUCCESS : HS_ARCH_ERROR;
}

unsigned long long hs_b200_launch_count(void) { return g_launches.load(); }

float hs_b200_last_kernel_ms(const hs_scratch_t *scratch) {
    return scratch ? scratch->lastMs : 0.0f;
}

/* Counters of the last finished scan: [0] raw records, [1] error, [2]
 * first-stage candidates, [3] byte-confirmed literals, [4] candidates that
 * passed the prefilter. */
hs_error_t hs_b200_last_counters(const hs_scratch_t *scratch, unsigned int out[8]) {
    if (!scratch || !out || scratch->pending) {
        return HS_INVALID;
    }
    memcpy(out, scratch->h_counters, CTR_COUNT * sizeof(u32));
    return HS_SUCCESS;
}

hs_error_t hs_b200_engine_segment_stats(const hs_scratch_t *scratch, unsigned long long out[4]) {
    if (!validScratch(scratch) || !out) {
        return HS_INVALID;
    }
    memset(out, 0, 4 * sizeof(unsigned long long));
    const SegArea *a = scratch->seg;
    if (!a) {
        return HS_SUCCESS;
    }
    out[0] = a->runs;
    out[1] = a->segments;
    if (a->d_stats) {
        DeviceGuard guard(scratch->device);
        if (cudaStreamSynchronize(scratch->stream) != cudaSuccess ||
            cudaMemcpy(out + 2, a->d_stats, SEGSTAT_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost) !=
                cudaSuccess) {
            return HS_UNKNOWN_ERROR;
        }
    }
    return HS_SUCCESS;
}

hs_error_t hs_b200_set_runtime_option(const char *key, int value) {
    initOpts();
    if (!key) {
        return HS_INVALID;
    }
    struct { const char *n; int *v; } k[] = {
        {"warps", &g_opts.warps},       {"tile_bytes", &g_opts.tileBytes},
        {"pf_dist", &g_opts.pfDist},    {"chunk_mb", &g_opts.chunkMB},
        {"initial_ring", &g_opts.initialRing}, {"heavy", &g_opts.heavy},
        {"gram", &g_opts.gram},         {"dfa_ilp", &g_opts.dfaIlp},
        {"engine_segment", &g_opts.engineSegment}};
    for (auto &x : k) {
        if (!strcmp(key, x.n)) {
            *x.v = value;
            return HS_SUCCESS;
        }
    }
    return HS_INVALID;
}

/* Acceleration primitives on a host buffer (src/nfa/accel.c:35 run_accel):
 * first position whose byte (pair) is in the class, or len. */
hs_error_t hs_b200_accel_find(unsigned int type, const unsigned char *params,
                              const unsigned char *buf, size_t len, unsigned long long *pos) {
    if (!params || (!buf && len) || !pos) {
        return HS_INVALID;
    }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        return HS_ARCH_ERROR;
    }
    u8 *d = nullptr;
    u64 *d_res = nullptr;
    CUDA_TRY(cudaMalloc(&d, HSB_ROUNDUP(len, 16) + 64));
    cudaError_t e = cudaMalloc(&d_res, 8);
    if (e == cudaSuccess) e = cudaMemset(d, 0, HSB_ROUNDUP(len, 16) + 64);
    if (e == cudaSuccess && len) e = cudaMemcpy(d, buf, len, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = launchAccelFind((int)type, params, d, len, d_res, 0);
    if (e == cudaSuccess) g_launches++;
    unsigned long long r = len;
    if (e == cudaSuccess) e = cudaMemcpy(&r, d_res, 8, cudaMemcpyDeviceToHost);
    cudaFree(d);
    cudaFree(d_res);
    if (e != cudaSuccess) {
        return e == cudaErrorInvalidValue ? HS_INVALID : HS_UNKNOWN_ERROR;
    }
    *pos = r;
    return HS_SUCCESS;
}

/* ---- scratch ---------------------------------------------------------------- */

static hs_error_t newScratch(hs_scratch **out) {
    initOpts();
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        return HS_ARCH_ERROR; /* no CPU scan path exists */
    }
    void *raw = g_scratch_alloc(sizeof(hs_scratch) + 64);
    hs_error_t r = checkAlloc(raw);
    if (r != HS_SUCCESS) {
        g_scratch_free(raw);
        return r;
    }
    hs_scratch *s = (hs_scratch *)HSB_ROUNDUP((uintptr_t)raw, 64);
    memset(s, 0, sizeof(*s));
    s->alloc_base = raw;
    s->magic = SCRATCH_MAGIC;
    cudaGetDevice(&s->device);
    cudaDeviceGetAttribute(&s->smCount, cudaDevAttrMultiProcessorCount, s->device);
    cudaDeviceGetAttribute(&s->maxSmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, s->device);
    s->images = new std::vector<DevImage *>();
    s->chunkEvents = new std::vector<cudaEvent_t>();
    s->tmpOff = new std::vector<u64>();
    cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->copyStream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreate(&s->evStart);
    if (e == cudaSuccess) e = cudaEventCreate(&s->evStop);
    if (e == cudaSuccess) {
        /* HSB200_BLOCKING_SYNC=1: sleep instead of spinning while a scan is awaited */
        const char *bs = getenv("HSB200_BLOCKING_SYNC");
        e = cudaEventCreateWithFlags(&s->evDone, cudaEventDisableTiming |
                                                      ((bs && *bs == '1') ? cudaEventBlockingSync : 0));
    }
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->evStage, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->evStage2, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMalloc(&s->d_counters, CTR_COUNT * sizeof(u32));
    if (e == cudaSuccess) e = cudaMallocHost(&s->h_counters, CTR_COUNT * sizeof(u32));
    if (e == cudaSuccess) {
        memset(s->h_counters, 0, CTR_COUNT * sizeof(u32));
        s->inlineCorpus = new hs_b200_corpus();
        s->inlineCorpus->device = s->device;
    }
    if (e != cudaSuccess || growRing(s, (u32)g_opts.initialRing) != HS_SUCCESS) {
        hs_free_scratch(s);
        return e == cudaErrorMemoryAllocation ? HS_NOMEM : HS_UNKNOWN_ERROR;
    }
    *out = s;
    return HS_SUCCESS;
}

hs_error_t hs_alloc_scratch(const hs_database_t *db, hs_scratch_t **scratch) {
    if (!db || !scratch) {
        return HS_INVALID;
    }
    hs_error_t r = dbIsValid(db);
    if (r != HS_SUCCESS) {
        return r;
    }
    hs_scratch *s = *scratch;
    if (s) {
        if (!validScratch(s)) {
            return HS_INVALID;
        }
        if (markInUse(s)) {
            return HS_SCRATCH_IN_USE;
        }
    } else {
        r = newScratch(&s);
        if (r != HS_SUCCESS) {
            *scratch = nullptr;
            return r;
        }
        s->in_use = 1;
    }
    DeviceGuard guard(s->device);
    DevImage *im = nullptr;
    r = findImage(s, db, &im);
    unmarkInUse(s);
    if (r != HS_SUCCESS) {
        if (!*scratch) {
            hs_free_scratch(s);
        }
        return r;
    }
    *scratch = s;
    return HS_SUCCESS;
}

hs_error_t hs_clone_scratch(const hs_scratch_t *src, hs_scratch_t **dest) {
    if (!dest || !validScratch(src)) {
        return HS_INVALID;
    }
    *dest = nullptr;
    DeviceGuard guard(src->device); /* the clone lives on the source's device */
    hs_scratch *s = nullptr;
    hs_error_t r = newScratch(&s);
    if (r != HS_SUCCESS) {
        return r;
    }
    for (const DevImage *im : *src->images) {
        /* rebuild from the source image's own copy of the database: the application may
         * have freed the original (legal in the reference, whose clone never touches it) */
        const hs_database_t *copy = (const hs_database_t *)(im->dbCopy.data() + im->dbCopyShift);
        DevImage *fresh = nullptr;
        r = buildImage(copy, &fresh);
        if (r != HS_SUCCESS) {
            hs_free_scratch(s);
            return r;
        }
        fresh->db = im->db; /* keep the identity the application knows */
        s->images->push_back(fresh);
    }
    r = growRing(s, src->outCap);
    if (r != HS_SUCCESS) {
        hs_free_scratch(s);
        return r;
    }
    *dest = s;
    return HS_SUCCESS;
}

hs_error_t hs_scratch_size(const hs_scratch_t *scratch, size_t *size) {
    if (!size || !validScratch(scratch)) {
        return HS_INVALID;
    }
    size_t n = sizeof(hs_scratch) + 64 + (size_t)scratch->outCap * sizeof(DevMatch);
    for (const DevImage *im : *scratch->images) {
        n += im->deviceBytes;
    }
    if (scratch->inlineCorpus) {
        n += scratch->inlineCorpus->capData;
    }
    if (scratch->rowsCorpus) {
        n += scratch->rowsCorpus->capData;
    }
    *size = n;
    return HS_SUCCESS;
}

hs_error_t hs_free_scratch(hs_scratch_t *s) {
    if (!s) {
        return HS_SUCCESS;
    }
    if (!validScratch(s)) {
        return HS_INVALID;
    }
    if (markInUse(s)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(s->device);
    s->magic = 0;
    if (s->stream) cudaStreamSynchronize(s->stream);
    if (s->images) {
        for (DevImage *im : *s->images) {
            freeImage(im);
        }
        delete s->images;
    }
    if (s->chunkEvents) {
        for (cudaEvent_t ev : *s->chunkEvents) {
            cudaEventDestroy(ev);
        }
        delete s->chunkEvents;
    }
    delete s->tmpOff;
    freeCorpus(s->inlineCorpus);
    cudaFree(s->d_out);
    cudaFree(s->d_order);
    freeCorpus(s->rowsCorpus);
    cudaFree(s->d_rows);
    delete s->seg;
    cudaFree(s->d_counters);
    if (s->h_counters) cudaFreeHost(s->h_counters);
    if (s->h_stage) cudaFreeHost(s->h_stage);
    if (s->h_stage2) cudaFreeHost(s->h_stage2);
    if (s->evStage) cudaEventDestroy(s->evStage);
    if (s->evStage2) cudaEventDestroy(s->evStage2);
    if (s->evStart) cudaEventDestroy(s->evStart);
    if (s->evStop) cudaEventDestroy(s->evStop);
    if (s->evDone) cudaEventDestroy(s->evDone);
    if (s->stream) cudaStreamDestroy(s->stream);
    if (s->copyStream) cudaStreamDestroy(s->copyStream);
    g_scratch_free(s->alloc_base);
    return HS_SUCCESS;
}

/* ---- corpus handles ------------------------------------------------------------ */

static hs_error_t setBlocks(hs_b200_corpus *c, const u64 *packed, const unsigned *lengths,
                            size_t nblocks, u64 total, u64 payload, cudaStream_t stream,
                            u32 uniPitch = 0, u32 uniLen = 0) {
    c->nblocks = nblocks;
    c->bytes = total;
    c->payload = payload;
    c->h_len.assign(lengths, lengths + nblocks);
    if (uniPitch && uniLen) { /* layoutBlocks already proved uniformity: no tables */
        c->uniformPitch = uniPitch;
        c->uniformLen = uniLen;
        return HS_SUCCESS;
    }
    c->uniformPitch = detectPitch(packed, lengths, nblocks);
    c->uniformLen = 0;
    if (c->uniformPitch && nblocks) {
        u32 l0 = lengths[0];
        for (size_t i = 1; i < nblocks && l0; i++) {
            if (lengths[i] != l0) {
                l0 = 0;
            }
        }
        c->uniformLen = l0;
    }
    if (nblocks && !c->uniformLen) {
        CUDA_TRY(cudaMemcpyAsync(c->d_off, packed, nblocks * sizeof(u64), cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaMemcpyAsync(c->d_len, lengths, nblocks * sizeof(u32), cudaMemcpyHostToDevice, stream));
    }
    return HS_SUCCESS;
}

hs_error_t hs_b200_corpus_upload(const char *data, const unsigned long long *offsets,
                                 const unsigned int *lengths, size_t nblocks, int device,
                                 hs_b200_corpus_t **corpus) {
    if (!corpus || (nblocks && (!data || !offsets || !lengths)) || nblocks > 0xfffffff0u) {
        return HS_INVALID;
    }
    *corpus = nullptr;
    if (cudaSetDevice(device) != cudaSuccess) {
        return HS_ARCH_ERROR;
    }
    hs_b200_corpus *c = new (std::nothrow) hs_b200_corpus();
    if (!c) {
        return HS_NOMEM;
    }
    c->device = device;
    std::vector<u64> packed;
    u64 total = 0, payload = 0;
    bool direct = false;
    u32 uniPitch = 0, uniLen = 0;
    layoutBlocks(offsets, lengths, nblocks, &packed, &total, &payload, &direct, &uniPitch, &uniLen);
    hs_error_t r = reserveCorpus(c, total, nblocks);
    if (r != HS_SUCCESS) {
        freeCorpus(c);
        return r;
    }
    cudaError_t e = cudaSuccess;
    if (direct) {
        e = cudaMemcpy(c->d_data, data + offsets[0], total, cudaMemcpyHostToDevice);
    } else {
        /* pack through a host buffer in 64 MiB pieces */
        std::vector<u8> stage;
        const size_t CH = 64u << 20;
        size_t i = 0;
        while (i < nblocks && e == cudaSuccess) {
            const u64 start = packed[i];
            size_t j = i;
            while (j < nblocks && packed[j] + lengths[j] - start <= CH) {
                j++;
            }
            if (j == i) {
                j = i + 1;
            }
            const u64 end = packed[j - 1] + lengths[j - 1];
            stage.assign(end - start, 0);
            for (size_t k = i; k < j; k++) {
                memcpy(stage.data() + (packed[k] - start), data + offsets[k], lengths[k]);
            }
            e = cudaMemcpy(c->d_data + start, stage.data(), end - start, cudaMemcpyHostToDevice);
            i = j;
        }
    }
    if (e == cudaSuccess) {
        /* zero the tail so the last tile's look-ahead reads defined bytes */
        e = cudaMemset(c->d_data + total, 0, HSB_ROUNDUP(total, 16) + 32 - total);
    }
    c->readableEnd = HSB_ROUNDUP(total, 16) + 16;
    if (e == cudaSuccess) {
        r = setBlocks(c, packed.data(), lengths, nblocks, total, payload, 0, uniPitch, uniLen);
        c->maxLen = nblocks ? *std::max_element(lengths, lengths + nblocks) : 0;
        if (r == HS_SUCCESS && cudaDeviceSynchronize() != cudaSuccess) {
            r = HS_UNKNOWN_ERROR;
        }
    } else {
        r = HS_UNKNOWN_ERROR;
    }
    if (r != HS_SUCCESS) {
        freeCorpus(c);
        return r;
    }
    *corpus = c;
    return HS_SUCCESS;
}

hs_error_t hs_b200_corpus_wrap(const void *d_data, size_t data_bytes,
                               const unsigned long long *offsets, const unsigned int *lengths,
                               size_t nblocks, int device, hs_b200_corpus_t **corpus) {
    if (!corpus || !d_data || (uintptr_t)d_data % 16 || (nblocks && (!offsets || !lengths)) ||
        nblocks > 0xfffffff0u) {
        return HS_INVALID;
    }
    *corpus = nullptr;
    u64 prevEnd = 0, payload = 0;
    for (size_t i = 0; i < nblocks; i++) {
        if (offsets[i] % 16 || offsets[i] < prevEnd || offsets[i] + lengths[i] > data_bytes) {
            return HS_INVALID;
        }
        prevEnd = offsets[i] + lengths[i];
        payload += lengths[i];
    }
    if (cudaSetDevice(device) != cudaSuccess) {
        return HS_ARCH_ERROR;
    }
    hs_b200_corpus *c = new (std::nothrow) hs_b200_corpus();
    if (!c) {
        return HS_NOMEM;
    }
    c->device = device;
    hs_error_t r = HS_SUCCESS;
    if (nblocks) {
        cudaError_t e = cudaMalloc(&c->d_off, nblocks * sizeof(u64));
        if (e == cudaSuccess) e = cudaMalloc(&c->d_len, nblocks * sizeof(u32));
        if (e != cudaSuccess) {
            freeCorpus(c);
            return HS_NOMEM;
        }
        c->capBlocks = nblocks;
    }
    c->d_data = (u8 *)d_data;
    /* the caller's buffer must be readable up to data_bytes rounded up to 16 */
    c->readableEnd = HSB_ROUNDUP((u64)data_bytes, 16);
    std::vector<u64> off(offsets, offsets + nblocks);
    r = setBlocks(c, off.data(), lengths, nblocks, prevEnd, payload, 0);
    c->maxLen = nblocks ? *std::max_element(lengths, lengths + nblocks) : 0;
    if (r == HS_SUCCESS && cudaDeviceSynchronize() != cudaSuccess) {
        r = HS_UNKNOWN_ERROR;
    }
    if (r != HS_SUCCESS) {
        freeCorpus(c);
        return r;
    }
    *corpus = c;
    return HS_SUCCESS;
}

hs_error_t hs_b200_corpus_free(hs_b200_corpus_t *corpus) {
    freeCorpus(corpus);
    return HS_SUCCESS;
}

size_t hs_b200_corpus_bytes(const hs_b200_corpus_t *corpus) {
    return corpus ? (size_t)corpus->payload : 0;
}

/* ---- device-resident scan --------------------------------------------------------- */

static hs_error_t checkScanArgs(const hs_database_t *db, hs_scratch_t *scratch) {
    const hs_error_t r = checkDb(db, MODE_BLOCK);
    if (r != HS_SUCCESS) {
        return r;
    }
    return validScratch(scratch) ? HS_SUCCESS : HS_INVALID;
}

/* A pass over no bytes: no records, on the host and, for the stream-ordered readers of the ring, on the device */
static hs_error_t emptyPass(hs_scratch *s, cudaStream_t st) {
    s->h_counters[CTR_MATCHES] = 0;
    s->h_counters[CTR_ERROR] = 0;
    s->pending = false;
    s->lastCount = 0;
    s->streamEpoch = nullptr;
    return cudaMemsetAsync(s->d_counters, 0, CTR_COUNT * sizeof(u32), st) == cudaSuccess ? HS_SUCCESS
                                                                                          : HS_UNKNOWN_ERROR;
}

static hs_error_t corpusPass(const hs_database_t *db, const hs_b200_corpus_t *corpus, hs_scratch_t *scratch,
                             void *cuda_stream, int out, void *d_out, size_t words_per_block, void *d_status);

hs_error_t hs_b200_scan_corpus_async(const hs_database_t *db, const hs_b200_corpus_t *corpus,
                                     hs_scratch_t *scratch, void *cuda_stream) {
    return corpusPass(db, corpus, scratch, cuda_stream, OUT_RECORDS, nullptr, 0, nullptr);
}

hs_error_t hs_b200_scan_corpus_finish(hs_scratch_t *scratch, unsigned long long *nrecords,
                                      const void **d_records) {
    if (!validScratch(scratch)) {
        return HS_INVALID;
    }
    DeviceGuard guard(scratch->device);
    u32 count = scratch->lastCount;
    if (scratch->pending) {
        hs_error_t r = finishScan(scratch, &count);
        if (r != HS_SUCCESS) {
            return r;
        }
    }
    if (nrecords) {
        *nrecords = count;
    }
    if (d_records) {
        /* on overflow the ring is reallocated below: hand out no pointer */
        *d_records = count > scratch->outCap ? nullptr : scratch->d_out;
    }
    if (count > scratch->outCap) {
        /* ring overflowed: grow so that a re-run succeeds */
        hs_error_t r = growRingFor(scratch, count);
        if (r != HS_SUCCESS) {
            return r;
        }
        return HS_INSUFFICIENT_SPACE;
    }
    return HS_SUCCESS;
}

/* ---- fused exchange over NVLink peer memory ----------------------------------- */

hs_error_t hs_b200_peer_buffer_alloc(size_t bytes, void **d_ptr, unsigned char handle[64]) {
    if (!d_ptr || !handle || !bytes) {
        return HS_INVALID;
    }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
    void *p = nullptr;
    CUDA_TRY(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        return HS_UNKNOWN_ERROR;
    }
    memcpy(handle, &h, 64);
    *d_ptr = p;
    return HS_SUCCESS;
}

hs_error_t hs_b200_peer_buffer_open(const unsigned char handle[64], void **d_ptr) {
    if (!handle || !d_ptr) {
        return HS_INVALID;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void *p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        return HS_UNKNOWN_ERROR;
    }
    *d_ptr = p;
    return HS_SUCCESS;
}

hs_error_t hs_b200_peer_buffer_read(const void *d_ptr, void *host_dst, size_t bytes) {
    if (!d_ptr || !host_dst) {
        return HS_INVALID;
    }
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(host_dst, d_ptr, bytes, cudaMemcpyDeviceToHost));
    return HS_SUCCESS;
}

hs_error_t hs_b200_peer_buffer_close(void *d_ptr, int opened) {
    if (!d_ptr) {
        return HS_SUCCESS;
    }
    cudaError_t e = opened ? cudaIpcCloseMemHandle(d_ptr) : cudaFree(d_ptr);
    return e == cudaSuccess ? HS_SUCCESS : HS_UNKNOWN_ERROR;
}

hs_error_t hs_b200_set_peer_exchange(hs_scratch_t *scratch, unsigned int nranks, unsigned int my_rank,
                                     void *const *peer_bases, size_t cap_per_rank,
                                     unsigned int block_base) {
    if (!validScratch(scratch) || nranks > MAX_PEERS ||
        (nranks && (!peer_bases || my_rank >= nranks || cap_per_rank == 0 || cap_per_rank > 0xfffffff0u))) {
        return HS_INVALID;
    }
    scratch->nPeers = nranks;
    scratch->myRank = my_rank;
    scratch->peerCap = (u32)cap_per_rank;
    scratch->blockBase = block_base;
    for (unsigned r = 0; r < nranks; r++) {
        scratch->peers[r] = (DevMatch *)peer_bases[r];
    }
    return HS_SUCCESS;
}

hs_error_t hs_b200_export_records_async(hs_scratch_t *scratch, void *d_dst, size_t cap,
                                        void *d_count, void *cuda_stream) {
    if (!validScratch(scratch) || !d_dst || !d_count) {
        return HS_INVALID;
    }
    DeviceGuard guard(scratch->device);
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
    const size_t n = std::min<size_t>(cap, scratch->outCap);
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(d_dst, scratch->d_out, n * sizeof(DevMatch), cudaMemcpyDeviceToDevice, st));
    }
    CUDA_TRY(cudaMemcpyAsync(d_count, scratch->d_counters + CTR_MATCHES, sizeof(u32),
                             cudaMemcpyDeviceToDevice, st));
    return HS_SUCCESS;
}

hs_error_t hs_b200_copy_records(hs_scratch_t *scratch, void *d_dst, size_t cap) {
    if (!scratch || !d_dst || scratch->pending) {
        return HS_INVALID;
    }
    DeviceGuard guard(scratch->device);
    const size_t n = std::min<size_t>(cap, std::min<u32>(scratch->lastCount, scratch->outCap));
    if (n) {
        /* the records are final once evDone fired (finish waited for it); use
         * the copy stream so a scan queued behind on the scan stream is not
         * waited for */
        CUDA_TRY(cudaMemcpyAsync(d_dst, scratch->d_out, n * sizeof(DevMatch),
                                 cudaMemcpyDeviceToDevice, scratch->copyStream));
        CUDA_TRY(cudaStreamSynchronize(scratch->copyStream));
    }
    return HS_SUCCESS;
}

hs_error_t hs_b200_fetch_matches(const hs_database_t *db, hs_scratch_t *scratch,
                                 hs_b200_match_t *out, size_t cap,
                                 unsigned long long *nmatches) {
    if (!scratch || !db || scratch->pending) {
        return HS_INVALID;
    }
    DeviceGuard guard(scratch->device);
    DevImage *im = nullptr;
    hs_error_t r = findImage(scratch, db, &im);
    if (r != HS_SUCCESS) {
        return r;
    }
    const u32 n = std::min(scratch->lastCount, scratch->outCap);
    std::vector<DevMatch> tmp(n);
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(tmp.data(), scratch->d_out, (size_t)n * sizeof(DevMatch),
                                 cudaMemcpyDeviceToHost, scratch->copyStream));
        CUDA_TRY(cudaStreamSynchronize(scratch->copyStream));
    }
    if (im->rules.comb.any()) {
        /* the combinations are evaluated per block, over the blocks of the corpus last scanned */
        const hs_b200_corpus *c = scratch->lastCorpus;
        r = c ? im->rules.deliver(&tmp, c->h_len.data(), c->h_len.size()) : HS_INVALID;
    } else {
        r = im->rules.deliver(&tmp, nullptr, 0);
    }
    if (r != HS_SUCCESS) {
        return r;
    }
    const size_t m = tmp.size();
    if (nmatches) {
        *nmatches = m;
    }
    if (out) {
        if (cap < m) {
            return HS_INSUFFICIENT_SPACE;
        }
        memcpy(out, tmp.data(), m * sizeof(DevMatch));
    }
    return HS_SUCCESS;
}

/* ---- the report rules on the device ---------------------------------------------------------
 *
 * ReportRules::deliver as kernels (order_kernels.h), enqueued behind the scan on its stream: the
 * delivered matches stay in device memory and the host never waits. */

static u32 bitWidth(u64 v) {
    u32 b = 0;
    for (; v; v >>= 1) {
        b++;
    }
    return b;
}

/* the image of `db` the scratch already holds (an order entry builds none: the scan built it) */
static DevImage *heldImage(hs_scratch *s, const hs_database_t *db) {
    const DbHeader *h = (const DbHeader *)db;
    for (DevImage *im : *s->images) {
        if (im->db == db && im->crc == h->crc32 && im->length == h->length) {
            return im;
        }
    }
    return nullptr;
}

static hs_error_t checkOrderArgs(const hs_database_t *db, hs_scratch_t *scratch, void *d_out, size_t cap,
                                 void *d_count, DevImage **im, u32 mode = MODE_BLOCK) {
    if (!db || !scratch || !d_count || (cap && !d_out)) {
        return HS_INVALID;
    }
    hs_error_t r = checkDb(db, mode);
    if (r != HS_SUCCESS) {
        return r;
    }
    if (!validScratch(scratch)) {
        return HS_INVALID;
    }
    if (dbRose(db)->ckeyCount) {
        return HS_INVALID; /* combination reports are evaluated per block on the host */
    }
    *im = heldImage(scratch, db);
    if (!*im) {
        return HS_INVALID;
    }
    return (*im)->orderStatus;
}

/* Enqueue the ordering of the records at `in` -- the record ring (ringCount = its count on the device,
 * inCap = its capacity) or n records -- into d_out[0, cap) and *d_count on `st`, with the temporaries
 * in the scratch: tile sums and digit histograms, two record buffers for the resolved records (each
 * input record becomes at most maxFanout), and for exhaustible ids a hash table of twice as many slots. */
static hs_error_t enqueueOrder(hs_scratch *s, const DevImage *im, const DevMatch *in, const u32 *ringCount, u32 inCap,
                               u32 inN, void *d_out, size_t cap, void *d_count, u32 maxPasses, cudaStream_t st) {
    const u64 n = ringCount ? inCap : inN;
    const u64 m = n * im->maxFanout;
    if (m >= 0xfffff000ull) {
        return HS_NOMEM; /* positions are 32-bit */
    }
    OrderParams p = im->orderTables;
    const u64 tiles = (std::max(n, m) + ORDER_TILE - 1) / ORDER_TILE;
    u64 slots = 0;
    if (p.anyEx && m) {
        for (slots = 2; slots < 2 * m; slots <<= 1) {
        }
        if (slots > 0x80000000ull) {
            return HS_NOMEM;
        }
    }
    size_t at = 0;
    auto carve = [&](size_t bytes) {
        const size_t o = at;
        at = HSB_ROUNDUP(at + bytes, 256);
        return o;
    };
    const size_t oSt = carve(sizeof(OrderState)), oTile = carve((tiles + 1) * 4), oHist = carve(256 * (tiles + 1) * 4),
                 oBin = carve(ORDER_MAX_PASSES * 256 * 4), oBuf0 = carve(m * sizeof(DevMatch)),
                 oBuf1 = carve(m * sizeof(DevMatch)), oKey = carve(slots * 8), oFirst = carve(slots * 4);
    if (at > s->orderBytes) {
        cudaFree(s->d_order); /* (synchronises with any ordering still using it) */
        s->d_order = nullptr;
        s->orderBytes = 0;
        CUDA_TRY(cudaMalloc(&s->d_order, at));
        s->orderBytes = at;
    }
    u8 *b = s->d_order;
    p.in = in;
    p.inCount = ringCount;
    p.inCap = inCap;
    p.inN = inN;
    p.st = (OrderState *)(b + oSt);
    p.buf[0] = (DevMatch *)(b + oBuf0);
    p.buf[1] = (DevMatch *)(b + oBuf1);
    p.bufCap = (u32)m;
    p.tileSum = (u32 *)(b + oTile);
    p.hist = (u32 *)(b + oHist);
    p.tileCap = (u32)tiles + 1;
    p.binTotal = (u32 *)(b + oBin);
    p.exKey = (u64 *)(b + oKey);
    p.exFirst = (u32 *)(b + oFirst);
    p.exSlots = (u32)slots;
    p.anyEx = slots != 0;
    p.out = (DevMatch *)d_out;
    p.outCap = cap;
    p.count = (unsigned long long *)d_count;
    if (slots) {
        CUDA_TRY(cudaMemsetAsync(b + oKey, 0xff, oFirst + slots * 4 - oKey, st));
    }
    unsigned launched = 0;
    const cudaError_t e = launchOrder(p, maxPasses, st, &launched);
    g_launches += launched;
    return e == cudaSuccess ? HS_SUCCESS : HS_UNKNOWN_ERROR;
}

hs_error_t hs_b200_order_matches_async(const hs_database_t *db, hs_scratch_t *scratch, void *d_out, size_t cap,
                                       void *d_count, void *cuda_stream) {
    DevImage *im = nullptr;
    /* the last scan a stream-set pass: its records are a stream database's */
    const bool streamPass = validScratch(scratch) && scratch->streamEpoch;
    hs_error_t r = checkOrderArgs(db, scratch, d_out, cap, d_count, &im, streamPass ? MODE_STREAM : MODE_BLOCK);
    if (r != HS_SUCCESS) {
        return r;
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(scratch->device);
    /* the key needs no more bits than the last scan's block count, its longest block and the id table; a
     * stream pass's `to` is a stream offset, which only the device knows (up to 64 bits: the device decides
     * the passes) */
    const u32 keyBits = bitWidth(im->orderTables.nIds ? im->orderTables.nIds - 1 : 0) +
                        (streamPass ? 64 : bitWidth(scratch->lastMaxLen + (u64)std::max(0, im->maxAdjust))) +
                        bitWidth(scratch->lastBlocks ? scratch->lastBlocks - 1 : 0);
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
    r = enqueueOrder(scratch, im, scratch->d_out, scratch->d_counters + CTR_MATCHES, scratch->outCap, 0, d_out, cap,
                     d_count, (keyBits + 7) / 8, st);
    unmarkInUse(scratch);
    return r;
}

hs_error_t hs_b200_order_records_async(const hs_database_t *db, hs_scratch_t *scratch, const void *d_recs, size_t n,
                                       void *d_out, size_t cap, void *d_count, void *cuda_stream) {
    DevImage *im = nullptr;
    hs_error_t r = checkOrderArgs(db, scratch, d_out, cap, d_count, &im);
    if (r != HS_SUCCESS) {
        return r;
    }
    if ((n && !d_recs) || n > 0xfffffff0u) {
        return HS_INVALID;
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(scratch->device);
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
    r = enqueueOrder(scratch, im, (const DevMatch *)d_recs, nullptr, 0, (u32)n, d_out, cap, d_count,
                     ORDER_MAX_PASSES, st);
    unmarkInUse(scratch);
    return r;
}

/* ---- row scans: a column of rows in device memory -------------------------------------------------------------- */

/* The staging corpus of a row scan (`bound` bytes packed, nrows blocks) and `need` bytes of temporaries for its
 * plan */
static hs_error_t reserveRows(hs_scratch *s, u64 bound, size_t nrows, size_t need) {
    if (!s->rowsCorpus) {
        s->rowsCorpus = new (std::nothrow) hs_b200_corpus();
        if (!s->rowsCorpus) {
            return HS_NOMEM;
        }
        s->rowsCorpus->device = s->device;
        s->rowsCorpus->deviceTables = true;
    }
    const u8 *before = s->rowsCorpus->d_alloc;
    hs_error_t r = reserveCorpus(s->rowsCorpus, bound, nrows);
    if (r != HS_SUCCESS) {
        return r;
    }
    if (s->rowsCorpus->d_alloc != before) {
        /* the front pad of a new allocation is zeroed on the legacy stream: done before any pass reads it */
        CUDA_TRY(cudaDeviceSynchronize());
    }
    if (need > s->rowsBytes) {
        cudaFree(s->d_rows); /* (synchronises with any pass still using it) */
        s->d_rows = nullptr;
        s->rowsBytes = 0;
        CUDA_TRY(cudaMalloc(&s->d_rows, need + need / 8));
        s->rowsBytes = need + need / 8;
    }
    return HS_SUCCESS;
}

/* The checks of a mask pass (out = OUT_MASK) or a first-match pass (OUT_FIRST) over nblocks blocks (after those of
 * its ordinary form), and its MaskOut: the caller's buffer (NULL only without blocks, as an empty torch tensor's;
 * words_per_block 32-bit words per block for a mask, one 8-byte entry for a first-match table) and the image's
 * tables, uploaded with it (uploadOrderTables). */
static hs_error_t maskArgs(const DevImage *im, int out, size_t nblocks, void *d_out, size_t words_per_block,
                           void *d_status, MaskOut *m) {
    if (im->orderStatus != HS_SUCCESS) {
        return im->orderStatus; /* an engine program the tables cannot hold */
    }
    const OrderParams &t = im->orderTables;
    const bool first = out == OUT_FIRST;
    if ((!d_out && nblocks) || (uintptr_t)d_out % (first ? 8 : 4) || (uintptr_t)d_status % 4 ||
        (!first && (words_per_block < (t.nIds + 31) / 32 || words_per_block > 0xffffffffu))) {
        return HS_INVALID;
    }
    m->bits = first ? nullptr : (u32 *)d_out;
    m->first = first ? (unsigned long long *)d_out : nullptr;
    m->slack = (u32)-im->rules.minAdjust;
    m->words = first ? 0 : (u32)words_per_block;
    m->nIds = t.nIds;
    m->ids = t.ids;
    m->progOff = t.progOff;
    m->progStart = t.progStart;
    m->reps = t.reps;
    m->nProg = t.nProg;
    m->rows = StreamRowsMap(); /* (a stream-set pass over rows sets it) */
    return HS_SUCCESS;
}

/* A mask or first-match pass over no bytes: no records, every word of the mask zero (every entry of the table all
 * ones), status 0 */
static hs_error_t emptyMaskPass(hs_scratch *s, cudaStream_t st, const MaskOut &m, size_t nblocks, u32 *status) {
    hs_error_t r = emptyPass(s, st);
    if (r == HS_SUCCESS && (clearOutput(m, nblocks, s->smCount, st) != cudaSuccess ||
                            (status && launchMaskStatus(s->d_counters, s->outCap, status, st) != cudaSuccess))) {
        r = HS_UNKNOWN_ERROR;
    }
    return r;
}

/* hs_b200_scan_corpus_mask_async / hs_b200_scan_rows_mask_async (out = OUT_MASK), their first-match forms
 * (OUT_FIRST, words_per_block unused) or their ordinary forms (OUT_RECORDS) */
static hs_error_t corpusPass(const hs_database_t *db, const hs_b200_corpus_t *corpus, hs_scratch_t *scratch,
                             void *cuda_stream, int out, void *d_out, size_t words_per_block, void *d_status) {
    if (!scratch || !corpus) {
        return HS_INVALID;
    }
    hs_error_t r = checkScanArgs(db, scratch);
    if (r != HS_SUCCESS) {
        return r;
    }
    MaskOut m;
    DevImage *im = nullptr;
    const bool mask = out != OUT_RECORDS;
    if (mask) {
        if (dbRose(db)->ckeyCount) {
            return HS_INVALID; /* a combination's reports depend on the order within a block */
        }
        im = heldImage(scratch, db);
        if (!im) {
            return HS_INVALID;
        }
        if (scratch->nPeers) {
            return HS_ARCH_ERROR;
        }
        r = maskArgs(im, out, corpus->nblocks, d_out, words_per_block, d_status, &m);
        if (r != HS_SUCCESS) {
            return r;
        }
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(scratch->device);
    r = mask ? HS_SUCCESS : findImage(scratch, db, &im);
    if (r == HS_SUCCESS) {
        cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
        if (corpus->bytes == 0 || corpus->nblocks == 0) {
            r = mask ? emptyMaskPass(scratch, st, m, corpus->nblocks, (u32 *)d_status) : emptyPass(scratch, st);
        } else {
            r = enqueueScan(scratch, im, corpus, st, nullptr, nullptr, nullptr, mask ? &m : nullptr, (u32 *)d_status);
        }
        scratch->lastCorpus = corpus;
        scratch->lastBlocks = corpus->nblocks;
        scratch->lastMaxLen = corpus->maxLen;
    }
    unmarkInUse(scratch);
    return r;
}

static hs_error_t rowsPass(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                           const unsigned long long *d_offsets, size_t nrows, hs_scratch_t *scratch, void *cuda_stream,
                           int out, void *d_out, size_t words_per_block, void *d_status) {
    if (!db || !scratch || !d_offsets || (uintptr_t)d_offsets % 8 || (!d_chars && chars_bytes) ||
        nrows > 0xfffffff0u) {
        return HS_INVALID;
    }
    hs_error_t r = checkScanArgs(db, scratch);
    if (r != HS_SUCCESS) {
        return r;
    }
    if (dbRose(db)->ckeyCount) {
        return HS_INVALID; /* combination reports are evaluated per block on the host, from the block lengths */
    }
    DevImage *im = heldImage(scratch, db);
    if (!im) {
        return HS_INVALID;
    }
    if (scratch->nPeers) {
        return HS_ARCH_ERROR;
    }
    MaskOut m;
    const bool mask = out != OUT_RECORDS;
    if (mask) {
        r = maskArgs(im, out, nrows, d_out, words_per_block, d_status, &m);
        if (r != HS_SUCCESS) {
            return r;
        }
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(scratch->device);
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
    /* the packed rows take at most their bytes plus 16 per row (a row's pad, or an empty row's 16 bytes) */
    const u64 bound = (u64)chars_bytes + 16 * (u64)nrows;
    if (nrows == 0) {
        r = mask ? emptyMaskPass(scratch, st, m, 0, (u32 *)d_status) : emptyPass(scratch, st);
    } else {
        const size_t ntiles = (nrows + ROWS_TILE - 1) / ROWS_TILE;
        r = reserveRows(scratch, bound, nrows, 256 + HSB_ROUNDUP(ntiles * sizeof(u64), 256) + ntiles * sizeof(u32));
    }
    hs_b200_corpus *c = scratch->rowsCorpus;
    if (r == HS_SUCCESS && nrows) {
        c->nblocks = nrows;
        c->bytes = bound;
        c->readableEnd = HSB_ROUNDUP(bound, 16) + 16;
        c->payload = chars_bytes;
        c->uniformPitch = 0;
        c->uniformLen = 0;
        RowsParams rp;
        rp.chars = (const u8 *)d_chars;
        rp.charsBytes = chars_bytes;
        rp.offsets = (const u64 *)d_offsets;
        rp.nrows = (u32)nrows;
        rp.corpus = c->d_data;
        rp.zeroEnd = HSB_ROUNDUP(bound, 16) + 32;
        rp.blockOff = c->d_off;
        rp.blockLen = c->d_len;
        rp.bad = reinterpret_cast<u32 *>(scratch->d_rows);
        rp.tilePad = reinterpret_cast<u64 *>(scratch->d_rows + 256);
        rp.tileBad = reinterpret_cast<u32 *>(scratch->d_rows + 256 +
                                             HSB_ROUNDUP((nrows + ROWS_TILE - 1) / ROWS_TILE * sizeof(u64), 256));
        rp.counters = scratch->d_counters;
        rp.outCap = scratch->outCap;
        r = enqueueScan(scratch, im, c, st, nullptr, nullptr, &rp, mask ? &m : nullptr, (u32 *)d_status);
    }
    scratch->lastCorpus = c;
    scratch->lastBlocks = nrows;
    scratch->lastMaxLen = chars_bytes; /* no row is longer; the device decides the radix passes the records need */
    unmarkInUse(scratch);
    return r;
}

hs_error_t hs_b200_scan_rows_async(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                                   const unsigned long long *d_offsets, size_t nrows, hs_scratch_t *scratch,
                                   void *cuda_stream) {
    return rowsPass(db, d_chars, chars_bytes, d_offsets, nrows, scratch, cuda_stream, OUT_RECORDS, nullptr, 0,
                    nullptr);
}

hs_error_t hs_b200_scan_corpus_mask_async(const hs_database_t *db, const hs_b200_corpus_t *corpus,
                                          hs_scratch_t *scratch, void *d_mask, size_t words_per_block,
                                          void *d_status, void *cuda_stream) {
    return corpusPass(db, corpus, scratch, cuda_stream, OUT_MASK, d_mask, words_per_block, d_status);
}

hs_error_t hs_b200_scan_rows_mask_async(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                                        const unsigned long long *d_offsets, size_t nrows, hs_scratch_t *scratch,
                                        void *d_mask, size_t words_per_block, void *d_status, void *cuda_stream) {
    return rowsPass(db, d_chars, chars_bytes, d_offsets, nrows, scratch, cuda_stream, OUT_MASK, d_mask, words_per_block,
                    d_status);
}

hs_error_t hs_b200_scan_corpus_first_async(const hs_database_t *db, const hs_b200_corpus_t *corpus,
                                           hs_scratch_t *scratch, void *d_first, void *d_status, void *cuda_stream) {
    return corpusPass(db, corpus, scratch, cuda_stream, OUT_FIRST, d_first, 0, d_status);
}

hs_error_t hs_b200_scan_rows_first_async(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                                         const unsigned long long *d_offsets, size_t nrows, hs_scratch_t *scratch,
                                         void *d_first, void *d_status, void *cuda_stream) {
    return rowsPass(db, d_chars, chars_bytes, d_offsets, nrows, scratch, cuda_stream, OUT_FIRST, d_first, 0, d_status);
}

/* ---- DFA engines in block mode ------------------------------------------------------
 *
 * nfaExecMcClellan8_B / nfaExecMcClellan16_B / nfaExecSheng_B (src/nfa/mcclellan.c:
 * 937-973, src/nfa/sheng.c:706-739) over every block of a resident corpus, offset 0
 * per block.  The callbacks the reference would fire (report, end offset) come back
 * as records {report, block, to}, ordered by (block, to, report). */
hs_error_t hs_b200_nfa_scan_corpus(const void *nfa, size_t nfa_len, const hs_b200_corpus_t *corpus,
                                   hs_b200_match_t *out, size_t cap, unsigned long long *nmatches,
                                   float *kernel_ms) {
    if (!corpus || (cap && !out) || !nmatches) {
        return HS_INVALID;
    }
    DfaParams p;
    {
        const hs_error_t er = engineParams(nfa, nfa_len, &p); /* HS_INVALID for a short or damaged engine */
        if (er != HS_SUCCESS) {
            return er;
        }
    }
    DeviceGuard guard(corpus->device);
    int smCount = 0, maxSmem = 0;
    cudaDeviceGetAttribute(&smCount, cudaDevAttrMultiProcessorCount, corpus->device);
    cudaDeviceGetAttribute(&maxSmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, corpus->device);
    u8 *d_nfa = nullptr;
    u32 *d_ctr = nullptr;
    DevMatch *d_out = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    SegArea seg;
    hs_error_t rv = HS_SUCCESS;
    u32 capDev = (u32)std::min<size_t>(std::max<size_t>(cap, 1u << 16), 0xfffffff0u);
    std::vector<DevMatch> host;
    cudaError_t e = cudaMalloc(&d_nfa, HSB_ROUNDUP(nfa_len, 16));
    if (e == cudaSuccess) e = cudaMemcpy(d_nfa, nfa, nfa_len, cudaMemcpyHostToDevice);
    p.nfa = d_nfa;
    if (e == cudaSuccess) e = cudaMalloc(&d_ctr, CTR_COUNT * sizeof(u32));
    if (e == cudaSuccess) e = cudaEventCreate(&ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&ev1);
    for (int attempt = 0; e == cudaSuccess && attempt < 3; attempt++) {
        e = cudaMalloc(&d_out, (size_t)capDev * sizeof(DevMatch));
        if (e != cudaSuccess) break;
        e = cudaMemset(d_ctr, 0, CTR_COUNT * sizeof(u32));
        if (e == cudaSuccess) e = cudaEventRecord(ev0, 0);
        if (e == cudaSuccess) e = launchEngine(p, corpus, d_out, capDev, d_ctr, smCount, maxSmem, &seg, 0);
        if (e == cudaSuccess) e = cudaEventRecord(ev1, 0);
        u32 ctr[CTR_COUNT] = {0};
        if (e == cudaSuccess) e = cudaMemcpy(ctr, d_ctr, sizeof(ctr), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) break;
        if (ctr[CTR_MATCHES] > capDev) { /* grow and run again */
            cudaFree(d_out);
            d_out = nullptr;
            capDev = ctr[CTR_MATCHES] + ctr[CTR_MATCHES] / 8 + 1024;
            continue;
        }
        host.resize(ctr[CTR_MATCHES]); /* reserved slots: the lanes' unused ones carry id 0xffffffff */
        if (!host.empty()) {
            e = cudaMemcpy(host.data(), d_out, host.size() * sizeof(DevMatch), cudaMemcpyDeviceToHost);
        }
        host.erase(std::remove_if(host.begin(), host.end(), [](const DevMatch &m) { return m.id == 0xffffffffu; }),
                   host.end());
        if (kernel_ms && e == cudaSuccess) {
            cudaEventElapsedTime(kernel_ms, ev0, ev1);
        }
        break;
    }
    if (e != cudaSuccess) {
        rv = e == cudaErrorMemoryAllocation ? HS_NOMEM : HS_UNKNOWN_ERROR;
    } else {
        std::sort(host.begin(), host.end(), RecordOrder());
        *nmatches = host.size();
        memcpy(out, host.data(), std::min(cap, host.size()) * sizeof(DevMatch));
        if (host.size() > cap) {
            rv = HS_INSUFFICIENT_SPACE;
        }
    }
    cudaFree(d_nfa);
    cudaFree(d_ctr);
    cudaFree(d_out);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    return rv;
}

/* ---- host-buffer scans -------------------------------------------------------------- */

/* Copy host blocks into the scratch's inline corpus and scan them, with the
 * host->device copy pipelined against the kernel in chunk_mb pieces. */
static hs_error_t scanHostBlocks(DevImage *im, hs_scratch *s, const char *data,
                                 const unsigned long long *offsets, const unsigned *lengths,
                                 size_t nblocks, std::vector<DevMatch> *matches,
                                 bool countOnly = false) {
    static const bool trace = getenv("HSB200_TRACE") != nullptr;
    DeviceGuard guard(s->device); /* every host-buffer scan (hs_scan, hs_b200_scan_blocks, streams) ends up here */
    const double t0 = nowMs();
    hs_b200_corpus *c = s->inlineCorpus;
    std::vector<u64> &packed = *s->tmpOff;
    u64 total = 0, payload = 0;
    bool direct = false;
    u32 uniPitch = 0, uniLen = 0;
    layoutBlocks(offsets, lengths, nblocks, &packed, &total, &payload, &direct, &uniPitch, &uniLen);
    matches->clear();
    if (total == 0) {
        return HS_SUCCESS;
    }
    const double tLayout = nowMs();
    hs_error_t r = reserveCorpus(c, total, nblocks);
    if (r != HS_SUCCESS) {
        return r;
    }
    c->readableEnd = HSB_ROUNDUP(total, 16) + 16;
    r = setBlocks(c, packed.data(), lengths, nblocks, total, payload, s->copyStream, uniPitch, uniLen);
    if (r != HS_SUCCESS) {
        return r;
    }
    const u64 chunk = (u64)std::max(1, g_opts.chunkMB) << 20;
    const size_t nchunks = (size_t)((total + chunk - 1) / chunk);
    while (s->chunkEvents->size() < nchunks + 1) {
        cudaEvent_t ev;
        CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        s->chunkEvents->push_back(ev);
    }
    /* zero the look-ahead bytes after the corpus */
    CUDA_TRY(cudaMemsetAsync(c->d_data + total, 0, HSB_ROUNDUP(total, 16) + 32 - total, s->copyStream));
    size_t blk = 0; /* first block of the next chunk (packed layout) */
    Upload up;
    up.nchunks = nchunks;
    up.chunk = [&](size_t ci, u64 *covered) -> hs_error_t {
        const u64 from = ci * chunk, to = std::min<u64>(total, from + chunk);
        /* packed layout: blocks that straddle the chunk edge go whole with the chunk they start in */
        const size_t b0 = blk;
        u64 end = from;
        while (!direct && blk < nblocks && packed[blk] < to) {
            end = std::max<u64>(end, packed[blk] + lengths[blk]);
            blk++;
        }
        *covered = std::min(direct ? to : (blk < nblocks ? packed[blk] : total), to);
        if (direct) {
            CUDA_TRY(cudaMemcpyAsync(c->d_data + from, data + offsets[0] + from, to - from,
                                     cudaMemcpyHostToDevice, s->copyStream));
        } else if (blk > b0) {
            /* unaligned host layout: pack this chunk's blocks (16-byte aligned starts,
             * zero gaps) into a pinned staging buffer and send it as one copy.  Two
             * buffers alternate. */
            const u64 start = packed[b0];
            const size_t need = (size_t)(end - start);
            u8 *&stage = (ci & 1) ? s->h_stage2 : s->h_stage;
            size_t &cap = (ci & 1) ? s->h_stage2Cap : s->h_stageCap;
            cudaEvent_t ev = (ci & 1) ? s->evStage2 : s->evStage;
            CUDA_TRY(cudaEventSynchronize(ev)); /* previous use of this buffer has been sent */
            if (need > cap) {
                if (stage) cudaFreeHost(stage);
                stage = nullptr;
                cap = 0;
                CUDA_TRY(cudaMallocHost(&stage, need + need / 4 + 4096));
                cap = need + need / 4 + 4096;
            }
            memset(stage, 0, need);
            for (size_t k = b0; k < blk; k++) {
                memcpy(stage + (packed[k] - start), data + offsets[k], lengths[k]);
            }
            CUDA_TRY(cudaMemcpyAsync(c->d_data + start, stage, need, cudaMemcpyHostToDevice, s->copyStream));
            CUDA_TRY(cudaEventRecord(ev, s->copyStream));
        }
        CUDA_TRY(cudaEventRecord((*s->chunkEvents)[ci], s->copyStream));
        CUDA_TRY(cudaStreamWaitEvent(s->stream, (*s->chunkEvents)[ci], 0));
        return HS_SUCCESS;
    };
    /* nobody will look at the order: when no report rule applies, the raw count IS the delivered count */
    const bool plain = countOnly && im->rules.rawCountDelivered();
    ScanTimes tm;
    r = scanRecords(s, im, c, &up, !plain, matches, &tm, lengths);
    if (r == HS_SUCCESS && trace) {
        fprintf(stderr, "[hs_b200 trace] host scan: layout %.3f ms, enqueue %.3f, wait %.3f, records %.3f, "
                        "postprocess %.3f (total %.3f, %zu chunks)\n",
                tLayout - t0, tm.enqueued - tLayout, tm.waited - tm.enqueued, tm.read - tm.waited,
                nowMs() - tm.read, nowMs() - t0, nchunks);
    }
    return r;
}

/* hs_scan, hs_b200_scan_blocks and _collect: check the database and the scratch,
 * mark the scratch in use, scan the blocks and hand the records to deliver() before
 * the mark is released.  skipShort (hs_scan): a block shorter than any match is not
 * scanned at all (src/runtime.c:346-350). */
static hs_error_t blockScan(const hs_database_t *db, hs_scratch *s, const char *data,
                            const unsigned long long *offsets, const unsigned *lengths, size_t nblocks,
                            bool countOnly, bool skipShort,
                            const std::function<hs_error_t(const std::vector<DevMatch> &)> &deliver) {
    hs_error_t r = checkScanArgs(db, s);
    if (r != HS_SUCCESS) {
        return r;
    }
    if (markInUse(s)) {
        return HS_SCRATCH_IN_USE;
    }
    if (!(skipShort && dbRose(db)->minWidth > lengths[0])) {
        DevImage *im = nullptr;
        std::vector<DevMatch> matches;
        r = findImage(s, db, &im);
        if (r == HS_SUCCESS) {
            r = scanHostBlocks(im, s, data, offsets, lengths, nblocks, &matches, countOnly);
        }
        if (r == HS_SUCCESS) {
            r = deliver(matches);
        }
    }
    unmarkInUse(s);
    return r;
}

hs_error_t hs_b200_scan_blocks(const hs_database_t *db, const char *data,
                               const unsigned long long *offsets, const unsigned int *lengths,
                               size_t nblocks, hs_scratch_t *scratch,
                               hs_b200_block_event_handler onEvent, void *context,
                               unsigned long long *nmatches) {
    if (!scratch || (nblocks && (!data || !offsets || !lengths)) || nblocks > 0xfffffff0u) {
        return HS_INVALID;
    }
    return blockScan(db, scratch, data, offsets, lengths, nblocks, onEvent == nullptr, false,
                     [&](const std::vector<DevMatch> &matches) {
                         unsigned long long delivered = 0;
                         if (!onEvent) {
                             delivered = matches.size();
                         } else {
                             u32 stopped = 0xffffffffu;
                             for (const DevMatch &m : matches) {
                                 if (m.block == stopped) {
                                     continue;
                                 }
                                 delivered++;
                                 if (onEvent(m.block, m.id, 0, m.to, 0, context)) {
                                     stopped = m.block;
                                 }
                             }
                         }
                         if (nmatches) {
                             *nmatches = delivered;
                         }
                         return HS_SUCCESS;
                     });
}

hs_error_t hs_b200_scan_blocks_collect(const hs_database_t *db, const char *data,
                                       const unsigned long long *offsets, const unsigned int *lengths,
                                       size_t nblocks, hs_scratch_t *scratch, hs_b200_match_t *out,
                                       size_t cap, unsigned long long *nmatches) {
    if (!scratch || (nblocks && (!data || !offsets || !lengths)) || nblocks > 0xfffffff0u || (cap && !out)) {
        return HS_INVALID;
    }
    return blockScan(db, scratch, data, offsets, lengths, nblocks, false, false,
                     [&](const std::vector<DevMatch> &matches) {
                         if (nmatches) {
                             *nmatches = matches.size();
                         }
                         memcpy(out, matches.data(), std::min(cap, matches.size()) * sizeof(DevMatch));
                         return matches.size() > cap ? HS_INSUFFICIENT_SPACE : HS_SUCCESS;
                     });
}

hs_error_t hs_scan(const hs_database_t *db, const char *data, unsigned int length,
                   unsigned int flags, hs_scratch_t *scratch, match_event_handler onEvent,
                   void *context) {
    (void)flags;
    if (!scratch || !data) {
        return HS_INVALID;
    }
    const unsigned long long off = 0;
    return blockScan(db, scratch, data, &off, &length, 1, false, true, [&](const std::vector<DevMatch> &matches) {
        for (const DevMatch &m : matches) {
            if (onEvent && onEvent(m.id, 0, m.to, 0, context)) {
                return HS_SCAN_TERMINATED; /* src/report.h:324-328 */
            }
        }
        return HS_SUCCESS;
    });
}

/* ---- streaming mode (src/runtime.c:542-977, pure-literal databases) ------------------
 *
 * A stream carries the last historyRequired (<= 7) bytes it has seen, its
 * offset, a broken/exhausted status and the single-match reports already
 * raised.  hs_scan_stream scans (history ++ write) as one block on the device
 * and delivers the matches that END inside the write, at stream offsets --
 * the restatement of pureLiteralStreamExec / hwlmExecStreaming
 * (src/runtime.c:801-829, src/hwlm/hwlm.c:201-239) with the look-behind made
 * explicit. */

struct hs_stream {
    u32 magic;
    const hs_database_t *db;
    u64 offset;
    u32 hreq, hlen;
    u8 hist[16];
    u8 status; /* 1 = terminated by the callback, 2 = all reports exhausted */
    std::unordered_set<u32> *seen;
};

static const u32 STREAM_MAGIC = 0x4d525453; /* "STRM" */

static bool validStream(const hs_stream *st) { return st && st->magic == STREAM_MAGIC && st->seen; }

static void resetStreamState(hs_stream *st) {
    st->offset = 0;
    st->hlen = 0;
    st->status = 0;
    st->seen->clear();
}

hs_error_t hs_open_stream(const hs_database_t *db, unsigned int flags, hs_stream_t **stream) {
    (void)flags;
    if (!stream) {
        return HS_INVALID;
    }
    *stream = nullptr;
    hs_error_t err = checkDb(db, MODE_STREAM);
    if (err != HS_SUCCESS) {
        return err;
    }
    const RoseEngine *rose = dbRose(db);
    if (rose->runtimeImpl != RUNTIME_PURE_LITERAL || rose->historyRequired > sizeof(((hs_stream *)0)->hist)) {
        return HS_ARCH_ERROR;
    }
    hs_stream *st = (hs_stream *)g_stream_alloc(sizeof(hs_stream));
    err = checkAlloc(st);
    if (err != HS_SUCCESS) {
        g_stream_free(st);
        return err;
    }
    memset(st, 0, sizeof(*st));
    st->magic = STREAM_MAGIC;
    st->db = db;
    st->hreq = rose->historyRequired;
    st->seen = new (std::nothrow) std::unordered_set<u32>();
    if (!st->seen) {
        g_stream_free(st);
        return HS_NOMEM;
    }
    *stream = st;
    return HS_SUCCESS;
}

/* One write of one stream (hs_scan_stream_internal, src/runtime.c:870-977):
 * scan look-behind ++ write as a block, deliver the matches that end inside the
 * write at stream offsets, roll the history forward.  The scratch is already
 * marked in use by the caller. */
static hs_error_t streamWrite(hs_stream *st, const char *data, unsigned int length, hs_scratch_t *scratch,
                              match_event_handler onEvent, void *context) {
    hs_error_t r = HS_SUCCESS;
    if (st->status & 1) {
        r = HS_SCAN_TERMINATED; /* the stream is broken: src/runtime.c:883-893 */
    } else if (!(st->status & 2) && length != 0) {
        DevImage *im = nullptr;
        r = findImage(scratch, st->db, &im);
        std::vector<DevMatch> matches;
        std::vector<char> buf;
        if (r == HS_SUCCESS) {
            buf.resize((size_t)st->hlen + length);
            memcpy(buf.data(), st->hist, st->hlen);
            memcpy(buf.data() + st->hlen, data, length);
            const unsigned long long off = 0;
            const unsigned total = (unsigned)buf.size();
            r = scanHostBlocks(im, scratch, buf.data(), &off, &total, 1, &matches);
        }
        if (r == HS_SUCCESS) {
            const RoseEngine *rose = dbRose(st->db);
            for (const DevMatch &m : matches) {
                if (m.to <= st->hlen) {
                    continue; /* ended in the look-behind: raised by an earlier write */
                }
                if (im->rules.exhaustible.count(m.id) && !st->seen->insert(m.id).second) {
                    continue; /* HS_FLAG_SINGLEMATCH: already raised on this stream */
                }
                if (onEvent && onEvent(m.id, 0, st->offset - st->hlen + m.to, 0, context)) {
                    st->status |= 1;
                    r = HS_SCAN_TERMINATED;
                    break;
                }
            }
            if (r == HS_SUCCESS) {
                if (rose->canExhaust && rose->ekeyCount && st->seen->size() >= im->rules.exhaustible.size()) {
                    st->status |= 2;
                }
                /* maintainHistoryBuffer (src/runtime.c:478-508) */
                const size_t keep = std::min<size_t>(buf.size(), st->hreq);
                memcpy(st->hist, buf.data() + buf.size() - keep, keep);
                st->hlen = (u32)keep;
                st->offset += length;
            }
        }
    }
    return r;
}

hs_error_t hs_scan_stream(hs_stream_t *st, const char *data, unsigned int length, unsigned int flags,
                          hs_scratch_t *scratch, match_event_handler onEvent, void *context) {
    (void)flags;
    if (!validStream(st) || !data || !validScratch(scratch)) {
        return HS_INVALID;
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    const hs_error_t r = streamWrite(st, data, length, scratch, onEvent, context);
    unmarkInUse(scratch);
    return r;
}

/* src/runtime.c:1106-1175: a temporary stream, one write per buffer, closed at
 * the end (pure-literal databases have no end-of-data reports). */
hs_error_t hs_scan_vector(const hs_database_t *db, const char *const *data, const unsigned int *length,
                          unsigned int count, unsigned int flags, hs_scratch_t *scratch,
                          match_event_handler onEvent, void *context) {
    (void)flags;
    if (!scratch || !data || !length) {
        return HS_INVALID;
    }
    hs_error_t err = checkDb(db, MODE_VECTORED);
    if (err != HS_SUCCESS) {
        return err;
    }
    if (!validScratch(scratch)) {
        return HS_INVALID;
    }
    const RoseEngine *rose = dbRose(db);
    if (rose->runtimeImpl != RUNTIME_PURE_LITERAL || rose->historyRequired > sizeof(((hs_stream *)0)->hist)) {
        return HS_ARCH_ERROR;
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    std::unordered_set<u32> seen;
    hs_stream st;
    memset(&st, 0, sizeof(st));
    st.magic = STREAM_MAGIC;
    st.db = db;
    st.hreq = rose->historyRequired;
    st.seen = &seen;
    hs_error_t r = HS_SUCCESS;
    for (unsigned int i = 0; i < count && r == HS_SUCCESS; i++) {
        if (!data[i]) {
            r = HS_INVALID; /* hs_scan_stream_internal: src/runtime.c:875 */
            break;
        }
        r = streamWrite(&st, data[i], length[i], scratch, onEvent, context);
    }
    unmarkInUse(scratch);
    return r;
}

hs_error_t hs_close_stream(hs_stream_t *st, hs_scratch_t *scratch, match_event_handler onEvent,
                           void *context) {
    (void)scratch; /* pure-literal databases have no end-of-data work (src/runtime.c:1005-1050) */
    (void)onEvent;
    (void)context;
    if (!validStream(st)) {
        return HS_INVALID;
    }
    st->magic = 0;
    delete st->seen;
    g_stream_free(st);
    return HS_SUCCESS;
}

hs_error_t hs_reset_stream(hs_stream_t *st, unsigned int flags, hs_scratch_t *scratch,
                           match_event_handler onEvent, void *context) {
    (void)flags;
    (void)scratch;
    (void)onEvent;
    (void)context;
    if (!validStream(st)) {
        return HS_INVALID;
    }
    resetStreamState(st);
    return HS_SUCCESS;
}

hs_error_t hs_copy_stream(hs_stream_t **to_id, const hs_stream_t *from_id) {
    if (!to_id) {
        return HS_INVALID;
    }
    *to_id = nullptr;
    if (!validStream(from_id)) {
        return HS_INVALID;
    }
    hs_stream *st = (hs_stream *)g_stream_alloc(sizeof(hs_stream));
    hs_error_t err = checkAlloc(st);
    if (err != HS_SUCCESS) {
        g_stream_free(st);
        return err;
    }
    memcpy(st, from_id, sizeof(*st));
    st->seen = new (std::nothrow) std::unordered_set<u32>(*from_id->seen);
    if (!st->seen) {
        g_stream_free(st);
        return HS_NOMEM;
    }
    *to_id = st;
    return HS_SUCCESS;
}

hs_error_t hs_reset_and_copy_stream(hs_stream_t *to_id, const hs_stream_t *from_id,
                                    hs_scratch_t *scratch, match_event_handler onEvent,
                                    void *context) {
    (void)scratch;
    (void)onEvent;
    (void)context;
    if (!validStream(to_id) || !validStream(from_id) || to_id == from_id) {
        return HS_INVALID;
    }
    if (to_id->db != from_id->db) {
        return HS_INVALID; /* src/runtime.c:758-760: streams of different databases */
    }
    std::unordered_set<u32> *keep = to_id->seen;
    *keep = *from_id->seen;
    memcpy(to_id, from_id, sizeof(*to_id));
    to_id->seen = keep;
    return HS_SUCCESS;
}

/* ---- stream compression (src/runtime.c:1177-1282, src/stream_compress_impl.h) ------
 * Flat form of a hs_stream: header {magic, database crc, status, look-behind
 * length, number of single-match ids already raised, stream offset}, the
 * look-behind bytes, the ids. */

namespace {
const u32 COMPRESS_MAGIC = 0x504d4353; /* "SCMP" */
struct CompressedHeader {
    u32 magic, crc, status, hlen, nseen, reserved;
    u64 offset;
};

size_t compressedSize(const hs_stream *st) {
    return sizeof(CompressedHeader) + st->hlen + 4 * st->seen->size();
}

/* fills *st (whose db, hreq and seen set are already in place) from buf */
bool expandInto(hs_stream *st, const char *buf, size_t size) {
    CompressedHeader h;
    if (size < sizeof(h)) {
        return false;
    }
    memcpy(&h, buf, sizeof(h));
    const DbHeader *dh = (const DbHeader *)st->db;
    if (h.magic != COMPRESS_MAGIC || h.crc != dh->crc32 || h.hlen > st->hreq || h.hlen > sizeof(st->hist) ||
        h.status > 3 || size != sizeof(h) + h.hlen + 4ull * h.nseen) {
        return false;
    }
    st->offset = h.offset;
    st->hlen = h.hlen;
    st->status = (u8)h.status;
    memcpy(st->hist, buf + sizeof(h), h.hlen);
    st->seen->clear();
    for (u32 i = 0; i < h.nseen; i++) {
        u32 id;
        memcpy(&id, buf + sizeof(h) + h.hlen + 4ull * i, 4);
        st->seen->insert(id);
    }
    return true;
}
} // namespace

hs_error_t hs_compress_stream(const hs_stream_t *st, char *buf, size_t buf_space, size_t *used_space) {
    if (!validStream(st) || !used_space || (buf_space && !buf)) {
        return HS_INVALID;
    }
    const size_t need = compressedSize(st);
    *used_space = need;
    if (buf_space < need) {
        return HS_INSUFFICIENT_SPACE;
    }
    CompressedHeader h;
    memset(&h, 0, sizeof(h));
    h.magic = COMPRESS_MAGIC;
    h.crc = ((const DbHeader *)st->db)->crc32;
    h.status = st->status;
    h.hlen = st->hlen;
    h.nseen = (u32)st->seen->size();
    h.offset = st->offset;
    memcpy(buf, &h, sizeof(h));
    memcpy(buf + sizeof(h), st->hist, st->hlen);
    size_t pos = sizeof(h) + st->hlen;
    std::vector<u32> ids(st->seen->begin(), st->seen->end());
    std::sort(ids.begin(), ids.end()); /* equal states compress to equal bytes */
    for (u32 id : ids) {
        memcpy(buf + pos, &id, 4);
        pos += 4;
    }
    return HS_SUCCESS;
}

hs_error_t hs_expand_stream(const hs_database_t *db, hs_stream_t **stream, const char *buf, size_t buf_size) {
    if (!stream || !buf) {
        return HS_INVALID;
    }
    *stream = nullptr;
    hs_stream_t *st = nullptr;
    hs_error_t err = hs_open_stream(db, 0, &st); /* same checks: validity, alignment, mode, engine */
    if (err != HS_SUCCESS) {
        return err;
    }
    if (!expandInto(st, buf, buf_size)) {
        hs_close_stream(st, nullptr, nullptr, nullptr);
        return HS_INVALID;
    }
    *stream = st;
    return HS_SUCCESS;
}

hs_error_t hs_reset_and_expand_stream(hs_stream_t *to_stream, const char *buf, size_t buf_size,
                                      hs_scratch_t *scratch, match_event_handler onEvent, void *context) {
    (void)context;
    if (!validStream(to_stream) || !buf) {
        return HS_INVALID;
    }
    if (onEvent && !validScratch(scratch)) {
        return HS_INVALID; /* pure-literal databases have no end-of-data reports to deliver */
    }
    /* expand into a copy first: a bad buffer must leave the stream as it was */
    hs_stream tmp = *to_stream;
    std::unordered_set<u32> seen;
    tmp.seen = &seen;
    if (!expandInto(&tmp, buf, buf_size)) {
        return HS_INVALID;
    }
    std::unordered_set<u32> *keep = to_stream->seen;
    *keep = seen;
    *to_stream = tmp;
    to_stream->seen = keep;
    return HS_SUCCESS;
}

/* ---- stream sets: many streams, one write each per call, state resident in HBM ------
 * (BASELINE config 4 shape: 16 M x 1 KB streams).  Per stream 16 bytes live in
 * HBM: 7 look-behind bytes + their count, and the 64-bit stream offset.  A scan
 * copies the writes into a pitched corpus (16-byte header per stream), a
 * kernel drops each stream's look-behind into its header, the block kernel
 * scans the lot (blocks = look-behind ++ write, found by division), records
 * come out at stream offsets, and a kernel rolls history and offsets forward. */

struct hs_b200_stream_set {
    const hs_database_t *db;
    int device;
    size_t nstreams;
    u32 histReq;
    u8 *d_hist;     /* 8 bytes per stream */
    u64 *d_offset;
    u32 *d_len;     /* per-write lengths when they differ */
    StreamMark *d_mark;
    u32 epoch;      /* of the mark (StreamMark): advanced by finishScan when it has seen the set marked */
    hs_b200_corpus corpus; /* the pitched corpus of a pass: the set's staging (hs_b200_streams_scan) or the
                            * caller's buffer (hs_b200_streams_scan_async); its block lengths and stream state
                            * are the above */
};

hs_error_t hs_b200_streams_open(const hs_database_t *db, size_t nstreams, int device,
                                hs_b200_stream_set_t **set) {
    if (!set || nstreams == 0 || nstreams > 0xfffffff0u) {
        return HS_INVALID;
    }
    *set = nullptr;
    hs_error_t err = checkDb(db, MODE_STREAM);
    if (err != HS_SUCCESS) {
        return err;
    }
    const RoseEngine *rose = dbRose(db);
    if (rose->runtimeImpl != RUNTIME_PURE_LITERAL || rose->historyRequired > 7 || rose->ekeyCount) {
        /* HS_FLAG_SINGLEMATCH state per stream is kept only by hs_scan_stream */
        return HS_ARCH_ERROR;
    }
    if (cudaSetDevice(device) != cudaSuccess) {
        return HS_ARCH_ERROR;
    }
    hs_b200_stream_set *s = new (std::nothrow) hs_b200_stream_set();
    if (!s) {
        return HS_NOMEM;
    }
    s->db = db;
    s->device = device;
    s->nstreams = nstreams;
    s->histReq = rose->historyRequired;
    s->d_hist = nullptr;
    s->d_offset = nullptr;
    s->d_len = nullptr;
    s->d_mark = nullptr;
    s->epoch = 0;
    cudaError_t e = cudaMalloc(&s->d_hist, nstreams * 8);
    if (e == cudaSuccess) e = cudaMalloc(&s->d_offset, nstreams * 8);
    if (e == cudaSuccess) e = cudaMalloc(&s->d_len, nstreams * 4);
    if (e == cudaSuccess) e = cudaMalloc(&s->d_mark, sizeof(StreamMark));
    if (e == cudaSuccess) e = cudaMemset(s->d_mark, 0, sizeof(StreamMark));
    if (e == cudaSuccess) e = cudaMemset(s->d_hist, 0, nstreams * 8);
    if (e == cudaSuccess) e = cudaMemset(s->d_offset, 0, nstreams * 8);
    if (e != cudaSuccess) {
        hs_b200_streams_close(s);
        return e == cudaErrorMemoryAllocation ? HS_NOMEM : HS_UNKNOWN_ERROR;
    }
    s->corpus.device = device;
    s->corpus.d_len = s->d_len;
    s->corpus.streamHist = s->d_hist;
    s->corpus.streamOffset = s->d_offset;
    *set = s;
    return HS_SUCCESS;
}

hs_error_t hs_b200_streams_close(hs_b200_stream_set_t *s) {
    if (!s) {
        return HS_SUCCESS;
    }
    DeviceGuard guard(s->device);
    cudaFree(s->d_hist);
    cudaFree(s->d_offset);
    cudaFree(s->d_len);
    cudaFree(s->d_mark);
    cudaFree(s->corpus.d_alloc);
    delete s;
    return HS_SUCCESS;
}

size_t hs_b200_streams_state_bytes(const hs_b200_stream_set_t *s) { return s ? s->nstreams * 16 : 0; }

hs_error_t hs_b200_streams_read_state(const hs_b200_stream_set_t *s, unsigned char *look_behind,
                                      unsigned long long *offsets) {
    if (!s) {
        return HS_INVALID;
    }
    DeviceGuard guard(s->device);
    CUDA_TRY(cudaDeviceSynchronize());
    if (look_behind) {
        CUDA_TRY(cudaMemcpy(look_behind, s->d_hist, s->nstreams * 8, cudaMemcpyDeviceToHost));
    }
    if (offsets) {
        CUDA_TRY(cudaMemcpy(offsets, s->d_offset, s->nstreams * 8, cudaMemcpyDeviceToHost));
    }
    return HS_SUCCESS;
}

static StreamPass streamPass(hs_b200_stream_set_t *set, const u32 *srcLen) {
    StreamPass sp;
    sp.hist = set->d_hist;
    sp.offset = set->d_offset;
    sp.len = set->d_len;
    sp.srcLen = srcLen;
    sp.histReq = set->histReq;
    sp.mark = set->d_mark;
    sp.epoch = &set->epoch;
    return sp;
}

/* The set's corpus over n * pitch bytes at d_data: stream b's write at b * pitch + 16 */
static hs_b200_corpus *streamCorpus(hs_b200_stream_set_t *set, u8 *d_data, u32 pitch, u32 uniformLen,
                                    u64 readableEnd) {
    hs_b200_corpus *c = &set->corpus;
    c->d_data = d_data;
    c->nblocks = set->nstreams;
    c->bytes = (u64)set->nstreams * pitch;
    c->readableEnd = readableEnd;
    c->payload = 0;
    c->uniformPitch = 0;
    c->uniformLen = uniformLen;
    c->streamPitch = pitch;
    return c;
}

/* Copy one write per stream into the set's pitched staging corpus, then run the pass's device sequence
 * (enqueueScan with the stream pass: look-behind in front of every write, scan, advance) with the
 * grow-and-rescan loop and the host ordering of scanRecords. */
static hs_error_t streamsScanImpl(hs_b200_stream_set_t *set, const char *data,
                                  const unsigned long long *offsets, const unsigned int *lengths,
                                  hs_scratch *s, std::vector<DevMatch> *matches) {
    const size_t n = set->nstreams;
    if (s->device != set->device) {
        return HS_INVALID; /* the set's state and the scratch's ring must share a device */
    }
    DeviceGuard guard(set->device);
    DevImage *im = nullptr;
    hs_error_t r = findImage(s, set->db, &im);
    if (r != HS_SUCCESS) {
        return r;
    }
    /* write lengths: uniform (config 4) or per stream */
    u32 maxLen = 0, uni = lengths[0];
    bool contiguous = true;
    for (size_t i = 0; i < n; i++) {
        maxLen = std::max(maxLen, lengths[i]);
        if (lengths[i] != uni) uni = 0;
        if (offsets[i] != offsets[0] + (u64)i * lengths[0]) contiguous = false;
    }
    if (maxLen == 0) {
        return HS_SUCCESS;
    }
    const u32 pitch = 16 + (u32)HSB_ROUNDUP((u64)maxLen, 16);
    hs_b200_corpus *c = &set->corpus;
    const u64 total = (u64)n * pitch;
    r = reserveCorpus(c, total, 0);
    if (r != HS_SUCCESS) {
        return r;
    }
    cudaStream_t st = s->stream;
    cudaError_t e;
    if (uni && contiguous) {
        e = cudaMemcpy2DAsync(c->d_data + 16, pitch, data + offsets[0], uni, uni, n,
                              cudaMemcpyHostToDevice, st);
    } else {
        /* ragged writes: pack on the host, one copy */
        std::vector<u8> pack((size_t)total, 0);
        for (size_t i = 0; i < n; i++) {
            memcpy(pack.data() + i * pitch + 16, data + offsets[i], lengths[i]);
        }
        e = cudaMemcpyAsync(c->d_data, pack.data(), total, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st); /* `pack` dies at scope end */
        if (e == cudaSuccess && !uni) {
            e = cudaMemcpyAsync(set->d_len, lengths, n * 4, cudaMemcpyHostToDevice, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
    }
    if (e == cudaSuccess) {
        e = cudaMemsetAsync(c->d_data + total, 0, 48, st);
    }
    if (e != cudaSuccess) {
        return HS_UNKNOWN_ERROR;
    }
    c = streamCorpus(set, c->d_data, pitch, uni, HSB_ROUNDUP(total, 16) + 16);
    const StreamPass sp = streamPass(set, nullptr);
    /* a rescan reads the staged writes again */
    return scanRecords(s, im, c, nullptr, true, matches, nullptr, nullptr, &sp);
}

/* hs_b200_streams_scan and _collect: check the arguments, mark the scratch in use,
 * scan and hand the records to deliver() before the mark is released. */
static hs_error_t streamSetScan(hs_b200_stream_set_t *set, const char *data, const unsigned long long *offsets,
                                const unsigned int *lengths, hs_scratch_t *scratch,
                                const std::function<hs_error_t(const std::vector<DevMatch> &)> &deliver) {
    if (!set || !data || !offsets || !lengths || !validScratch(scratch)) {
        return HS_INVALID;
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    std::vector<DevMatch> matches;
    hs_error_t r = streamsScanImpl(set, data, offsets, lengths, scratch, &matches);
    if (r == HS_SUCCESS) {
        r = deliver(matches);
    }
    unmarkInUse(scratch);
    return r;
}

hs_error_t hs_b200_streams_scan(hs_b200_stream_set_t *set, const char *data,
                                const unsigned long long *offsets, const unsigned int *lengths,
                                hs_scratch_t *scratch, hs_b200_block_event_handler onEvent,
                                void *context, unsigned long long *nmatches) {
    return streamSetScan(set, data, offsets, lengths, scratch, [&](const std::vector<DevMatch> &matches) {
        if (nmatches) {
            *nmatches = matches.size();
        }
        if (onEvent) {
            for (const DevMatch &m : matches) {
                onEvent(m.block, m.id, 0, m.to, 0, context);
            }
        }
        return HS_SUCCESS;
    });
}

hs_error_t hs_b200_streams_scan_collect(hs_b200_stream_set_t *set, const char *data,
                                        const unsigned long long *offsets,
                                        const unsigned int *lengths, hs_scratch_t *scratch,
                                        hs_b200_match_t *out, size_t cap,
                                        unsigned long long *nmatches) {
    if (!nmatches || (cap && !out)) {
        return HS_INVALID;
    }
    return streamSetScan(set, data, offsets, lengths, scratch, [&](const std::vector<DevMatch> &matches) {
        *nmatches = matches.size();
        memcpy(out, matches.data(), std::min(cap, matches.size()) * sizeof(DevMatch));
        /* the stream state HAS advanced; the first cap records are valid */
        return matches.size() > cap ? HS_INSUFFICIENT_SPACE : HS_SUCCESS;
    });
}

/* hs_b200_streams_scan_mask_async when mask is set, else hs_b200_streams_scan_async */
static hs_error_t streamsPass(hs_b200_stream_set_t *set, void *d_writes, size_t pitch, const unsigned int *d_lengths,
                              unsigned int uniform_length, hs_scratch_t *scratch, void *cuda_stream, bool mask,
                              void *d_mask, size_t words_per_block, void *d_status) {
    if (!set || !d_writes || (uintptr_t)d_writes % 16 || pitch < 32 || pitch % 16 || pitch > 0xfffffff0u ||
        (!d_lengths && uniform_length > pitch - 16) || !validScratch(scratch) || scratch->device != set->device) {
        return HS_INVALID;
    }
    if (mask && scratch->nPeers) {
        return HS_ARCH_ERROR;
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(set->device);
    DevImage *im = nullptr;
    hs_error_t r = findImage(scratch, set->db, &im);
    MaskOut m;
    if (r == HS_SUCCESS && mask) {
        r = maskArgs(im, OUT_MASK, set->nstreams, d_mask, words_per_block, d_status, &m);
        if (r != HS_SUCCESS) {
            unmarkInUse(scratch);
            return r;
        }
    }
    if (r == HS_SUCCESS) {
        cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
        /* no uniform length and no device lengths: no stream has a write, which the scan reads from the
         * set's length table */
        if (!d_lengths && !uniform_length &&
            cudaMemsetAsync(set->d_len, 0, set->nstreams * sizeof(u32), st) != cudaSuccess) {
            r = HS_UNKNOWN_ERROR;
        }
        /* the caller's buffer as it is: nothing before it and nothing past the last stream is read */
        const u64 bytes = (u64)set->nstreams * pitch;
        hs_b200_corpus *c = streamCorpus(set, (u8 *)d_writes, (u32)pitch, d_lengths ? 0 : uniform_length, bytes);
        const StreamPass sp = streamPass(set, d_lengths);
        if (r == HS_SUCCESS) {
            /* a mask pass: the confirm kernel finds the stream as the block and drops the look-behind's ends, as it
             * does for records, and the status is written after the advance has taken the set's verdict */
            r = enqueueScan(scratch, im, c, st, nullptr, &sp, nullptr, mask ? &m : nullptr, (u32 *)d_status);
        }
        scratch->lastCorpus = c;
        scratch->lastBlocks = set->nstreams;
        scratch->lastMaxLen = 0;
    }
    unmarkInUse(scratch);
    return r;
}

hs_error_t hs_b200_streams_scan_async(hs_b200_stream_set_t *set, void *d_writes, size_t pitch,
                                      const unsigned int *d_lengths, unsigned int uniform_length,
                                      hs_scratch_t *scratch, void *cuda_stream) {
    return streamsPass(set, d_writes, pitch, d_lengths, uniform_length, scratch, cuda_stream, false, nullptr, 0,
                       nullptr);
}

hs_error_t hs_b200_streams_scan_mask_async(hs_b200_stream_set_t *set, void *d_writes, size_t pitch,
                                           const unsigned int *d_lengths, unsigned int uniform_length,
                                           hs_scratch_t *scratch, void *d_mask, size_t words_per_block,
                                           void *d_status, void *cuda_stream) {
    return streamsPass(set, d_writes, pitch, d_lengths, uniform_length, scratch, cuda_stream, true, d_mask,
                       words_per_block, d_status);
}

hs_error_t hs_b200_streams_reset_async(hs_b200_stream_set_t *set, const unsigned int *d_streams, size_t count,
                                       void *cuda_stream) {
    if (!set || (d_streams && count > 0xffffffffu)) {
        return HS_INVALID;
    }
    DeviceGuard guard(set->device);
    const u32 n = d_streams ? (u32)count : (u32)set->nstreams;
    if (launchStreamReset(set->d_hist, set->d_offset, d_streams, n, (u32)set->nstreams, set->d_mark, set->epoch,
                          (cudaStream_t)cuda_stream) != cudaSuccess) {
        return HS_UNKNOWN_ERROR;
    }
    g_launches += n != 0;
    return HS_SUCCESS;
}

/* A stream-set pass over no rows: nothing to scan, but it takes the set's verdict like every other pass, so that
 * behind a pass that overflowed or was bad in this epoch it commits nothing either and finish reports that epoch's
 * outcome (HS_INSUFFICIENT_SPACE, HS_INVALID) */
static hs_error_t emptyStreamPass(hs_scratch *s, hs_b200_stream_set *set, cudaStream_t st, u32 *status) {
    CUDA_TRY(cudaMemsetAsync(s->d_counters, 0, CTR_COUNT * sizeof(u32), st));
    CUDA_TRY(cudaEventRecord(s->evStart, st));
    CUDA_TRY(cudaEventRecord(s->evStop, st));
    CUDA_TRY(launchStreamVerdict(s->d_counters, s->outCap, set->d_mark, set->epoch, st));
    g_launches++;
    if (status) { /* a mask pass over no rows: a mask of no words, and the verdict's status */
        CUDA_TRY(launchMaskStatus(s->d_counters, s->outCap, status, st));
        g_launches++;
    }
    CUDA_TRY(cudaMemcpyAsync(s->h_counters, s->d_counters, CTR_COUNT * sizeof(u32), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(s->evDone, st));
    s->pending = true;
    return HS_SUCCESS;
}

/* hs_b200_streams_scan_rows_mask_async when mask is set, else hs_b200_streams_scan_rows_async */
static hs_error_t streamsRowsPass(hs_b200_stream_set_t *set, const void *d_chars, size_t chars_bytes,
                                  const unsigned long long *d_offsets, const unsigned int *d_stream_ids, size_t nrows,
                                  hs_scratch_t *scratch, void *cuda_stream, bool mask, void *d_mask,
                                  size_t words_per_block, void *d_status) {
    if (!set || !d_offsets || (uintptr_t)d_offsets % 8 || (!d_chars && chars_bytes) || (!d_stream_ids && nrows) ||
        (uintptr_t)d_stream_ids % 4 || nrows > 0xfffffff0u || !validScratch(scratch) || scratch->device != set->device) {
        return HS_INVALID;
    }
    DevImage *im = heldImage(scratch, set->db);
    if (!im) {
        return HS_INVALID;
    }
    if (scratch->nPeers) {
        return HS_ARCH_ERROR; /* the exchanged records would be the scan's, not the rewritten ones */
    }
    MaskOut m;
    if (mask) {
        const hs_error_t r = maskArgs(im, OUT_MASK, nrows, d_mask, words_per_block, d_status, &m);
        if (r != HS_SUCCESS) {
            return r;
        }
    }
    if (markInUse(scratch)) {
        return HS_SCRATCH_IN_USE;
    }
    DeviceGuard guard(set->device);
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : scratch->stream;
    /* a group's block takes its rows' bytes, at most 7 look-behind bytes and at most 15 of pad (16 for an empty
     * group), and the table's unused entries are empty blocks 16 bytes apart behind the last one */
    const u64 bound = (u64)chars_bytes + 32 * (u64)nrows;
    const size_t n = nrows, tiles = (n + ROWS_TILE - 1) / ROWS_TILE;
    size_t at = 0;
    auto carve = [&](size_t bytes) {
        const size_t o = at;
        at = HSB_ROUNDUP(at + bytes, 256);
        return o;
    };
    const size_t oHead = carve(sizeof(StreamRowsHead)), oDigits = carve(256 * tiles * 4), oTileA = carve(tiles * 8),
                 oTileB = carve(tiles * 8), oPairs0 = carve(n * 8), oPairs1 = carve(n * 8), oPos = carve(n * 8),
                 oGroup = carve(n * 4), oFirst = carve((n + 1) * 4), oGPos = carve((n + 1) * 8),
                 oStream = carve(n * 4), oHl = carve(n * 4), oBase = carve(n * 8);
    hs_error_t r = nrows ? reserveRows(scratch, bound, nrows, at)
                         : emptyStreamPass(scratch, set, st, mask ? (u32 *)d_status : nullptr);
    hs_b200_corpus *c = scratch->rowsCorpus;
    if (r == HS_SUCCESS && nrows) {
        c->nblocks = nrows;
        c->bytes = bound;
        c->readableEnd = HSB_ROUNDUP(bound, 16) + 16;
        c->payload = chars_bytes;
        c->uniformPitch = 0;
        c->uniformLen = 0;
        u8 *b = scratch->d_rows;
        StreamRowsParams p;
        p.chars = (const u8 *)d_chars;
        p.charsBytes = chars_bytes;
        p.offsets = (const u64 *)d_offsets;
        p.ids = d_stream_ids;
        p.nrows = (u32)nrows;
        p.nstreams = (u32)set->nstreams;
        p.passes = (bitWidth(set->nstreams - 1) + 7) / 8;
        p.lookBehind = set->d_hist;
        p.streamOffset = set->d_offset;
        p.histReq = set->histReq;
        p.mark = set->d_mark;
        p.epoch = set->epoch;
        p.corpus = c->d_data;
        p.zeroEnd = HSB_ROUNDUP(bound, 16) + 32;
        p.blockOff = c->d_off;
        p.blockLen = c->d_len;
        p.out = scratch->d_out;
        p.outCap = scratch->outCap;
        p.counters = scratch->d_counters;
        p.head = (StreamRowsHead *)(b + oHead);
        p.tileDigits = (u32 *)(b + oDigits);
        p.tileA = (u64 *)(b + oTileA);
        p.tileB = (u64 *)(b + oTileB);
        p.pairs[0] = (uint2 *)(b + oPairs0);
        p.pairs[1] = (uint2 *)(b + oPairs1);
        p.posOf = (u64 *)(b + oPos);
        p.groupOf = (u32 *)(b + oGroup);
        p.gFirst = (u32 *)(b + oFirst);
        p.gPos = (u64 *)(b + oGPos);
        p.gStream = (u32 *)(b + oStream);
        p.gHl = (u32 *)(b + oHl);
        p.gBase = (u64 *)(b + oBase);
        if (mask) { /* the confirm kernel maps each match to its row through the pass's tables */
            m.rows = streamRowsMap(p);
        }
        r = enqueueScan(scratch, im, c, st, nullptr, nullptr, nullptr, mask ? &m : nullptr, (u32 *)d_status, &p);
    }
    /* the pass belongs to the set's epoch: finish moves the set on when it sees the pass marked, and the ordering
     * takes the records for a stream database's */
    scratch->streamEpoch = &set->epoch;
    scratch->lastCorpus = c;
    scratch->lastBlocks = nrows;
    scratch->lastMaxLen = 0;
    unmarkInUse(scratch);
    return r;
}

hs_error_t hs_b200_streams_scan_rows_async(hs_b200_stream_set_t *set, const void *d_chars, size_t chars_bytes,
                                           const unsigned long long *d_offsets, const unsigned int *d_stream_ids,
                                           size_t nrows, hs_scratch_t *scratch, void *cuda_stream) {
    return streamsRowsPass(set, d_chars, chars_bytes, d_offsets, d_stream_ids, nrows, scratch, cuda_stream, false,
                           nullptr, 0, nullptr);
}

hs_error_t hs_b200_streams_scan_rows_mask_async(hs_b200_stream_set_t *set, const void *d_chars, size_t chars_bytes,
                                                const unsigned long long *d_offsets, const unsigned int *d_stream_ids,
                                                size_t nrows, hs_scratch_t *scratch, void *d_mask,
                                                size_t words_per_block, void *d_status, void *cuda_stream) {
    return streamsRowsPass(set, d_chars, chars_bytes, d_offsets, d_stream_ids, nrows, scratch, cuda_stream, true,
                           d_mask, words_per_block, d_status);
}

} /* extern "C" */
