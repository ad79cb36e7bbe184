/*
 * kernels.h -- launch interface between the C-ABI shim (api_device.cu) and the
 * sm_90a scan kernels (scan_kernels.cu).  Plain PODs only.
 */
#ifndef HSB200_KERNELS_H
#define HSB200_KERNELS_H

#include <cuda_runtime.h>

#include "../ref_layout.h"

/* Kernel launches and the dynamic shared-memory window are spelled through two
 * macros so that the same sources also compile as plain C++ for the SIMT
 * emulator of tests/emu (TEST infrastructure, -DHSB_HOST_EMU: kernel logic under
 * `pytest -m "not gpu"`).  In the product build they are exactly the CUDA forms;
 * libhs_b200.so contains no emulator and has no CPU scan path. */
#ifdef HSB_HOST_EMU
#define HSB_LAUNCH(kern, grid, block, smem, stream, ...) \
    hsb_emu::launch(dim3(grid), dim3(block), smem, [=]() { kern(__VA_ARGS__); })
#define HSB_DYNAMIC_SMEM(name) u8 *name = hsb_emu::dynamicSmem()
#define HSB_NOINLINE __attribute__((noinline))
#define HSB_GRID_CONSTANT
#else
#define HSB_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#define HSB_DYNAMIC_SMEM(name) extern __shared__ __align__(128) u8 name[]
#define HSB_NOINLINE __noinline__
/* kernel parameters whose address is taken (passed by reference into the out-of-line
 * drains) stay in the constant bank instead of being copied to every thread's stack */
#define HSB_GRID_CONSTANT __grid_constant__
#endif

namespace hsb {

/* First-stage ("shift-OR") filter variants.  An entry read at sampled position
 * x holds SLOTS bytes; byte p has bit b SET iff no literal of bucket b can end
 * at position x+p given the bytes at x (FDR: src/fdr/fdr.c:157-327; Teddy:
 * src/fdr/teddy.c:918-969 -- see DESIGN.md section 3 for the derivation). */
enum FilterKind {
    FK_BYTE32 = 0, /* index = 1 byte; u32 entry (4 slots x 8 buckets); table
                      replicated per lane (bank-conflict free).  8-bucket Teddy, noodle */
    FK_PAIR32 = 4, /* index = (class of byte 0, class of byte 1), 5 bits each, classes
                      from a per-lane byte table; u32 entry; both tables replicated per
                      lane (bank-conflict free).  FDR sets, and fat Teddy with its 16
                      buckets folded onto 8 bits.  Table image: 256 class words
                      (c0 << 7 | c1 << 12), then 1024 pair entries */
    FK_GRAM4 = 5,  /* index = classes of the FOUR bytes ending at a position (5 bits each) into
                      a 1 Mbit bitmap in shared memory; no buckets.  Large FDR sets whose
                      literals are all >= 4 bytes.  Table image: 256 class words
                      (4 * c); ScanParams.bitmap = the bitmap (bitmapBytes), bit c[e] of word
                      c[e-3] + 33 c[e-2] + 1025 c[e-1] */
    FK_OUTFIX = 6, /* no literal first stage at all: a database of one outfix or several, its engines run on
                      the DFA / NFA kernels (dfa_kernels.cu) */
};

enum ConfirmKind {
    CK_FDR = 0,    /* hash confirm: FDRConfirm / LitInfo (src/fdr/fdr_confirm.h) */
    CK_NOODLE = 1, /* single literal: noodTable msk/cmp (src/hwlm/noodle_internal.h) */
};

enum { MAX_PEERS = 8 };
enum { CTR_MATCHES = 0, CTR_ERROR = 1, CTR_CANDIDATES = 2, CTR_CONFIRMED = 3,
       CTR_PREFILTER_PASS = 4, CTR_CANDQ = 5 /* candidates handed to the confirm kernel */,
       CTR_STREAM = 6 /* a stream-set pass that did not commit: STREAM_MARKED, | STREAM_BAD_LENGTH; a row scan
                       * whose row table is bad: STREAM_BAD_LENGTH */,
       CTR_COUNT = 8 };

/* Every scan kernel stops at the prefilter and appends the surviving candidates
 * to a list in HBM; confirmKernel finishes them, one thread per candidate.  The
 * list is the SECOND half of the record ring the scratch allocated (records [outCap, 2 * outCap) of ScanParams.out), so no launch
 * parameter changes; if it overflows, the record count is raised above outCap
 * and the caller's grow-and-rescan path takes over. */
struct DevCand {
    u64 g;       /* corpus position of the candidate's last byte */
    u32 buckets; /* first-stage bucket bits */
    u32 pad;
};
enum { ERR_BAD_OPCODE = 1, ERR_INTERNAL = 2 };

/* a report instruction an engine's program reaches (db_walk.h ProgReport) */
struct OrderRep {
    u32 onmatch;
    s32 adjust;
    u64 lo, hi;    /* CHECK_BOUNDS on the record's end offset */
    u32 logical;   /* SET_LOGICAL: the record becomes a logical-key record */
    u32 pad;
};

/* A stream-set pass over rows (StreamRowsParams): the tables that map a match in a group's block back to the row
 * of the batch that holds its last byte (srRewriteKernel for records, the confirm kernel for a mask). */
struct StreamRowsMap {
    const uint2 *sorted; /* (stream, row) pairs in group order */
    const u64 *posOf;    /* per sorted position: the bytes of the sorted rows before it */
    const u64 *gPos;     /* per group: posOf of its first row */
    const u32 *gFirst;   /* per group (+ 1): its first sorted position */
    const u32 *gHl;      /* per group: the look-behind bytes at the front of its block */
};

/* The sorted position of the row of group g that holds sorted-row byte `at` (posOf's count): the last of the
 * group's rows that starts at or before it, so that an empty row holds no byte. */
__device__ __forceinline__ u32 streamRowAt(const u32 *gFirst, const u64 *posOf, u32 g, u64 at) {
    u32 a = gFirst[g], b = gFirst[g + 1];
    while (b - a > 1) {
        const u32 mid = a + ((b - a) >> 1);
        if (posOf[mid] <= at) {
            a = mid;
        } else {
            b = mid;
        }
    }
    return a;
}

/* A match-mask pass (hs_b200_scan_corpus_mask_async / hs_b200_scan_rows_mask_async): where a record would be
 * written, the match sets bit r % 32 of bits[block * words + r / 32] instead, r = the rank of its report id in
 * ids[0, nIds) (DeviceRules.ids).  An engine's record (a report program) first becomes the reports its program
 * raises, through the program tables the ordering uses (resolve.h).  In a stream-set mask pass over rows
 * (hs_b200_streams_scan_rows_mask_async) a block is a group of the batch: rows.sorted is set, and the bit goes to
 * the row that holds the match's last byte (resolve.h maskRowReport).
 * A first-match pass (hs_b200_scan_corpus_first_async / hs_b200_scan_rows_first_async) is described by the same
 * structure with `first` set instead of `bits`: where a record would be written, the match lowers first[block] to
 * (to << 32) | id (resolve.h firstReport), and the engine walks stop once nothing they find can be lower. */
enum OutKind { OUT_RECORDS = 0, OUT_MASK = 1, OUT_FIRST = 2 };
struct MaskOut {
    u32 *bits;       /* null: the pass writes records, or the first-match table */
    u32 words;       /* per block */
    u32 nIds;
    const u32 *ids;
    const u32 *progOff, *progStart;
    const OrderRep *reps;
    u32 nProg;
    StreamRowsMap rows; /* rows.sorted null: a block is a mask row */
    unsigned long long *first; /* a first-match pass: one entry per block, ~0 = none */
    u32 slack;       /* a first-match pass: how far before its raw end offset a report may lie (minus the smallest
                      * offset_adjust of the database's report programs, literal and engine) */
};

struct ScanParams {
    /* corpus: position 0 = first byte of the packed corpus; bytes
     * [-16, paddedBytes + 16) are readable; blocks start 16-byte aligned */
    const u8 *corpus;
    u64 corpusBytes;       /* end of the last block */
    u64 readableEnd;       /* multiple of 16, >= corpusBytes: loads may read up to here */
    u32 tileFirst;         /* tiles [tileFirst, tileFirst + ntiles) are scanned */
    u32 ntiles;
    u32 tileBytes;         /* multiple of 512 */
    u32 pfDist;            /* L2 prefetch distance: in 512-byte steps (pair, gram kernels),
                            * in 1 KiB iterations (wide kernel) */
    const u64 *blockOff;   /* ascending, 16-byte aligned */
    const u32 *blockLen;
    u32 nblocks;
    u32 uniformPitch;      /* != 0: blockOff[i] == i * uniformPitch */
    u32 uniformLen;        /* != 0 (with uniformPitch): every block has this length; no table reads */
    /* stream sets (hs_b200_streams_*): stream b's write at b * streamPitch + 16,
     * preceded by its look-behind; 8 bytes of state per stream (7 history bytes,
     * right-aligned, + their count) and the stream offset live in HBM */
    u32 streamPitch;
    const u8 *streamHist;
    const u64 *streamOffset;
    /* database image */
    const u8 *bc;          /* RoseEngine bytecode (device copy) */
    const u8 *table;       /* first-stage table in HBM (copied to smem) */
    u32 tableBytes;
    const u8 *bitmap;      /* second-stage prefilter (copied to smem), may be null; FK_PAIR32: the
                            * (32 KiB) bitmap goes to the class rows' upper halves */
    u32 bitmapBytes;       /* power of two >= 16, or 0 = no prefilter */
    u32 bitmapShift;       /* 32 - log2(bits) */
    u32 keyBytes;          /* 1..4: literal tail bytes hashed into the bitmap */
    u32 pairBytes;         /* FK_PAIR32: shared-memory bytes of the pair table = 4 KiB x classes of the
                            * second byte (<= 128 KiB) */
    u32 bitmapBits;        /* FK_PAIR32: bits of the first-level bitmap; index = mulhi(key * K, bits) */
    u32 bucketFold;        /* 1 = 16 confirm buckets (fat Teddy) behind 8 first-stage bits: bit i of a
                            * candidate stands for buckets i and i + 8 */
    const u32 *bitmap2;    /* optional second-level bitmap in HBM/L2 (large literal sets) */
    u32 bitmap2Shift;      /* 32 - log2(bits); 0 = none */
    u32 confOff;           /* CK_FDR: offset of the confirm base in bc */
    u32 engineOff;         /* CK_NOODLE: offset of the noodTable in bc */
    u32 confirmKind;
    u64 groups;
    /* output */
    DevMatch *out;
    u32 outCap;
    u32 *counters;
    /* fused exchange (multi-GPU): every record is also stored, over NVLink,
     * into slot [myRank][1 + i] of each peer's exchange buffer (peer-mapped
     * pointers; layout [nPeers][peerCap + 1] records, slot 0 = count) */
    u32 nPeers;
    u32 myRank;
    u32 peerCap;
    u32 blockBase;           /* added to block indices in exchanged records */
    DevMatch *peers[MAX_PEERS];
    MaskOut mask;            /* mask.bits != null: a mask pass (the confirm kernel sets bits, writes no records);
                              * mask.first != null: a first-match pass (confirmFirstKernel) */
};

struct LaunchCfg {
    int kind;      /* FilterKind: FK_BYTE32 = wide kernel, FK_PAIR32 = pair kernel, FK_GRAM4 = gram kernel */
    int slotBase;  /* FK_PAIR32: 0 = slots 0..3 (reference numbering), 1 = slots 1..4 */
    int heavy;     /* FK_PAIR32: 1 = one queue entry per word with candidates (saturating sets) */
    int grid;      /* CTAs (one per SM) */
    int warps;     /* per CTA: up to 32 (wide kernel) or 28 (pair, gram) */
    size_t smemBytes;
};

/* Dynamic shared memory the scan kernel of `kind` needs with queueWarps warps
 * (tableBytes: FK_PAIR32 = the pair table's shared-memory bytes; bitmapBytes:
 * FK_BYTE32 = the prefilter bitmap). */
size_t scanSmemBytes(int kind, u32 tableBytes, u32 bitmapBytes, int queueWarps);

/* Scan tiles [p.tileFirst, p.tileFirst + p.ntiles) up to the candidate list;
 * launchConfirm must follow on the same stream. */
cudaError_t launchScan(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream);

/* Finish the candidates the scan kernel left in the list (same stream, after it). */
cudaError_t launchConfirm(const LaunchCfg &cfg, const ScanParams &p, cudaStream_t stream);

/* Publish the record count of a finished scan into slot 0 of this rank's
 * region in every peer's exchange buffer (runs after the scan on its stream). */
cudaError_t launchPublishCount(const ScanParams &p, cudaStream_t stream);

/* The two ends of a mask or first-match pass: fill the n words of the caller's mask with 0 (a first-match table
 * with all ones: ones = true) after the counters are cleared, before the scan, and write its status from the pass's
 * counters (after the scan): 0 when the output is valid, 1 when hs_b200_scan_corpus_finish will not return
 * HS_SUCCESS (an error, a bad row table or a candidate-list overflow). */
cudaError_t launchMaskClear(u32 *bits, u64 n, int smCount, cudaStream_t stream, bool ones = false);
cudaError_t launchMaskStatus(const u32 *counters, u32 outCap, u32 *status, cudaStream_t stream);

/* A stream set's pass state in device memory.  A pass whose record ring or candidate list overflowed, or
 * whose device lengths were bad, does not advance its streams and marks the set; every later pass or reset on
 * a marked set commits nothing, and a later pass raises its record count above the ring, so that its ordering
 * reports the overflow.  Marks belong to an epoch of the set: when the host has seen a mark
 * (hs_b200_scan_corpus_finish) it moves the set to the next epoch, and the passes and resets enqueued from then
 * on, which carry the new epoch, find the set unmarked -- the passes and resets enqueued before stay without
 * effect however late they run, and no clear has to be ordered after them. */
struct StreamMark {
    u32 marked;  /* epoch + 1 of the mark, 0 = none */
    u32 need;    /* the largest record count a pass of the mark's epoch reported: what the ring must hold */
    u32 bad;     /* epoch + 1 of a pass with a write length above pitch - 16, 0 = none */
    u32 pad;
};
enum { STREAM_MARKED = 1, STREAM_BAD_LENGTH = 2 };

/* The verdict of a stream-set pass after its scan: may it commit?  It may not when the set is marked in this epoch,
 * the pass is bad, the scan failed or the record ring or candidate list overflowed; then `first` (one thread of the
 * launch) marks the set, remembers the largest record count since the mark and raises the pass's count above the
 * ring.  Every thread reaches the same verdict, because only a "no" is written (a mark of an earlier epoch is one
 * the host has seen: it counts as none). */
__device__ __forceinline__ bool streamPassCommits(u32 *counters, u32 outCap, StreamMark *mark, u32 epoch, bool first) {
    const u32 count = counters[CTR_MATCHES];
    const bool marked = mark->marked == epoch + 1, bad = mark->bad == epoch + 1;
    if (marked || bad || counters[CTR_ERROR] || count > outCap) {
        if (first) {
            const u32 need = max(max(marked ? mark->need : 0u, count), outCap + 1);
            mark->need = need;
            mark->marked = epoch + 1;
            counters[CTR_MATCHES] = need;
            counters[CTR_STREAM] = STREAM_MARKED | (bad ? (u32)STREAM_BAD_LENGTH : 0u);
        }
        return false;
    }
    return true;
}

/* stream-set helpers, each given the set's epoch at enqueue time: write every stream's look-behind in front of
 * its write (and, given srcLens, take the caller's device lengths into lens, a length above pitch - 16
 * becoming 0 and marking the pass bad) / roll history and offsets forward after a scan, only if the pass may
 * commit / end the flows of the listed streams (idx = null: all), unless the set is marked */
cudaError_t launchStreamAssemble(u8 *corpus, const u8 *hist, u32 nstreams, u32 pitch, const u32 *srcLens,
                                 u32 *lens, StreamMark *mark, u32 epoch, cudaStream_t stream);
cudaError_t launchStreamAdvance(const u8 *corpus, u8 *hist, u64 *offsets, const u32 *lens, u32 uniformLen,
                                u32 nstreams, u32 pitch, u32 histReq, u32 *counters, u32 outCap, StreamMark *mark,
                                u32 epoch, cudaStream_t stream);
cudaError_t launchStreamReset(u8 *hist, u64 *offsets, const u32 *idx, u32 count, u32 nstreams,
                              const StreamMark *mark, u32 epoch, cudaStream_t stream);

/* one engine of a fused launch (DfaParams.engines): its bytes in device memory and the DfaParams fields
 * that differ from engine to engine */
struct DfaEngine {
    const u8 *nfa;
    u32 tableBytes;
    u32 states;
    u32 squashes;
    u32 pad;
};

/* A piece of a block walked by one lane (DfaParams.segs): bytes [start, start + len) of block `block`.
 * A block that is not cut is one segment with both flags. */
struct DfaSeg {
    u32 block, start, len, flags;
};
enum { SEG_FIRST = 1, SEG_LAST = 2 };
/* the passes of a segmented engine run (DfaParams.segMode; DESIGN.md section 10f) */
enum { SEG_SPECULATE = 1, /* every segment j > 0 of a cut block: guess[j] from a warm-up walk, end[j] from guess[j] */
       SEG_JOIN = 2,      /* (a round) segment j re-walks from end[j - 1] where that is not guess[j] */
       SEG_CHECK = 5,     /* segment j where end[j - 1] is not guess[j]: the lowest such j per block into segOpen */
       SEG_SETTLE = 3,    /* one lane per cut block chains its segments from segOpen on: guess[j] becomes the true
                           * start */
       SEG_EMIT = 4 };    /* every segment walks from its true start and writes its records */
/* DfaParams.segStats: segments re-walked by SEG_JOIN / SEG_SETTLE, and the bytes walked again (up to where the
 * re-walk met the guess's walk) */
enum { SEGSTAT_WALKS = 0, SEGSTAT_BYTES = 1, SEGSTAT_COUNT = 2 };

/* DFA engines in block mode (dfa_kernels.cu): McClellan 8 / 16, Sheng -- the engine's
 * own bytes (struct NFA first) in device memory, one thread per block. */
struct DfaParams {
    const u8 *corpus;
    u64 readableEnd;
    const u64 *blockOff;
    const u32 *blockLen;
    u32 nblocks;
    u32 uniformPitch, uniformLen;
    const u8 *nfa;
    u32 kind;        /* NFA.type: NFA_MCCLELLAN_8 / NFA_MCCLELLAN_16 / NFA_SHENG */
    u32 tableBytes;  /* McClellan: bytes of the successor table (staged in shared memory if it fits) */
    u32 ilp;         /* blocks walked by one lane at a time: 1 or 2 (runtime option dfa_ilp) */
    u32 states;      /* McClellan-8: state_count (<= 256): rows of the byte-indexed table built in shared memory */
    u32 squashes;    /* LimEx: some exception squashes (LIMEX_SQUASH_CYCLIC / _REPORT): the kernel reads the squash masks */
    DevMatch *out;   /* {report, block, offset after the last byte} */
    u32 outCap;
    u32 *counters;   /* CTR_MATCHES */
    u64 toTag;       /* ORed into every record's offset: ENGINE_RECORD (db_walk.h) when the engine's records
                      * share the ring with a literal matcher's, else 0 */
    /* != null: ONE launch over nengines engines of this kind (device memory), each over every block; the grid
     * is engine-major, the CTAs of engines[i] come i-th, and its nfa, tableBytes and squashes stand in for the
     * fields above.  tableBytes and states then hold the largest engine's, which size the shared memory. */
    const DfaEngine *engines;
    u32 nengines;
    /* != null: a segmented run (launchDfaSegments sets the fields below): a lane's unit is segs[i] (the
     * cut blocks cuts[i] = {first segment, segments} in SEG_SETTLE), walked as pass segMode.  segStates holds
     * per engine of the launch guess[nsegs] then end[nsegs], states of the engine kind's size. */
    const DfaSeg *segs;
    u32 nsegs;
    u32 segMode;
    const uint2 *cuts;
    u32 ncuts;
    u32 warm;        /* bytes of the warm-up walk in front of a segment (SEG_SPECULATE) */
    u8 *segStates;
    unsigned long long *segStats; /* SEGSTAT_COUNT counters, accumulated */
    u32 *segOpen;    /* per engine of the launch, per block: the first segment whose start is not settled (SEG_CHECK;
                      * all ones = none), cleared by the caller */
    MaskOut mask;    /* mask.bits != null: a mask pass (the accepts set bits, no slot is reserved or written);
                      * mask.first != null: a first-match pass (the accepts lower the block's entry) */
};
cudaError_t launchDfa(const DfaParams &p, int smCount, int maxSmem, cudaStream_t stream);

/* The segment plan of an engine run: lanes an engine launch keeps resident, and the bytes of one
 * segment's two states (guess, end) per engine. */
u32 dfaResidentLanes(u32 kind, int smCount);
u32 dfaStateBytes(u32 kind);
/* The segmented walk of p (p.segs ... set, segMode ignored): SEG_SPECULATE, `rounds` SEG_JOIN rounds,
 * SEG_CHECK, SEG_SETTLE, SEG_EMIT; *launches receives the kernels launched. */
cudaError_t launchDfaSegments(const DfaParams &p, int smCount, int maxSmem, u32 rounds, cudaStream_t stream,
                              unsigned *launches);

/* ---- the report rules on the device (order_kernels.h): raw records -> delivered matches ---- */

enum { ORDER_THREADS = 256, ORDER_ITEMS = 8, ORDER_TILE = ORDER_THREADS * ORDER_ITEMS,
       ORDER_MAX_PASSES = 16 /* 8-bit digits of a key of 32 (block) + 64 (to) + 32 (id) bits */ };

/* device-side progress of one ordering */
struct OrderState {
    u64 maxTo;
    u32 n;           /* input records (0 after a ring overflow) */
    u32 m;           /* records after resolution */
    u32 kept;        /* records after dedupe and exhaustion */
    u32 maxBlock, maxId;
    u32 unknownIds;  /* some record carries an id outside the id table: the key holds ids, not ranks */
    u32 overflow;
    u32 passes;      /* radix passes the key needs */
    u32 idBits, toBits, blockBits;
};

struct OrderParams {
    /* the database's tables (DeviceRules) */
    u32 shape;                /* DbShape */
    const u32 *progOff, *progStart;
    const OrderRep *reps;
    u32 nProg;
    const u32 *ids;
    const u8 *idEx;
    u32 nIds;
    u32 anyEx;
    /* input: n records at `in`; with inCount, n = *inCount (the scan's record count), and a count above
     * inCap is a ring overflow */
    const DevMatch *in;
    const u32 *inCount;
    u32 inCap;
    u32 inN;
    /* temporaries, sized by the caller: resolved records up to bufCap; tiles of max(inCap, bufCap) */
    OrderState *st;
    DevMatch *buf[2];
    u32 bufCap;
    u32 *tileSum;
    u32 *hist;       /* [256][tileCap] per pass */
    u32 tileCap;
    u32 *binTotal;   /* [ORDER_MAX_PASSES][256] */
    u64 *exKey;      /* anyEx: hash table of (block, id rank) -> first record, exSlots (a power of two) */
    u32 *exFirst;
    u32 exSlots;
    /* output */
    DevMatch *out;
    u64 outCap;
    unsigned long long *count;
};
/* Enqueue the whole ordering on `stream`, with at most maxPasses radix passes (the key needs no more for
 * the input at hand); *launches receives the number of kernels launched. */
cudaError_t launchOrder(const OrderParams &p, u32 maxPasses, cudaStream_t stream, unsigned *launches);

/* ---- row scans (rows_kernels.h): rows at any byte of a device column -> a packed corpus and its plan ---- */

enum { ROWS_THREADS = 256, ROWS_ITEMS = 8, ROWS_TILE = ROWS_THREADS * ROWS_ITEMS,
       ROWS_SPAN = 4096 /* packed bytes per warp of the repack */ };

struct RowsParams {
    /* row i = chars[offsets[i], offsets[i + 1]) */
    const u8 *chars;
    u64 charsBytes;
    const u64 *offsets;
    u32 nrows;
    /* the packed corpus (position 0; bytes [0, zeroEnd) are written, pads and slack zero) and its block table */
    u8 *corpus;
    u64 zeroEnd;
    u64 *blockOff;
    u32 *blockLen;
    /* temporaries: per tile of ROWS_TILE rows its padded bytes (then their exclusive prefix) and a bad row */
    u64 *tilePad;
    u32 *tileBad;
    u32 *bad;        /* the verdict: the table is bad */
    /* the pass's counters: a bad table sets STREAM_BAD_LENGTH in CTR_STREAM and raises CTR_MATCHES above outCap */
    u32 *counters;
    u32 outCap;
};
/* Enqueue the plan and the repack (after the counters are cleared, before the scan); *launches: kernels launched */
cudaError_t launchRowPlan(const RowsParams &p, int smCount, cudaStream_t stream, unsigned *launches);

/* The segment plan of an engine run over a packed row corpus whose lengths only the device knows: every row longer
 * than cutAbove is cut into segLen-byte segments.  segs[segCap] and cuts[cutCap] are sized by the host's bound,
 * segFirst has nrows + 1 entries. */
struct RowSegParams {
    const u32 *blockLen;
    u32 nrows;
    u32 segLen, cutAbove;
    DfaSeg *segs;
    u32 segCap;
    uint2 *cuts;
    u32 cutCap;
    u32 *segFirst;
};
cudaError_t launchRowSegments(const RowSegParams &p, int smCount, cudaStream_t stream, unsigned *launches);

/* ---- stream-set passes over rows (stream_rows_kernels.h): rows tagged with their stream -> one block per stream ---- */

/* zeroed by the host before every pass */
struct StreamRowsHead {
    u32 bad;          /* the batch is bad: a stream id at or above nstreams, a bad row, a stream's block past 32 bits */
    u32 groups;       /* D: the distinct streams of the batch */
    u32 kept;         /* records the rewrite kept */
    u32 applied;      /* the rewrite ran (the pass may commit) */
    u64 packedEnd;    /* end of the last group's block */
    u32 digits[4 * 256]; /* per radix pass of the stream ids: the count of every digit value */
};

struct StreamRowsParams {
    /* row r = chars[offsets[r], offsets[r + 1]), written to stream ids[r] */
    const u8 *chars;
    u64 charsBytes;
    const u64 *offsets;
    const u32 *ids;
    u32 nrows;
    u32 nstreams;
    u32 passes;         /* 8-bit radix passes the stream ids need */
    /* the set: 8 bytes of look-behind per stream (7 bytes + their count), 64-bit offsets, the mark */
    u8 *lookBehind;
    u64 *streamOffset;
    u32 histReq;
    StreamMark *mark;
    u32 epoch;
    /* the packed corpus (bytes [0, zeroEnd) are written) and its block table, one block per group */
    u8 *corpus;
    u64 zeroEnd;
    u64 *blockOff;
    u32 *blockLen;
    /* the pass's record ring (2 * outCap records: the second half is free once the confirm kernel has run) */
    DevMatch *out;
    u32 outCap;
    u32 *counters;
    /* temporaries: tiles of ROWS_TILE entries */
    StreamRowsHead *head;
    u32 *tileDigits;    /* [256][tiles] */
    u64 *tileA, *tileB; /* [tiles] */
    uint2 *pairs[2];    /* [nrows] (stream, row): the sort's two buffers */
    u64 *posOf;         /* per sorted position: the bytes of the sorted rows before it */
    u32 *groupOf;       /* per sorted position: its group */
    u32 *gFirst;        /* per group (+ 1): its first sorted position */
    u64 *gPos;          /* per group (+ 1): posOf of its first row */
    u32 *gStream, *gHl; /* per group: its stream, and the look-behind bytes at the front of its block */
    u64 *gBase;         /* per group: the stream offset of its block's first byte */
};
/* Enqueue the grouping and the packing (after the counters are cleared, before the scan; the head zeroed) */
cudaError_t launchStreamRowsPlan(const StreamRowsParams &p, int smCount, cudaStream_t stream, unsigned *launches);
/* Enqueue the rewrite of the records and the advance of the streams (after the scan); a mask pass has no records
 * and only advances */
cudaError_t launchStreamRowsCommit(const StreamRowsParams &p, bool mask, int smCount, cudaStream_t stream,
                                   unsigned *launches);
/* The row map of a pass (StreamRowsMap), for its mask */
StreamRowsMap streamRowsMap(const StreamRowsParams &p);
/* The verdict of a pass over no rows (streamPassCommits on the cleared counters) */
cudaError_t launchStreamVerdict(u32 *counters, u32 outCap, StreamMark *mark, u32 epoch, cudaStream_t stream);

/* accel primitives (src/nfa/shufti.c, truffle.c, vermicelli.h): first
 * position in [0,len) whose byte is in the class, or len. */
cudaError_t launchAccelFind(int type, const u8 *params, const u8 *d_buf, u64 len,
                            u64 *d_result, cudaStream_t stream);

} // namespace hsb
#endif
