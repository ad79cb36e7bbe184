/*
 * hs_b200.h -- C ABI of libhs_b200.so, the H100-native block-mode scan runtime
 * for Hyperscan databases.
 *
 * Part 1 re-declares, with identical names, argument meaning and error
 * behaviour, the subset of the reference's public API (src/hs_common.h,
 * src/hs_compile.h, src/hs_runtime.h of intel/hyperscan 5.4.2) that sits on the
 * block-mode hot path, so that an application linked against libhs can be
 * re-linked against libhs_b200 (`#include <hs.h>` keeps working through
 * include/hs.h).  Each entry cites the reference declaration it replaces.
 *
 * Part 2 adds the batched / device-resident entry points a GPU needs to be fed
 * efficiently (hsbench scans a corpus of many blocks: tools/hsbench/main.cpp:
 * 503-527).  Plain pointers and sizes only; no torch / C++ types.
 */
#ifndef HS_B200_H
#define HS_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------
 * Part 1: reference-compatible API
 * ---------------------------------------------------------------------- */

struct hs_database;
typedef struct hs_database hs_database_t;   /* src/hs_common.h:47 */
struct hs_scratch;
typedef struct hs_scratch hs_scratch_t;     /* src/hs_runtime.h:60 */
typedef int hs_error_t;                     /* src/hs_common.h:52 */

/* error codes: src/hs_common.h:478-588 */
#define HS_SUCCESS 0
#define HS_INVALID (-1)
#define HS_NOMEM (-2)
#define HS_SCAN_TERMINATED (-3)
#define HS_COMPILER_ERROR (-4)
#define HS_DB_VERSION_ERROR (-5)
#define HS_DB_PLATFORM_ERROR (-6)
#define HS_DB_MODE_ERROR (-7)
#define HS_BAD_ALIGN (-8)
#define HS_BAD_ALLOC (-9)
#define HS_SCRATCH_IN_USE (-10)
#define HS_ARCH_ERROR (-11)
#define HS_INSUFFICIENT_SPACE (-12)
#define HS_UNKNOWN_ERROR (-13)

/* pattern flags: src/hs_compile.h:869-1005 */
#define HS_FLAG_CASELESS 1
#define HS_FLAG_DOTALL 2
#define HS_FLAG_MULTILINE 4
#define HS_FLAG_SINGLEMATCH 8
#define HS_FLAG_ALLOWEMPTY 16
#define HS_FLAG_UTF8 32
#define HS_FLAG_UCP 64
#define HS_FLAG_PREFILTER 128
#define HS_FLAG_SOM_LEFTMOST 256
#define HS_FLAG_COMBINATION 512
#define HS_FLAG_QUIET 1024

/* cpu features / tune: src/hs_compile.h:1011-1110 */
#define HS_CPU_FEATURES_AVX2 (1ULL << 2)
#define HS_CPU_FEATURES_AVX512 (1ULL << 3)
#define HS_CPU_FEATURES_AVX512VBMI (1ULL << 4)
#define HS_TUNE_FAMILY_GENERIC 0
#define HS_TUNE_FAMILY_ICX 10

/* modes: src/hs_compile.h:1156-1210 */
#define HS_MODE_BLOCK 1
#define HS_MODE_NOSTREAM 1
#define HS_MODE_STREAM 2
#define HS_MODE_VECTORED 4
#define HS_MODE_SOM_HORIZON_LARGE (1U << 24)
#define HS_MODE_SOM_HORIZON_MEDIUM (1U << 25)
#define HS_MODE_SOM_HORIZON_SMALL (1U << 26)

typedef struct hs_compile_error {   /* src/hs_compile.h:70-97 */
    char *message;
    int expression;
} hs_compile_error_t;

typedef struct hs_platform_info {   /* src/hs_compile.h:134-165 */
    unsigned int tune;
    unsigned long long cpu_features;
    unsigned long long reserved1;
    unsigned long long reserved2;
} hs_platform_info_t;

/* hs_expr_ext.flags (src/hs_compile.h:264-279): which fields are set.  The regex route takes min_offset,
 * max_offset (bounds on the match end: CHECK_BOUNDS in the report programs) and min_length (a length counter
 * in the automaton); edit / Hamming distance are refused. */
#define HS_EXT_FLAG_MIN_OFFSET 1ULL
#define HS_EXT_FLAG_MAX_OFFSET 2ULL
#define HS_EXT_FLAG_MIN_LENGTH 4ULL
#define HS_EXT_FLAG_EDIT_DISTANCE 8ULL
#define HS_EXT_FLAG_HAMMING_DISTANCE 16ULL

typedef struct hs_expr_ext {        /* src/hs_compile.h:214-262 */
    unsigned long long flags;
    unsigned long long min_offset;
    unsigned long long max_offset;
    unsigned long long min_length;
    unsigned edit_distance;
    unsigned hamming_distance;
} hs_expr_ext_t;

typedef struct hs_expr_info {       /* src/hs_compile.h:169-216 */
    unsigned int min_width;
    unsigned int max_width;
    char unordered_matches;
    char matches_at_eod;
    char matches_only_at_eod;
} hs_expr_info_t;

typedef void *(*hs_alloc_t)(size_t size);   /* src/hs_common.h:271 */
typedef void (*hs_free_t)(void *ptr);       /* src/hs_common.h:280 */

/* src/hs_runtime.h:68-129 -- `to` is the offset after the last byte of the
 * match; `from` is 0 (no SOM); non-zero return stops the scan. */
typedef int (*match_event_handler)(unsigned int id, unsigned long long from,
                                   unsigned long long to, unsigned int flags,
                                   void *context);

/* --- compile (host CPU; src/hs_compile.h:360-854).  This build carries a
 * literal compiler: hs_compile_lit* take any bytes; hs_compile* take a regex
 * that denotes a FINITE set of strings -- literal text and PCRE escapes,
 * groups, alternation, character classes without negation, the bounded
 * repeats ?, {n}, {n,m} (at most 4096 strings per expression) -- each string
 * becoming one literal under the expression's id.  An expression set that is
 * not such a set (unbounded repeats, ".", negated / POSIX classes, \d \w \s \h \v,
 * \b \B, "^" \A "$" \z \Z where the reference takes them, option groups (?ims-ims),
 * \Q..\E, ...; hs_compile_ext_multi with min_offset / max_offset / min_length) is compiled, in block
 * mode, to ONE engine -- a McClellan DFA when the determinised automaton is small, else a LimEx NFA (32- to
 * 512-state model) -- inside a single-outfix database
 * (ROSE_RUNTIME_SINGLE_OUTFIX) when its positions fit -- DESIGN.md section 10b.
 * Where they do not fit only because of expressions that are finite sets of
 * literals, those go to a literal matcher beside that engine instead
 * (ROSE_RUNTIME_FULL_ROSE, block mode) -- DESIGN.md section 10d.
 * Anything else (look-around, back-references, UTF-8 / UCP, larger sets, ...) yields
 * HS_COMPILER_ERROR with an explanatory hs_compile_error_t, exactly as the
 * reference reports unsupported constructs.
 * Logical combinations (HS_FLAG_COMBINATION, with HS_FLAG_QUIET on any expression) are
 * compiled in block mode, over either kind of database (DESIGN.md section 10c); in
 * streaming and vectored mode they are a compile error, and so is HS_FLAG_QUIET
 * together with HS_FLAG_SINGLEMATCH on an expression that is not a combination. */
hs_error_t hs_compile(const char *expression, unsigned int flags,
                      unsigned int mode, const hs_platform_info_t *platform,
                      hs_database_t **db, hs_compile_error_t **error);
hs_error_t hs_compile_multi(const char *const *expressions,
                            const unsigned int *flags, const unsigned int *ids,
                            unsigned int elements, unsigned int mode,
                            const hs_platform_info_t *platform,
                            hs_database_t **db, hs_compile_error_t **error);
hs_error_t hs_compile_ext_multi(const char *const *expressions,
                                const unsigned int *flags,
                                const unsigned int *ids,
                                const hs_expr_ext_t *const *ext,
                                unsigned int elements, unsigned int mode,
                                const hs_platform_info_t *platform,
                                hs_database_t **db, hs_compile_error_t **error);
hs_error_t hs_compile_lit(const char *expression, unsigned flags,
                          const size_t len, unsigned mode,
                          const hs_platform_info_t *platform,
                          hs_database_t **db, hs_compile_error_t **error);
hs_error_t hs_compile_lit_multi(const char *const *expressions,
                                const unsigned *flags, const unsigned *ids,
                                const size_t *lens, unsigned elements,
                                unsigned mode,
                                const hs_platform_info_t *platform,
                                hs_database_t **db, hs_compile_error_t **error);
hs_error_t hs_free_compile_error(hs_compile_error_t *error);
/* src/hs_compile.h:760-854; *info is allocated with the misc allocator */
hs_error_t hs_expression_info(const char *expression, unsigned int flags,
                              hs_expr_info_t **info, hs_compile_error_t **error);
hs_error_t hs_expression_ext_info(const char *expression, unsigned int flags,
                                  const hs_expr_ext_t *ext, hs_expr_info_t **info,
                                  hs_compile_error_t **error);
hs_error_t hs_populate_platform(hs_platform_info_t *platform);

/* --- database container (src/hs_common.h:84-262; format src/database.h) */
hs_error_t hs_free_database(hs_database_t *db);
hs_error_t hs_serialize_database(const hs_database_t *db, char **bytes,
                                 size_t *length);
hs_error_t hs_deserialize_database(const char *bytes, const size_t length,
                                   hs_database_t **db);
hs_error_t hs_deserialize_database_at(const char *bytes, const size_t length,
                                      hs_database_t *db);
hs_error_t hs_stream_size(const hs_database_t *database, size_t *stream_size);
hs_error_t hs_database_size(const hs_database_t *database, size_t *size);
hs_error_t hs_serialized_database_size(const char *bytes, const size_t length,
                                       size_t *deserialized_size);
hs_error_t hs_database_info(const hs_database_t *database, char **info);
hs_error_t hs_serialized_database_info(const char *bytes, size_t length,
                                       char **info);

/* --- allocators (src/hs_common.h:288-439; src/alloc.c:38-109) */
hs_error_t hs_set_allocator(hs_alloc_t alloc_func, hs_free_t free_func);
hs_error_t hs_set_database_allocator(hs_alloc_t alloc_func, hs_free_t free_func);
hs_error_t hs_set_misc_allocator(hs_alloc_t alloc_func, hs_free_t free_func);
hs_error_t hs_set_scratch_allocator(hs_alloc_t alloc_func, hs_free_t free_func);
hs_error_t hs_set_stream_allocator(hs_alloc_t alloc_func, hs_free_t free_func);

const char *hs_version(void);               /* src/hs_common.h:449 */
hs_error_t hs_valid_platform(void);         /* src/hs_common.h:467: here it
                                             * answers "is a CUDA device usable" */

/* --- scratch + scan (src/hs_runtime.h:479-609; src/runtime.c:316,
 * src/scratch.c:244) */
hs_error_t hs_alloc_scratch(const hs_database_t *db, hs_scratch_t **scratch);
hs_error_t hs_clone_scratch(const hs_scratch_t *src, hs_scratch_t **dest);
hs_error_t hs_scratch_size(const hs_scratch_t *scratch, size_t *scratch_size);
hs_error_t hs_free_scratch(hs_scratch_t *scratch);

hs_error_t hs_scan(const hs_database_t *db, const char *data,
                   unsigned int length, unsigned int flags,
                   hs_scratch_t *scratch, match_event_handler onEvent,
                   void *context);

/* --- streaming mode (src/hs_runtime.h:148-475; src/runtime.c:542-977).  Built
 * for literal databases compiled with HS_MODE_STREAM (literals up to 8 bytes:
 * the pure-literal streaming runtime of the reference, src/runtime.c:801-829).
 */
struct hs_stream;
typedef struct hs_stream hs_stream_t;       /* src/hs_runtime.h:54 */
hs_error_t hs_open_stream(const hs_database_t *db, unsigned int flags, hs_stream_t **stream);
hs_error_t hs_scan_stream(hs_stream_t *id, const char *data, unsigned int length,
                          unsigned int flags, hs_scratch_t *scratch,
                          match_event_handler onEvent, void *ctxt);
hs_error_t hs_close_stream(hs_stream_t *id, hs_scratch_t *scratch,
                           match_event_handler onEvent, void *ctxt);
hs_error_t hs_reset_stream(hs_stream_t *id, unsigned int flags, hs_scratch_t *scratch,
                           match_event_handler onEvent, void *context);
hs_error_t hs_copy_stream(hs_stream_t **to_id, const hs_stream_t *from_id);
hs_error_t hs_reset_and_copy_stream(hs_stream_t *to_id, const hs_stream_t *from_id,
                                    hs_scratch_t *scratch, match_event_handler onEvent,
                                    void *context);

/* Stream compression (src/hs_runtime.h:365-366, 395-397, 438-443;
 * src/runtime.c:1177-1282): a stream's state as a flat byte string.  The
 * format is private to a build, as in the reference; what is promised is the
 * round trip: a stream expanded from the bytes continues exactly as the
 * compressed one would have.  hs_compress_stream with too small a buffer
 * (NULL/0 allowed) returns HS_INSUFFICIENT_SPACE and the size needed. */
hs_error_t hs_compress_stream(const hs_stream_t *stream, char *buf, size_t buf_space,
                              size_t *used_space);
hs_error_t hs_expand_stream(const hs_database_t *db, hs_stream_t **stream, const char *buf,
                            size_t buf_size);
hs_error_t hs_reset_and_expand_stream(hs_stream_t *to_stream, const char *buf, size_t buf_size,
                                      hs_scratch_t *scratch, match_event_handler onEvent,
                                      void *context);

/* --- vectored mode (src/hs_runtime.h:484-527; src/runtime.c:1106-1175): the
 * `count` buffers are scanned as ONE stream in the order given -- matches may
 * span buffers and `to` counts from the start of the first buffer.  Needs a
 * database compiled with HS_MODE_VECTORED (HS_DB_MODE_ERROR otherwise); built,
 * like streaming, for literals of up to 8 bytes. */
hs_error_t hs_scan_vector(const hs_database_t *db, const char *const *data,
                          const unsigned int *length, unsigned int count,
                          unsigned int flags, hs_scratch_t *scratch,
                          match_event_handler onEvent, void *context);

/* ------------------------------------------------------------------------
 * Part 2: H100 batch / device-resident extension
 * ---------------------------------------------------------------------- */

/* One match record as the device writes it (16 bytes; SURVEY.md section 8d).
 * Raw records of a database with logical combinations (HS_FLAG_COMBINATION) also
 * hold logical-key records: bit 63 of `to` set, `id` = the logical key of a
 * sub-expression that matched, `to` & ~(1 << 63) = where.  No match offset reaches
 * 2^63, and every id is a valid user id, so the bit is what tells them apart.  The
 * ordered forms (callbacks, _collect, hs_b200_fetch_matches,
 * hs_b200_postprocess_blocks) replace them with the combination reports.  Raw
 * records of a database with a literal matcher beside an engine (DESIGN.md
 * section 10d) hold the engine's records with bit 62 of `to` set and `id` = a
 * report program's offset; the ordered forms resolve them into reports. */
typedef struct hs_b200_match {
    unsigned int id;             /* report id the user registered */
    unsigned int block;          /* index of the block in the batch */
    unsigned long long to;       /* end offset within the block */
} hs_b200_match_t;

/* Per-block callback for batched scans: like match_event_handler plus the
 * block index.  Non-zero return stops delivery for THAT block (the block's
 * scan is "terminated", like HS_SCAN_TERMINATED for one hs_scan call). */
typedef int (*hs_b200_block_event_handler)(unsigned int block, unsigned int id,
                                           unsigned long long from,
                                           unsigned long long to,
                                           unsigned int flags, void *context);

/* Scan `nblocks` independent blocks held in HOST memory: block i is
 * data[offsets[i] .. offsets[i]+lengths[i]).  Equivalent to nblocks hs_scan()
 * calls (one per hsbench DataBlock), performed as one H2D copy, one kernel
 * launch and one D2H of the match list; callbacks are replayed on the calling
 * thread in (block, to) order.  onEvent may be NULL (matches are only
 * counted).  *nmatches (optional) receives the number of matches delivered. */
hs_error_t hs_b200_scan_blocks(const hs_database_t *db, const char *data,
                               const unsigned long long *offsets,
                               const unsigned int *lengths, size_t nblocks,
                               hs_scratch_t *scratch,
                               hs_b200_block_event_handler onEvent,
                               void *context, unsigned long long *nmatches);

/* Same, the delivered matches written to `out` in (block, to, id) order (the order
 * the callbacks would fire in, all report rules applied) instead of one callback
 * per match.  With logical combinations the order within one (block, to) is the
 * reference's: the expressions' reports by id, then the combination reports the
 * offset completes, by combination (in the order the combinations were given).  HS_INSUFFICIENT_SPACE: more than `cap` matches (*nmatches tells; the
 * first cap are valid). */
hs_error_t hs_b200_scan_blocks_collect(const hs_database_t *db, const char *data,
                                       const unsigned long long *offsets,
                                       const unsigned int *lengths, size_t nblocks,
                                       hs_scratch_t *scratch, hs_b200_match_t *out, size_t cap,
                                       unsigned long long *nmatches);

/* Device-resident corpus handle: the packed, 16-byte-aligned copy of a set of
 * blocks in HBM plus its block table. */
struct hs_b200_corpus;
typedef struct hs_b200_corpus hs_b200_corpus_t;

/* Upload a corpus (host -> HBM).  `device` is the CUDA ordinal. */
hs_error_t hs_b200_corpus_upload(const char *data,
                                 const unsigned long long *offsets,
                                 const unsigned int *lengths, size_t nblocks,
                                 int device, hs_b200_corpus_t **corpus);
/* Wrap a corpus that is ALREADY in HBM (e.g. a torch tensor): d_data is a
 * device pointer, block starts must be 16-byte aligned within it; offsets and
 * lengths are host arrays (copied). */
hs_error_t hs_b200_corpus_wrap(const void *d_data, size_t data_bytes,
                               const unsigned long long *offsets,
                               const unsigned int *lengths, size_t nblocks,
                               int device, hs_b200_corpus_t **corpus);
hs_error_t hs_b200_corpus_free(hs_b200_corpus_t *corpus);
size_t hs_b200_corpus_bytes(const hs_b200_corpus_t *corpus);

/* Enqueue one scan of the whole corpus on `cuda_stream` (a cudaStream_t, or
 * NULL for the scratch's own stream) and return without synchronising.
 * Results stay in HBM inside the scratch. */
hs_error_t hs_b200_scan_corpus_async(const hs_database_t *db,
                                     const hs_b200_corpus_t *corpus,
                                     hs_scratch_t *scratch, void *cuda_stream);
/* Wait for the last enqueued scan; report how many raw match records it
 * produced and the device pointer of the record array (hs_b200_match_t[]).
 * Returns HS_INSUFFICIENT_SPACE if the record ring overflowed (after growing
 * the ring so that a re-run succeeds). */
hs_error_t hs_b200_scan_corpus_finish(hs_scratch_t *scratch,
                                      unsigned long long *nrecords,
                                      const void **d_records);
/* Copy up to `cap` raw records of the last finished scan into another device
 * buffer (e.g. a torch tensor that is then all-gathered over NCCL). */
hs_error_t hs_b200_copy_records(hs_scratch_t *scratch, void *d_dst, size_t cap);
/* Stream-ordered form for pipelines that never touch the host between a scan
 * and the exchange of its records: enqueue, on `cuda_stream` (the stream the
 * scan was enqueued on), a device-to-device copy of the first `cap` slots of
 * the record ring into d_dst and of the 32-bit record count into *d_count
 * (low word of a zeroed 64-bit slot).  Slots beyond the count hold stale data. */
hs_error_t hs_b200_export_records_async(hs_scratch_t *scratch, void *d_dst, size_t cap,
                                        void *d_count, void *cuda_stream);
/* Fused scan + all-gather over NVLink peer memory (one process per GPU).
 * Every rank allocates an exchange buffer of nranks x (cap + 1) records with
 * hs_b200_peer_buffer_alloc (cudaMalloc + cudaIpcGetMemHandle; the 64-byte
 * handle is sent to the other ranks by any means), opens the others' buffers
 * with hs_b200_peer_buffer_open (cudaIpcOpenMemHandle, peer access enabled),
 * and registers all bases -- its own included, in rank order -- with
 * hs_b200_set_peer_exchange.  From then on the scan kernel itself stores each
 * match record into slot [my_rank][1 + i] of EVERY rank's buffer as it is
 * found (block index + block_base), and slot [my_rank][0] receives the count
 * when the scan completes: no separate collective.  Records beyond `cap` are
 * only kept in the local ring (the count tells).  nranks = 0 disables it. */
hs_error_t hs_b200_peer_buffer_alloc(size_t bytes, void **d_ptr, unsigned char handle[64]);
hs_error_t hs_b200_peer_buffer_open(const unsigned char handle[64], void **d_ptr);
hs_error_t hs_b200_peer_buffer_read(const void *d_ptr, void *host_dst, size_t bytes);
hs_error_t hs_b200_peer_buffer_close(void *d_ptr, int opened);
hs_error_t hs_b200_set_peer_exchange(hs_scratch_t *scratch, unsigned int nranks,
                                     unsigned int my_rank, void *const *peer_bases,
                                     size_t cap_per_rank, unsigned int block_base);
/* Apply the host-side report rules to `n` raw records held in host memory
 * (in place; e.g. the concatenation of all ranks' records after the
 * all-gather): sort by (block, to, id), one record per (block, id, to),
 * HS_FLAG_SINGLEMATCH reports keep their first match per block.  Host only
 * (needs no CUDA device).  A database with logical combinations is refused
 * (HS_INVALID): its reports depend on the block lengths, see below. */
hs_error_t hs_b200_postprocess_matches(const hs_database_t *db,
                                       hs_b200_match_t *recs, size_t n,
                                       unsigned long long *nout);
/* The same for the raw records of blocks 0 .. nblocks-1 whose lengths are given,
 * for any database, written to `out`: with logical combinations, the logical-key
 * records are evaluated block by block as hs_scan would (a combination that is
 * true with none of its sub-expressions matched reports at the block's end), and
 * the order within one (block, to) is as for hs_b200_scan_blocks_collect.  Records
 * of blocks >= nblocks are dropped.  HS_INSUFFICIENT_SPACE: more than `cap` records
 * (*nout tells).  Host only. */
hs_error_t hs_b200_postprocess_blocks(const hs_database_t *db,
                                      const hs_b200_match_t *recs, size_t n,
                                      const unsigned int *lengths, size_t nblocks,
                                      hs_b200_match_t *out, size_t cap,
                                      unsigned long long *nout);
/* Copy the records of the last finished scan to the host, apply the
 * host-side report rules (dedupe per (id,to); HS_FLAG_SINGLEMATCH keeps the
 * first match per id and block), sort by (block, to, id).  `out` may be NULL
 * to query the count.  With logical combinations the combination reports are
 * added (order as for hs_b200_scan_blocks_collect); they need the block lengths
 * of the corpus last scanned, which must not have been freed. */
hs_error_t hs_b200_fetch_matches(const hs_database_t *db, hs_scratch_t *scratch,
                                 hs_b200_match_t *out, size_t cap,
                                 unsigned long long *nmatches);

/* Stream sets: `nstreams` streams of one HS_MODE_STREAM literal database whose
 * state (7 look-behind bytes + count, 64-bit offset: 16 bytes per stream) stays
 * in HBM between calls.  hs_b200_streams_scan() gives every stream one write
 * (stream i: data[offsets[i] .. +lengths[i]), HOST memory; zero-length = no
 * write) and delivers matches as (stream index, id, to = stream offset),
 * ordered by (stream, to).  Equivalent to one hs_scan_stream() per stream.
 * Databases with HS_FLAG_SINGLEMATCH patterns are refused (HS_ARCH_ERROR): their
 * per-stream exhaustion state is kept only by hs_scan_stream. */
struct hs_b200_stream_set;
typedef struct hs_b200_stream_set hs_b200_stream_set_t;
hs_error_t hs_b200_streams_open(const hs_database_t *db, size_t nstreams, int device,
                                hs_b200_stream_set_t **set);
hs_error_t hs_b200_streams_scan(hs_b200_stream_set_t *set, const char *data,
                                const unsigned long long *offsets,
                                const unsigned int *lengths, hs_scratch_t *scratch,
                                hs_b200_block_event_handler onEvent, void *context,
                                unsigned long long *nmatches);
/* Same, the ordered matches written to `out` (stream index in `block`) instead
 * of a callback per match.  HS_INSUFFICIENT_SPACE: more than `cap` matches
 * (*nmatches tells; the first cap are valid and the streams have advanced). */
hs_error_t hs_b200_streams_scan_collect(hs_b200_stream_set_t *set, const char *data,
                                        const unsigned long long *offsets,
                                        const unsigned int *lengths, hs_scratch_t *scratch,
                                        hs_b200_match_t *out, size_t cap,
                                        unsigned long long *nmatches);
size_t hs_b200_streams_state_bytes(const hs_b200_stream_set_t *set);
hs_error_t hs_b200_streams_close(hs_b200_stream_set_t *set);

/* Introspection used by tests and bench.py. */
typedef struct hs_b200_db_info {
    unsigned int runtime_impl;   /* RoseEngine.runtimeImpl */
    unsigned int hwlm_type;      /* 16 noodle, 12 FDR/Teddy, 0 none */
    unsigned int engine_id;      /* FDR: 0; Teddy: 3..18; single-outfix databases: the engine's NFAEngineType
                                  * (LimEx 0..5, McClellan-8 / -16 6 / 7, Sheng 17), its state count in num_literals */
    unsigned int fdr_domain;
    unsigned int fdr_stride;
    unsigned int num_literals;   /* HWLM literal fragments */
    unsigned int bytecode_len;
    unsigned int min_width;
} hs_b200_db_info_t;
hs_error_t hs_b200_db_info(const hs_database_t *db, hs_b200_db_info_t *info);

/* Process-wide build tunable (the analogue of the reference tools' -G Grey
 * overrides and of the engine "hints" its unit tests use,
 * unit/internal/fdr.cpp:114-137).  Keys: "force_engine" (-1 auto, 0 FDR, 3..18
 * Teddy engine id), "fdr_domain" (9..15), "fdr_stride" (1,2,4), "max_domain",
 * "allow_teddy", "allow_fat_teddy", "allow_flood", "allow_noodle"; "outfix_engine"
 * (0: literal matchers as usual; 1 DFA chosen by size, 2 McClellan-8, 3 McClellan-16,
 * 4 Sheng, 5 LimEx-32: hs_compile_lit* in block mode emit a database whose only matcher
 * is that engine over the whole literals, run as an outfix -- ROSE_RUNTIME_SINGLE_OUTFIX,
 * src/runtime.c:245-280; the reference's hs_scan and this one both scan it); "regex_dfa"
 * (1, the default: a regular-expression set whose determinised automaton has at most 1 024
 * states runs as a McClellan DFA; 0: always as a LimEx NFA); key "reset" restores the
 * defaults. */
hs_error_t hs_b200_set_build_option(const char *key, int value);

/* Acceleration primitives (src/nfa/accel.h:46-121; shuftiExec src/nfa/shufti.c:150,
 * truffleExec src/nfa/truffle.c:118, vermicelliExec / vermicelliDoubleExec
 * src/nfa/vermicelli.h:43,172) on the device: *pos = first position in
 * [0, len) whose byte (pair) is in the class, or len.  type = the reference's
 * AccelType: 1 VERM, 2 VERM_NOCASE, 3 DVERM, 4 DVERM_NOCASE (params = c1[,c2],
 * upper case for NOCASE), 13 SHUFTI (params = lo[16], hi[16]), 15 TRUFFLE
 * (params = mask1[16] (bytes < 0x80), mask2[16]). */
hs_error_t hs_b200_accel_find(unsigned int type, const unsigned char *params,
                              const unsigned char *buf, size_t len,
                              unsigned long long *pos);

/* Table builder at the boundary the reference's unit tests use (hwlmBuild(),
 * unit/internal/fdr.cpp:140-165): raw HWLM table for literals (bytes, nocase,
 * noruns, id); engine -1 auto, 0 FDR (domain 9, stride 1 like the reference's
 * unit-test hint), 3..18 Teddy id.  Returns the size or -1. */
long hs_b200_test_build_hwlm(const char *const *lits, const size_t *lens,
                             const unsigned *nocase, const unsigned *noruns,
                             const unsigned *ids, unsigned n, int engine, void *out,
                             size_t cap);

/* ---- DFA engines (part of the regex half of the path; SURVEY.md section 8a rows a18, a19, a21) ----
 *
 * The reference's DFA engines in block mode, from the engines' own serialized bytes
 * (`struct NFA` header, src/nfa/nfa_internal.h:84-126, followed by `struct mcclellan`
 * or `struct sheng`): replaces nfaExecMcClellan8_B / nfaExecMcClellan16_B
 * (src/nfa/mcclellan.c:937-973) and nfaExecSheng_B (src/nfa/sheng.c:706-739), the
 * entry points the block runtime uses for its anchored table (src/rose/block.c:42-91)
 * and its small-write engine (src/runtime.c:285-315).  Run over every block of a
 * resident corpus (offset 0 per block); every callback (report, end) the reference
 * would fire comes back as a record {id = report, block, to = end}, ordered by
 * (block, to, id).  HS_ARCH_ERROR: engine type or feature (wide states) not built;
 * HS_INSUFFICIENT_SPACE: more than `cap` records (*nmatches tells). */
hs_error_t hs_b200_nfa_scan_corpus(const void *nfa, size_t nfa_len, const hs_b200_corpus_t *corpus,
                                   hs_b200_match_t *out, size_t cap, unsigned long long *nmatches,
                                   float *kernel_ms);

/* Emit such engines on the host (the reference's compile side -- parser, Glushkov
 * graph, determinisation -- stays out of scope; what can be given is a literal set,
 * for which the Aho-Corasick automaton is built, or a finished DFA table).
 * kind: 0 auto (Sheng <= 16 states, McClellan8 <= 256, else McClellan16), 1 McClellan8,
 * 2 McClellan16, 3 Sheng; sherman != 0: McClellan16 stores states close to the start
 * state's row as 32-byte Sherman exception lists.  State 0 is the dead state.
 * report_off / eod_off: nstates + 1 offsets into reports / eod_reports.
 * Return the size written to `out`, or -1. */
long hs_b200_dfa_from_literals(const char *const *lits, const size_t *lens, const unsigned *caseless,
                               const unsigned *reports, unsigned n, int anchored, int kind, int sherman,
                               void *out, size_t cap);
long hs_b200_dfa_from_table(unsigned nstates, const unsigned short *next, unsigned start_anchored,
                            unsigned start_floating, const unsigned *report_off, const unsigned *reports,
                            const unsigned *eod_off, const unsigned *eod_reports, int kind, int sherman,
                            void *out, size_t cap);

/* LimEx NFA, 32-state model (src/nfa/limex_internal.h:102-203), emitted in the reference's
 * layout from a literal set (position automaton, <= 31 literal bytes in total) or from a
 * finished NFA: reach256[b] = states that may be on after byte b; succ[i] = successor set of
 * state i; init / init_ds = states a top switches on at offset 0 / later; squash_kind[i]
 * (0 none, 1 cyclic, 3 report: src/nfa/limex_internal.h:98-103) with squash_mask[i];
 * report_off / eod_off: nstates + 1 offsets into reports / eod_reports.  The engine runs
 * on hs_b200_nfa_scan_corpus like the DFAs (block-mode semantics of an outfix: one top at
 * offset 0, nfaExecLimEx32_Q over the block, then _testEOD).  Size written, or -1. */
long hs_b200_limex32_from_literals(const char *const *lits, const size_t *lens, const unsigned *caseless,
                                   const unsigned *reports, unsigned n, void *out, size_t cap);
long hs_b200_limex32_from_spec(unsigned nstates, const unsigned *reach256, unsigned init, unsigned init_ds,
                               const unsigned *succ, const unsigned *squash_mask,
                               const unsigned char *squash_kind, const unsigned *report_off,
                               const unsigned *reports, const unsigned *eod_off, const unsigned *eod_reports,
                               void *out, size_t cap);
/* the same over 64-bit state sets: up to 64 states; more than 32 are emitted as the 64-state
 * model (struct LimExNFA64, nfaExecLimEx64_Q); hs_b200_limex32_from_literals does the same
 * for literal sets of up to 63 bytes in total */
long hs_b200_limex_from_spec64(unsigned nstates, const unsigned long long *reach256, unsigned long long init,
                               unsigned long long init_ds, const unsigned long long *succ,
                               const unsigned long long *squash_mask, const unsigned char *squash_kind,
                               const unsigned *report_off, const unsigned *reports, const unsigned *eod_off,
                               const unsigned *eod_reports, void *out, size_t cap);
/* ... and over state sets of `words` 64-bit words each (words <= 8: up to 512 states; every set argument is
 * `words` little-endian words per set, reach256 = 256 sets, succ / squash_mask = nstates sets): emitted as the
 * smallest of the 32 / 64 / 128 / 256 / 512-state models that holds nstates (struct LimExNFA128 ...,
 * nfaExecLimEx128_Q ...; an automaton of 257-384 states takes the 512-state model) */
long hs_b200_limex_from_spec_wide(unsigned nstates, unsigned words, const unsigned long long *reach256,
                                  const unsigned long long *init, const unsigned long long *init_ds,
                                  const unsigned long long *succ, const unsigned long long *squash_mask,
                                  const unsigned char *squash_kind, const unsigned *report_off,
                                  const unsigned *reports, const unsigned *eod_off, const unsigned *eod_reports,
                                  void *out, size_t cap);

/* Test hook: pure-literal block database whose literal programs are raw
 * instruction bytes (layouts: src/rose/rose_program.h:214-724).  `area` is
 * placed at bytecode offset hs_b200_test_program_base(); prog_off[i] = offset of
 * literal i's program inside `area` (8-byte aligned).  Lets the tests reach every
 * opcode of roseRunProgram_l (src/rose/program_runtime.c:3101-3522) on the device
 * and on the unmodified reference runtime from the same bytes. */
unsigned hs_b200_test_program_base(void);
hs_error_t hs_b200_test_compile_programs(const char *const *lits, const size_t *lens,
                                         const unsigned *nocase, const unsigned *prog_off,
                                         unsigned n, const void *area, size_t area_len,
                                         unsigned ekey_count, const unsigned *inv_dkey,
                                         unsigned dkey_count, hs_database_t **db);

/* Device binding.  A scratch owns CUDA streams, events, the match-record ring and
 * the device images of its databases on the CUDA device that was current when
 * hs_alloc_scratch created it (hs_clone_scratch: the source's device); corpus handles and
 * stream sets name their device explicitly.  Like the reference (src/hs_runtime.h:530-541:
 * any thread may use any scratch, one scan at a time), every entry point switches to
 * the object's device for the duration of the call and restores the caller's current
 * device, so a thread whose current device differs -- e.g. a fresh thread, device 0 --
 * can scan with a scratch that lives on another GPU. */

/* Runtime tunables (process-wide; also HSB200_* environment variables): the scan
 * geometry -- "warps" per CTA (0 = 28), "tile_bytes", "pf_dist" (L2 prefetch
 * distance, -1 = the kernel's own), "chunk_mb" (host->device pipeline granularity),
 * "initial_ring" (match records) -- and switches that force either side of a choice
 * the library makes from the database: "gram" (class 4-gram first stage for FDR sets:
 * 0 never, 1 from 10 000 prefilter keys, 2 whenever all literals have 4 bytes),
 * "heavy" (class-pair candidate path: per-word queue entries 0 never / 1 and 2
 * always) and "dfa_ilp" (DFA kernels: blocks per lane, 1).  "gram" applies to
 * scratches allocated afterwards.  The defaults are the measured best (DESIGN.md
 * section 3); the others exist for A/B runs (tools/sweep.py) and tests.  Any other
 * key: HS_INVALID. */
hs_error_t hs_b200_set_runtime_option(const char *key, int value);

/* Counters of the last finished scan: [0] raw records, [1] error, [2]
 * first-stage candidates, [3] byte-confirmed literals, [4] candidates that
 * passed the prefilter. */
hs_error_t hs_b200_last_counters(const hs_scratch_t *scratch, unsigned int out[8]);

/* Number of kernel launches issued by this library since load (bench.py's
 * "gpu_launches"), and elapsed device time of the last scan kernel in ms
 * (CUDA events on the launching stream). */
unsigned long long hs_b200_launch_count(void);
float hs_b200_last_kernel_ms(const hs_scratch_t *scratch);

#ifdef __cplusplus
}
#endif
#endif /* HS_B200_H */
