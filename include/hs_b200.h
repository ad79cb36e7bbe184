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
/* HS_FLAG_UTF8: the expression is UTF-8 (validated; "Expression is not valid UTF-8." otherwise) and its
 * characters are code points, matched as their 1- to 4-byte encodings ("." and negated classes match whole
 * encoded characters); \w \d \s, POSIX classes and \b keep their ASCII meaning; widths and offsets count
 * bytes.  Refused: \p / \P, \X, and HS_FLAG_CASELESS on a non-ASCII character (DESIGN.md section 10b).
 * HS_FLAG_UCP: refused wherever it could change the meaning (it needs the Unicode property tables); a finite
 * set of ASCII literals compiles as without it. */
#define HS_FLAG_UTF8 32
#define HS_FLAG_UCP 64
/* HS_FLAG_PREFILTER: the expression is rewritten into one whose matches are a superset of its own, to be
 * confirmed by the application (with PCRE, say): a back-reference becomes a copy of its group when that group is
 * one character position (caseless where the reference is), else any byte sequence; look-around becomes nothing; atomic groups, possessive quantifiers and
 * conditional groups become their plain forms; an expression whose automaton would be too large has its bounded
 * repeats widened, then its min_length dropped, until it fits.  An expression with none of these compiles to the
 * same database as without the flag.  Refused with HS_FLAG_SOM_LEFTMOST, in a combination's sub-expression and
 * by hs_compile_lit* (DESIGN.md section 10b, "Prefilter mode"). */
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
 * Expressions in UTF-8 mode (HS_FLAG_UTF8) take either route.
 * Anything else (look-around, back-references without HS_FLAG_PREFILTER, UCP, ...) yields
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

/* The report rules on the device: the same delivered matches as hs_b200_fetch_matches /
 * hs_b200_postprocess_matches -- same records, same (block, to, id) order, same count -- computed by
 * kernels and written to device memory, enqueued on a CUDA stream with no host synchronisation.
 * Every database shape the device scans is taken (pure literal, single outfix, literals beside an
 * outfix); a database with logical combinations is refused (HS_INVALID), as are NULL arguments
 * (d_out may be NULL only with cap = 0) and a scratch that holds no image of `db` (one that was not
 * allocated for it).  Temporaries live in the scratch, which must not be used by another call
 * until the ordering has been enqueued. */
#define HS_B200_ORDER_RING_OVERFLOW (~0ULL)
/* Enqueue, on cuda_stream (the one the scan was enqueued on; NULL = the scratch's stream), the
 * delivery of the last scan enqueued with hs_b200_scan_corpus_async: the matches
 * hs_b200_fetch_matches would return, written to d_out[0, cap) (hs_b200_match_t[]) and their count
 * to *d_count (an unsigned long long in device memory; it may exceed cap, and then only the first
 * cap are written).  If the scan's record ring overflowed, *d_count = HS_B200_ORDER_RING_OVERFLOW:
 * hs_b200_scan_corpus_finish then returns HS_INSUFFICIENT_SPACE and grows the ring as it does
 * for every overflow, and the caller scans again. */
hs_error_t hs_b200_order_matches_async(const hs_database_t *db, hs_scratch_t *scratch,
                                       void *d_out, size_t cap, void *d_count, void *cuda_stream);
/* The same for n raw records already in device memory (e.g. the all-gathered records of several
 * ranks, block indices already global): what the host report rules make of them
 * (hs_b200_postprocess_matches for a pure-literal database; for a database with an engine, whose
 * records carry report programs, the delivery hs_b200_fetch_matches applies).  Records whose id
 * names no report program of the engine are dropped. */
hs_error_t hs_b200_order_records_async(const hs_database_t *db, hs_scratch_t *scratch,
                                       const void *d_recs, size_t n, void *d_out, size_t cap,
                                       void *d_count, void *cuda_stream);

/* Scan a column of rows that is already in device memory, such as a torch jagged tensor or an Arrow large_string
 * column: row i is d_chars[d_offsets[i], d_offsets[i + 1]), with nrows + 1 offsets in device memory (8-byte
 * aligned); d_offsets[0] may be above 0, and neither d_chars nor any row needs an alignment.  The pass is enqueued
 * on cuda_stream (NULL = the scratch's stream) and returns without a host wait: the device checks the offsets,
 * packs the rows into staging memory of the scratch (grown in the call) and scans them, for every database shape
 * hs_b200_scan_corpus_async takes.  Nothing outside [d_chars, d_chars + chars_bytes) and the offsets is read, and
 * neither is written; both stay valid until the pass completes.  d_chars may be NULL when chars_bytes is 0.
 * The records go into the scratch's ring as for hs_b200_scan_corpus_async (block = row index, to = end offset
 * within the row), and hs_b200_scan_corpus_finish, hs_b200_fetch_matches, hs_b200_export_records_async and
 * hs_b200_order_matches_async serve the pass: the delivered matches equal hs_b200_scan_blocks_collect's over the
 * same rows from host memory.  A ring overflow is as for a corpus scan: finish returns HS_INSUFFICIENT_SPACE and
 * grows the ring, and the caller enqueues the pass again.  A row table that decreases, ends past chars_bytes or
 * holds a row of 4 GiB or more fails the pass: no records, the ordering reports HS_B200_ORDER_RING_OVERFLOW and
 * finish returns HS_INVALID; the next pass is unaffected.  Refused at once: HS_INVALID for NULL arguments,
 * misaligned offsets, nrows above 0xfffffff0, a scratch that holds no image of `db` and a database with logical
 * combinations (their reports need the row lengths on the host); HS_DB_MODE_ERROR for a database not in block
 * mode; HS_ARCH_ERROR for a scratch with a peer exchange registered. */
hs_error_t hs_b200_scan_rows_async(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                                   const unsigned long long *d_offsets, size_t nrows, hs_scratch_t *scratch,
                                   void *cuda_stream);

/* Match masks: which report ids fire in which block, as a bit matrix of fixed size in device memory instead of
 * match records -- the answer a filter or a tagger needs, with no record ring to overflow and nothing to order.
 *
 * The report ids a database can deliver, ascending and distinct: column r of a match mask is ids[r].  *count
 * receives their number; ids may be NULL with cap 0 to query it (HS_INSUFFICIENT_SPACE: cap below *count, nothing
 * written).  Host only (needs no CUDA device); every database shape the device scans is taken, and for a database
 * with logical combinations the list holds the combinations' ids too. */
hs_error_t hs_b200_report_ids(const hs_database_t *db, unsigned int *ids, size_t cap, size_t *count);
/* The same pass as hs_b200_scan_corpus_async / hs_b200_scan_rows_async, but instead of match records it writes
 * d_mask: nblocks rows of words_per_block 32-bit words (device memory, 4-byte aligned; NULL only when there are no
 * blocks).  Bit r of row b (word
 * r / 32, bit r % 32) is set iff hs_scan of block b would deliver at least one match with id ids[r] -- equivalently,
 * iff hs_b200_fetch_matches after the ordinary pass holds a record (b, *, ids[r]).  The pass writes every word of
 * the mask, zeroes included; words_per_block >= ceil(count / 32), with ids and count as hs_b200_report_ids gives
 * them.  d_status (optional, a device u32): 0 when the mask is valid, non-zero when the pass must be enqueued again
 * after hs_b200_scan_corpus_finish (candidate-list overflow: HS_INSUFFICIENT_SPACE, list grown; bad row table:
 * HS_INVALID), so that a pipeline can test it on the device with no host wait.  The pass is enqueued on
 * cuda_stream (NULL = the scratch's stream) and returns at once; d_mask and d_status stay valid until it completes.
 * A mask pass writes no records: after it, hs_b200_scan_corpus_finish reports 0 records (or the overflow above),
 * hs_b200_fetch_matches delivers none, hs_b200_order_matches_async writes a count of 0 (HS_B200_ORDER_RING_OVERFLOW
 * after an overflow) and hs_b200_export_records_async a count of 0.  Refused at once, as the ordinary calls refuse
 * them: HS_INVALID for NULL or misaligned arguments, a scratch that holds no image of `db`, words_per_block too
 * small and a database with logical combinations (their reports depend on the order within a block);
 * HS_DB_MODE_ERROR for a database not in block mode; HS_ARCH_ERROR for a scratch with a peer exchange registered. */
hs_error_t hs_b200_scan_corpus_mask_async(const hs_database_t *db, const hs_b200_corpus_t *corpus,
                                          hs_scratch_t *scratch, void *d_mask, size_t words_per_block,
                                          void *d_status, void *cuda_stream);
hs_error_t hs_b200_scan_rows_mask_async(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                                        const unsigned long long *d_offsets, size_t nrows,
                                        hs_scratch_t *scratch, void *d_mask, size_t words_per_block,
                                        void *d_status, void *cuda_stream);
/* First-match passes: the passes of hs_b200_scan_corpus_async / hs_b200_scan_rows_async, but instead of match records
 * they write one entry per block (per row) to d_first (nblocks or nrows unsigned long longs, device memory, 8-byte
 * aligned; NULL only when there are no blocks).  Entry b is ((to << 32) | id) of the first match that
 * hs_b200_fetch_matches would deliver for block b after the ordinary pass, in its (block, to, id) order -- the match
 * hs_scan of block b passes to a callback that returns non-zero on its first call -- or ~0ULL when block b delivers
 * nothing.  `to` is relative to the block (the row).  Every entry is written.  The entry is exact under dedupe,
 * HS_FLAG_SINGLEMATCH, min_offset / max_offset and min_length: a match competes only after the checks that decide
 * its delivery.  The engine walks stop once nothing they can still find would come first, so a block with many
 * matches costs about as much as one whose first match is as early.  d_status (optional, a device u32) is 0 when the
 * table is valid and 1 when hs_b200_scan_corpus_finish asks for the pass again (a candidate-list overflow:
 * HS_INSUFFICIENT_SPACE, list grown; a bad row table: HS_INVALID).  No records are written: finish reports 0
 * records, and fetch, export and both orderings serve 0.  Refused at once, as the mask passes refuse: HS_INVALID for
 * NULL or misaligned arguments, a scratch that holds no image of `db` and a database with logical combinations;
 * HS_DB_MODE_ERROR for a database not in block mode; HS_ARCH_ERROR for a scratch with a peer exchange registered. */
hs_error_t hs_b200_scan_corpus_first_async(const hs_database_t *db, const hs_b200_corpus_t *corpus,
                                           hs_scratch_t *scratch, void *d_first, void *d_status, void *cuda_stream);
hs_error_t hs_b200_scan_rows_first_async(const hs_database_t *db, const void *d_chars, size_t chars_bytes,
                                         const unsigned long long *d_offsets, size_t nrows, hs_scratch_t *scratch,
                                         void *d_first, void *d_status, void *cuda_stream);

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
/* A pass over writes that are already in device memory, enqueued on cuda_stream (NULL = the scratch's
 * stream) with no host wait.  Stream i's write is at d_writes + i * pitch + 16, d_lengths[i] bytes long
 * (device memory), or uniform_length bytes when d_lengths is NULL; length 0 = no write.  d_writes is
 * 16-byte aligned, pitch a multiple of 16 and at least 32, every length at most pitch - 16.  The 16 bytes
 * in front of each write belong to the library during the pass (the stream's look-behind is written
 * there); the bytes after a write may hold anything and take part in no match.  Nothing outside
 * [d_writes, d_writes + nstreams * pitch) is read or written.  d_writes and d_lengths stay valid until the
 * pass completes, and all passes of one set go on one CUDA stream.
 * The records go into the scratch's ring as for hs_b200_scan_corpus_async (block = stream index, to =
 * stream offset), and hs_b200_scan_corpus_finish, hs_b200_fetch_matches, hs_b200_export_records_async and
 * hs_b200_order_matches_async serve the pass; the ordered matches equal hs_b200_streams_scan_collect's.
 * The streams advance on the device, and only when the pass's ring and candidate list did not overflow.
 * Otherwise the streams stay as they were and the set is marked: every later pass on it commits nothing
 * and its ordering reports HS_B200_ORDER_RING_OVERFLOW, and every later hs_b200_streams_reset_async on it
 * commits nothing either, until hs_b200_scan_corpus_finish returns HS_INSUFFICIENT_SPACE and grows the ring
 * (the set must still be open).  The passes and resets enqueued before that call stay without effect; those
 * enqueued after it commit.  The caller then enqueues again, in their order, the passes and resets from the
 * first pass whose ordering reported the overflow on.  A device length above pitch - 16 fails the pass in
 * the same way, and finish returns HS_INVALID.  HS_INVALID at once: NULL arguments, a misaligned buffer, a
 * bad pitch, a uniform length above pitch - 16, a scratch on another device than the set. */
hs_error_t hs_b200_streams_scan_async(hs_b200_stream_set_t *set, void *d_writes, size_t pitch,
                                      const unsigned int *d_lengths, unsigned int uniform_length,
                                      hs_scratch_t *scratch, void *cuda_stream);
/* A pass over a batch of writes as traffic arrives: rows in device memory, each tagged with its stream, in
 * arrival order.  Row r is d_chars[d_offsets[r], d_offsets[r + 1]) (the layout of hs_b200_scan_rows_async: nrows + 1
 * offsets in device memory, 8-byte aligned, d_offsets[0] may be above 0, no row needs an alignment) and is written
 * to stream d_stream_ids[r] (nrows ids in device memory).  The pass is equivalent to hs_scan_stream of row r on
 * stream d_stream_ids[r] for r = 0 .. nrows - 1 in order: a stream may receive any number of rows anywhere in the
 * batch, a match may span its rows, an empty row is a write of nothing, and the streams the batch does not name
 * are neither read nor written.  Enqueued on cuda_stream (NULL = the scratch's stream) with no host wait; the
 * device groups the rows by stream and packs them into staging memory of the scratch (grown in the call).  Nothing
 * outside [d_chars, d_chars + chars_bytes), the offsets and the ids is read, and none of them is written; they stay
 * valid until the pass completes.  d_chars may be NULL when chars_bytes is 0, d_stream_ids when nrows is 0.
 * The records go into the scratch's ring with block = the row that holds the match's last byte and to = the stream
 * offset of the match's end; ordered by (block, to, id) they are the callbacks of the loop above, in order.
 * hs_b200_scan_corpus_finish, hs_b200_fetch_matches, hs_b200_export_records_async and
 * hs_b200_order_matches_async serve the pass, with nrows blocks.  Commit, mark and epoch are those of
 * hs_b200_streams_scan_async, and passes of both kinds and hs_b200_streams_reset_async mix freely on one set, on
 * one CUDA stream.  A bad batch fails the pass as a bad length does there (no records, the streams stay, the
 * ordering reports HS_B200_ORDER_RING_OVERFLOW, finish returns HS_INVALID): offsets that decrease or end past
 * chars_bytes, a stream id at or above the set's stream count, or one stream receiving 4 GiB minus its
 * look-behind or more in the batch.  A batch of no rows scans nothing and delivers no records, but takes the set's
 * verdict like any pass: behind a pass that overflowed or was bad in the same epoch, its ordering reports
 * HS_B200_ORDER_RING_OVERFLOW and finish returns that outcome (HS_INSUFFICIENT_SPACE, HS_INVALID).
 * HS_INVALID at once: NULL arguments, misaligned offsets or ids, nrows above 0xfffffff0, a scratch on another
 * device than the set or holding no image of the set's database; HS_ARCH_ERROR for a scratch with a peer
 * exchange registered. */
hs_error_t hs_b200_streams_scan_rows_async(hs_b200_stream_set_t *set, const void *d_chars, size_t chars_bytes,
                                           const unsigned long long *d_offsets, const unsigned int *d_stream_ids,
                                           size_t nrows, hs_scratch_t *scratch, void *cuda_stream);
/* Stream-set passes into a match mask: the same passes as hs_b200_streams_scan_async and
 * hs_b200_streams_scan_rows_async, but instead of match records they write d_mask, as hs_b200_scan_corpus_mask_async
 * does (words_per_block >= ceil(count / 32) with count from hs_b200_report_ids, device memory, 4-byte aligned).  A
 * mask row is the block the ordinary pass's records carry: nstreams rows for the pitched pass (row = stream index),
 * nrows rows for the pass over rows (row = the batch row that holds the match's last byte).  Bit r of row b is set
 * iff the ordinary pass, ordered by hs_b200_order_matches_async, delivers a match with block b and id ids[r]; every
 * word is written, spare words included.  Otherwise the pass is the ordinary one: the look-behind and offsets
 * advance as they would, commit, mark and epoch are those of hs_b200_streams_scan_async, and mask passes, record
 * passes and hs_b200_streams_reset_async mix freely on one set and one CUDA stream.  For a flow tagger the answer
 * of a tick is then of fixed size, needs no ordering, and a dense tick cannot overflow the record ring and mark the
 * set.  (Masks of successive passes may be ORed by the caller to cover a flow's lifetime.)
 * d_status (optional, a device u32) is 0 when the pass committed and 1 when it did not: a candidate-list overflow
 * (finish: HS_INSUFFICIENT_SPACE, list grown), a bad length or batch (finish: HS_INVALID), or a set marked earlier
 * in the epoch (finish returns that epoch's outcome).  hs_b200_scan_corpus_finish returns what it returns for the
 * ordinary pass, and the caller enqueues the passes and resets again from the first one that did not commit.  No
 * records are written: finish reports 0 records (or the overflow), and fetch, export and both orderings serve 0.
 * Refused at once: what the ordinary calls refuse, with the same codes, and HS_INVALID for words_per_block too
 * small, a NULL d_mask when the pass has mask rows and a misaligned d_mask or d_status; HS_ARCH_ERROR for a
 * scratch with a peer exchange registered. */
hs_error_t hs_b200_streams_scan_mask_async(hs_b200_stream_set_t *set, void *d_writes, size_t pitch,
                                           const unsigned int *d_lengths, unsigned int uniform_length,
                                           hs_scratch_t *scratch, void *d_mask, size_t words_per_block,
                                           void *d_status, void *cuda_stream);
hs_error_t hs_b200_streams_scan_rows_mask_async(hs_b200_stream_set_t *set, const void *d_chars, size_t chars_bytes,
                                                const unsigned long long *d_offsets, const unsigned int *d_stream_ids,
                                                size_t nrows, hs_scratch_t *scratch, void *d_mask,
                                                size_t words_per_block, void *d_status, void *cuda_stream);
/* End the flows of the `count` streams listed in d_streams (device memory; NULL = every stream): their
 * look-behind becomes empty and their offset 0, in stream order on cuda_stream.  Indices at or above
 * nstreams are ignored.  Nothing is delivered: a pure-literal stream database has no end-of-data reports.
 * On a marked set (see hs_b200_streams_scan_async) the reset commits nothing and is enqueued again with the
 * passes.  cuda_stream is the stream the set's passes run on: NULL here is the legacy default stream, which
 * does not order against the scratch's own stream (what hs_b200_streams_scan_async takes for NULL).  Before
 * a hs_b200_streams_scan, the caller synchronises cuda_stream. */
hs_error_t hs_b200_streams_reset_async(hs_b200_stream_set_t *set, const unsigned int *d_streams, size_t count,
                                       void *cuda_stream);
size_t hs_b200_streams_state_bytes(const hs_b200_stream_set_t *set);
/* The set's state, copied to host memory once every pass and reset enqueued on it has run (the call synchronises
 * the device): 8 bytes per stream into look_behind (the look-behind bytes, oldest first, and their count in byte 7)
 * and the 64-bit stream offsets into offsets, nstreams of each; either may be NULL.  For tests and diagnostics. */
hs_error_t hs_b200_streams_read_state(const hs_b200_stream_set_t *set, unsigned char *look_behind,
                                      unsigned long long *offsets);
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
    unsigned int engine_count;   /* engines run as outfixes (RoseEngine.queueCount): 0 for a pure-literal database,
                                  * 1 beside or without a literal matcher, K for a set split over K engines */
} hs_b200_db_info_t;
/* HS_INVALID also for a database of several outfixes whose queue table, state scatter plan or EOD iterator
 * does not fit its engine count or its bytecode (such a database is refused at scratch allocation too). */
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
 * always), "dfa_ilp" (DFA kernels: blocks per lane, 1) and "engine_segment"
 * (engine runs of regular-expression databases and hs_b200_nfa_scan_corpus: 0 = cut
 * blocks longer than twice the segment length into segments walked by lanes of their
 * own when the blocks, times the engines of the run, leave more than half of the
 * resident lanes idle; N > 0 = cut every block longer than N bytes into N-byte
 * segments, and a scan whose segment area (engines x segments x two states, with the
 * plan) would pass 1 GiB fails with HS_NOMEM; -1 = never cut, one lane per block.  The
 * matches are the same in every setting; DESIGN.md section 10f).
 * "gram" applies to scratches allocated afterwards.  The defaults are the measured
 * best (DESIGN.md section 3); the others exist for A/B runs (tools/sweep.py) and tests.
 * Any other key: HS_INVALID. */
hs_error_t hs_b200_set_runtime_option(const char *key, int value);

/* What the segmented engine runs on this scratch have done since it was allocated:
 * out[0] engine runs that cut blocks, out[1] segments they walked, out[2] segments
 * re-walked because the start state guessed for them was wrong, out[3] bytes of those
 * re-walks, each counted up to the 16-byte piece where it met the walk from the guess.
 * The segments of a run over rows scanned by hs_b200_scan_rows_async are its segment table's size, which
 * the host bounds from the row count and the chars' size: at least the segments walked.
 * Waits for the scratch's stream. */
hs_error_t hs_b200_engine_segment_stats(const hs_scratch_t *scratch, unsigned long long out[4]);

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
