/*
 * sdbgpu.h -- C ABI of the H100-native KNN / HNSW / graph-expansion engine.
 *
 * This is the drop-in boundary for SurrealDB's vector-similarity and graph-scan hot path
 * (SURVEY.md section 8b).  The reference has NO FFI of its own (pure Rust, SURVEY F4/F5), so each
 * entry point below names the Rust-internal seam it replaces; INTEGRATION.md shows the
 * `extern "C"` block and the operator wrappers a maintainer adds behind a `gpu-knn` cargo feature.
 * Paths are relative to surrealdb/core/src in the reference checkout.
 *
 * Conventions
 *  - plain pointers and sizes only; no C++/torch types cross the boundary.
 *  - every function is thread-safe per handle family: concurrent searches on one corpus/hnsw/graph
 *    handle are serialised internally (one in-flight search per handle); mutation
 *    (append/finalize) must not race with searches -- the same RW discipline the reference applies
 *    to its HNSW graph (idx/trees/hnsw/index.rs:55,224,350).
 *  - errors: integer status + thread-local message (sdb_last_error); nothing unwinds across the ABI.
 *  - "rows" are scan positions: the caller appends vectors in the reference's scan order (record-key
 *    byte order, i.e. what TableScan yields) and maps returned row numbers back to RecordIds.
 *  - NO CPU FALLBACK: if no CUDA device is usable every entry point fails with SDB_ECUDA.
 */
#ifndef SDBGPU_H
#define SDBGPU_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sdb_ctx sdb_ctx;       /* one CUDA device: streams, scratch, TMA driver entry points   */
typedef struct sdb_corpus sdb_corpus; /* device-resident N x D vector column (+ norms, screen copy)    */
typedef struct sdb_hnsw sdb_hnsw;     /* device-resident HNSW layers (CSR) + element vectors           */
typedef struct sdb_graph sdb_graph;   /* device-resident CSR adjacency of one (direction, edge table)  */

typedef enum {
  SDB_OK = 0,
  SDB_EINVAL = 1,     /* bad argument                                                               */
  SDB_EDIM = 2,       /* dimension mismatch -> Error::InvalidVectorDimension (idx/trees/vector.rs:643) */
  SDB_ENOMEM = 3,
  SDB_ECUDA = 4,      /* CUDA runtime/driver failure, or no sm_90 device                            */
  SDB_ECANCELLED = 5, /* cancel flag observed -> Error::QueryCancelled (exec/operators/knn_topk.rs:186) */
  SDB_EUNSUPPORTED = 6,
  SDB_EOVERFLOW = 7,  /* caller-provided output capacity too small / too many batches in flight      */
  SDB_ENCCL = 8       /* NCCL failure (multi-GPU entry points)                                      */
} sdb_status;

/* catalog::Distance (catalog/schema/index.rs:247-284).  COSINE and EUCLIDEAN are screened on the tensor cores and
 * re-ranked exactly; PEARSON is screened on the tensor cores as the cosine of the rows and the query centred on their
 * own means, and re-ranked exactly; MANHATTAN and CHEBYSHEV are screened by the f32 L1 / L-infinity SIMT screen
 * (SDB_SCREEN_SIMT_F32) and re-ranked exactly, and so is MINKOWSKI of an integer order 1 .. 8 (f32 Lp screen);
 * HAMMING and JACCARD (k <= 256) are ranked by exact counts of every row, batched over the queries (the count path,
 * no screen and no proof: mismatches for HAMMING, distinct and shared values for JACCARD); MINKOWSKI of any other
 * order and HAMMING / JACCARD with k > 256 run through the exact kernel (sequential f64, Distance::compute op for op). */
typedef enum {
  SDB_CHEBYSHEV = 0,
  SDB_COSINE = 1,
  SDB_EUCLIDEAN = 2,
  SDB_HAMMING = 3,
  SDB_JACCARD = 4,
  SDB_MANHATTAN = 5,
  SDB_MINKOWSKI = 6,
  SDB_PEARSON = 7
} sdb_metric;

/* element type of the rows handed to sdb_corpus_append (catalog VectorType, index.rs:321-334).
 * Brute-force KnnTopK holds Vec<Number>: F64 covers arbitrary Number::Float rows, F32 covers rows whose
 * values are f32-representable (the BASELINE configs).  COSINE / EUCLIDEAN corpora of either type are screened on the
 * tensor cores (F64: when the bf16 / int8 copies, 3 bytes per element, fit beside the rows at creation; otherwise the
 * corpus is ranked by the exact kernel alone).  The f32 SIMT screen of COSINE / EUCLIDEAN needs F32 rows: on F64 it
 * means the exact kernel.  MANHATTAN / CHEBYSHEV corpora of either type are screened by the f32 L1 / L-infinity screen
 * (f64 rows rounded to f32 as the screen reads them; rows with an element beyond f32 range are ranked exactly), and
 * MINKOWSKI corpora of an integer order 1 .. 8 by the f32 Lp screen in the same way.
 * HAMMING corpora of either type take the count path: f64 rows are compared on all 64 bits, f32 rows as the exact
 * kernel widens them to f64; no row is special (zero, NaN and +-inf are ordinary values for equality).  JACCARD
 * corpora take it the same way when their first-occurrence state (one bit per element and 4 bytes per row) fits
 * beside the rows at creation; otherwise the exact kernel ranks them.
 * PEARSON corpora of either type are screened on the tensor cores when the bf16 / int8 copies of the centred rows and
 * 16 bytes of moments per row fit beside the rows at creation; otherwise the exact kernel ranks them. */
typedef enum { SDB_F32 = 0, SDB_F64 = 1 } sdb_dtype;

/* element type of an HNSW index: catalog::VectorType (catalog/schema/index.rs:321-335), numbered as the SerializedVector
 * variants (idx/trees/vector.rs:34-40).  An index of type T holds, and its searches take, vectors of T: double, float,
 * int64_t, int32_t, int16_t. */
typedef enum { SDB_VT_F64 = 0, SDB_VT_F32 = 1, SDB_VT_I64 = 2, SDB_VT_I32 = 3, SDB_VT_I16 = 4 } sdb_vector_type;

/* which screening kernel sdb_knn_bruteforce uses (results are identical for all; this only moves the performance
 * point).  AUTO: cosine corpora whose normalised rows quantise well (largest relative int8 error <= 0.02 once the few
 * outlier rows are set aside) start on the int8 tensor-core screen, everything else on the bf16 one; queries whose
 * proof fails climb to finer screens (bf16, then the f32 stream) before the exact kernel.  MANHATTAN / CHEBYSHEV corpora
 * (k <= 256) are screened by SDB_SCREEN_SIMT_F32 for AUTO and every TC request (4096, then 16384 candidates per query,
 * then the exact kernel), except that AUTO ranks a batch of one query with the exact kernel (faster for a single query);
 * NONE_EXACT keeps them on the exact kernel.  MINKOWSKI corpora of an integer order 1 .. 8 take the same ladder, a
 * single query included (their exact kernel is bound by a pow() per element); other orders keep the exact kernel.
 * HAMMING corpora (1 <= k <= 256) take the count path for AUTO and every screen request but NONE_EXACT, which keeps the
 * exact kernel, except that AUTO ranks a batch of one query with the exact kernel (faster for a single query);
 * JACCARD corpora with their first-occurrence state take the same path, a single query included (their exact kernel
 * is O(D^2) per row); sdb_knn_last_stats reports it as screen_used = SDB_SCREEN_SIMT_F32, n_passes = 1, n_fallback = 0.  PEARSON corpora (k <= 256) follow the cosine ladder on the centred rows
 * (int8, then bf16, then the exact kernel; no f32 stream): SIMT_F32 and NONE_EXACT mean the exact kernel. */
typedef enum {
  SDB_SCREEN_AUTO = 0,
  SDB_SCREEN_SIMT_F32 = 1,   /* f32 SIMT screen: streaming dot products; MANHATTAN / CHEBYSHEV / MINKOWSKI: Lp;
                                HAMMING / JACCARD: the count path                                           */
  SDB_SCREEN_TC_BF16 = 2,    /* wgmma bf16 operands, f32 accumulation                                    */
  SDB_SCREEN_NONE_EXACT = 3, /* no screen: exact f64 kernel for every query                              */
  SDB_SCREEN_TC_INT8 = 4     /* wgmma s8, int8 copy of the normalised (pearson: centred) rows; falls back to bf16 */
} sdb_screen;

/* counters of the last brute-force call on a corpus (diagnostics / bench roofline arithmetic) */
typedef struct {
  uint32_t screen_used;      /* sdb_screen actually run                                        */
  uint32_t n_passes;         /* threshold-refinement passes of the screen                      */
  uint32_t n_fallback;       /* queries re-run through the exact kernel (verification failed)  */
  uint32_t n_special_rows;   /* rows with zero / non-finite norm (always exact-ranked)         */
  uint64_t n_candidates;     /* largest candidate set of any query that reached the exact re-rank */
  uint64_t n_reranked;       /* exact f64 distances computed by the re-rank kernel             */
  uint64_t kernel_launches;  /* kernels launched by this call                                  */
  float screen_ms;           /* device time of the screening kernels (CUDA events)             */
  float total_ms;            /* device time of the whole call                                  */
  uint64_t n_survivors;      /* screened rows that passed a threshold and were gathered (all queries) */
  uint32_t n_repaired;       /* queries whose proof failed on the batch's screen and succeeded on a finer one
                                (re-screened as a small batch of their own; never reached the exact kernel) */
  uint32_t reserved0;
} sdb_knn_stats;

/* ---- context -------------------------------------------------------------------------------- */
sdb_status sdb_ctx_create(int device, sdb_ctx** out);
void sdb_ctx_destroy(sdb_ctx*);
const char* sdb_last_error(void); /* thread-local; valid until the next call on this thread */
const char* sdb_version(void);
void* sdb_pinned_alloc(size_t bytes); /* cudaHostAlloc: staging buffers for append / queries */
void sdb_pinned_free(void*);
/* Cancellation of whatever runs on this context, from any thread: the counterpart of the reference's ctx.is_done()
 * polls (exec/operators/knn_topk.rs:186, idx/trees/hnsw/index.rs:437, hnsw/layer.rs:533).  Brute force polls between
 * kernel phases and before every exact fallback, the HNSW walk before every query (inside the kernel), graph expansion
 * before every hop / BFS level.  A cancelled call returns SDB_ECANCELLED and its outputs are undefined.  The flag stays
 * up until sdb_ctx_cancel_reset.  (sdb_knn_bruteforce additionally takes a per-call flag.) */
void sdb_ctx_cancel(sdb_ctx*);
void sdb_ctx_cancel_reset(sdb_ctx*);
/* total kernels launched through this context since creation (bench's gpu_launches) */
/* Host-only diagnostic (needs no GPU): the sequence of corpus tiles (256 rows each) the screen of one batch visits --
 * the streaming schedule's main launch (its probe tiles are returned separately) or, with streaming = 0, the passes of
 * the multi-pass schedule.  No reference seam; exists so that "every tile is screened exactly once" can be tested on
 * the CPU for any corpus size.  out_tiles / out_probe_tiles may be NULL (counts only). */
sdb_status sdb_debug_schedule(uint64_t n_rows, uint32_t cand_cap, uint32_t k, uint32_t nq, int streaming,
                              uint32_t* out_tiles, uint64_t cap_tiles, uint64_t* out_n, uint32_t* out_probe_tiles,
                              uint32_t cap_probe, uint32_t* out_n_probe);
/* Test-only diagnostics of the brute-force screens (no reference seam): the state the exactness proof rests on, so that
 * tests can compare every intermediate with a plain reference.  Every output may be NULL.
 * sdb_debug_corpus_state, on a finalized F32 corpus, an F64 one that has screen copies, or an F64 MANHATTAN /
 * CHEBYSHEV / MINKOWSKI one (n_pad = rows rounded up to 256):
 *   out_f[4]    i8_scale, max_rel_qerr, bf16_rel_err, max_norm (MANHATTAN: the largest sum_i |x^_i| of a screened
 *               row; CHEBYSHEV and MINKOWSKI of any order: the largest |x^_i|)
 *   out_u[5]    n_special, n_outliers, dim_pad, dim_pad8, n_pad
 *   out_i8      [n_pad][dim_pad8] int8 copy of the normalised rows (cosine corpora; PEARSON: of dx / |dx|)
 *   out_bf16    [n_pad][dim_pad] bf16 copy (bit patterns; PEARSON: of the centred rows dx = x - mean(x))
 *   out_snorm   [n_pad] screening norm (cosine 1/|x|, euclidean |x|^2, pearson 1/|dx|; NaN: never a screen candidate)
 *   out_special [n_special] rows ranked exactly on every query
 * PEARSON corpora qualify when they hold their screen copies. */
sdb_status sdb_debug_corpus_state(sdb_corpus*, float* out_f, uint32_t* out_u, int8_t* out_i8, uint16_t* out_bf16,
                                  float* out_snorm, uint32_t* out_special);
/* sdb_debug_screen_batch: one batch of nq host queries screened with `screen` (TC_INT8, TC_BF16 or SIMT_F32) at the
 * first rung of the ladder, through the production sequence (streaming = 0: the multi-pass schedule), with exactly
 * cand_cap (>= 4096) candidate slots per query (F64 corpora with screen copies: TC_INT8 or TC_BF16 only; MANHATTAN / CHEBYSHEV corpora, F32 or F64: SIMT_F32, where
 * beps bounds |s~ - d| and the score is -s~; MINKOWSKI corpora of an integer order 1 .. 8, F32 or F64: SIMT_F32, where
 * the score is the f32 norm -n~ of the batch's scaled power sum and beps bounds |n~ - d|; PEARSON corpora with screen copies, F32 or F64: TC_INT8 or TC_BF16, where
 * the scores are those of the unit query -dq/|dq| against dx, qmag is 1 and the proof adds eps_ref).  The ladder
 * and the exact fallback do not run: flags are as the batch
 * left them.  score_all != 0 instead runs one pass-0 launch over every tile (SIMT: tau = -inf) with max(cand_cap,
 * n_pad) slots and selects nothing: out_a then holds every score of that kernel, and out_b / out_rr are untouched.
 * Let cap be the slots per query.
 *   out_qf[nq][9]  tau, margin, bscale, beps, tau2, beps2, int8 query scale, int8 query residual, qbferr
 *                  (the int8 figures are NaN on euclidean corpora)
 *   out_qmag[nq]   |q| in the reference's f64 arithmetic
 *   out_qu[nq][6]  flags, qflags, entries the stage-A selections gathered before capping (the largest over the
 *                  batch's selections; score_all: the list's count), n_a, n_b, n_e
 *   out_q8[nq][dim_pad8], out_qbf16[nq][dim_pad]  the query's int8 and bf16 copies
 *   out_a[nq][cap][3]   stage-A kept list: row, screen score (f32 bits), the f32 re-score of stage B (f32 bits, NaN
 *                       when stage B did not run); entries past n_a are (0xFFFFFFFF, NaN, NaN)
 *   out_b[nq][cap][2]   stage-B kept list: row, score; past n_b (0xFFFFFFFF, NaN)
 *   out_rr[nq][cap + 1024]  rows of the exact re-rank (n_e: stage-B rows, then the special rows); past n_e 0xFFFFFFFF */
sdb_status sdb_debug_screen_batch(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k, sdb_screen screen,
                                  int streaming, uint32_t cand_cap, int score_all, float* out_qf, double* out_qmag,
                                  uint32_t* out_qu, int8_t* out_q8, uint16_t* out_qbf16, uint32_t* out_a,
                                  uint32_t* out_b, uint32_t* out_rr);
/* sdb_debug_screen_batch_filtered: the same batch with a row filter per query (filters, n_filters, query_filter as in
 * sdb_knn_bruteforce_filtered; sdb_debug_screen_batch is this call with filters = NULL).  The queries are classified as
 * sdb_knn_bruteforce_filtered classifies them (direct regime or screened, FiltArg mask_hits); mask_hits = -1 keeps that
 * rule's choice, 0 and 1 force the int8 consumers' hit-mask filtering off or on.  A batch that mixes direct and
 * screened queries returns SDB_EUNSUPPORTED (unless score_all).  What the lists hold with a filter:
 *   score_all   pass 0 with the filter: the tensor-core screens write every row and NaN the scores of the rows the
 *               query's filter rejects (cand_filter_list); SIMT_F32 never appends a rejected row
 *   out_b       the passing special rows follow the stage-B rows in the query's list (score +inf), so n_e = n_b and
 *               out_rr holds no special rows beyond them
 *   all-direct  no screen pass runs (n_passes = 0): out_a and out_b are the direct list (every passing row that is
 *               neither skipped nor removed, score +inf), tau is -inf and the gathered count is 0 */
sdb_status sdb_debug_screen_batch_filtered(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k,
                                           sdb_screen screen, int streaming, uint32_t cand_cap, int score_all,
                                           float* out_qf, double* out_qmag, uint32_t* out_qu, int8_t* out_q8,
                                           uint16_t* out_qbf16, uint32_t* out_a, uint32_t* out_b, uint32_t* out_rr,
                                           const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                           int mask_hits);
/* sdb_debug_screen_batch_ranked: sdb_debug_screen_batch_filtered for the ranking (fn, order) of sdb_corpus_order_topk
 * instead of KNN's; SDB_EINVAL for a ranking the screens do not serve on the corpus.  SDB_FN_DOT on a COSINE or
 * EUCLIDEAN corpus (TC_BF16, or SIMT_F32 on F32 rows): the scores are the dots of the rows with the query (DESC) or
 * with its negation (ASC), out_qbf16 is the bf16 copy of that query, bscale is 1 and beps bounds the score's
 * distance from the exact dot; the exact re-rank still ranks the query itself.  The cross views of a COSINE or
 * EUCLIDEAN corpus (cosine distance / similarity in the order KNN does not take, euclidean distance ASC on COSINE and
 * DESC on either): the scores, the query copy (q or -q), bscale and beps are the view's -- cosine acc/|x| in
 * similarity x |q| units, euclidean 2 acc - |x|^2 or farthest-first 2 acc + |x|^2 in squared-distance units -- and the
 * special rows of out_rr are the view's (the cross special list where the view reads the other metric's norm). */
sdb_status sdb_debug_screen_batch_ranked(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k,
                                         sdb_screen screen, int streaming, uint32_t cand_cap, int score_all,
                                         float* out_qf, double* out_qmag, uint32_t* out_qu, int8_t* out_q8,
                                         uint16_t* out_qbf16, uint32_t* out_a, uint32_t* out_b, uint32_t* out_rr,
                                         const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                         int mask_hits, int fn, int order);
/* Test-only: device and pinned buffers the library holds right now, process-wide (count and bytes).  Buffers handed to
 * the caller (sdb_pinned_alloc, sdb_graph_expand_device) are not counted.  Either output may be NULL. */
void sdb_debug_live_allocations(uint64_t* count, uint64_t* bytes);
uint64_t sdb_ctx_kernel_launches(const sdb_ctx*);
/* the cudaStream_t every kernel of this context is launched on (so a harness can bracket calls with
 * CUDA events on the launching stream) */
void* sdb_ctx_stream(const sdb_ctx*);

/* ---- brute-force KNN: replaces KnnTopK::execute (exec/operators/knn_topk.rs:166-267) and the
 *      legacy QueryExecutor::knn (idx/planner/executor.rs:283-311) ----------------------------- */
sdb_status sdb_corpus_create(sdb_ctx*, uint32_t dim, sdb_dtype, sdb_metric, uint64_t capacity_rows, sdb_corpus** out);
void sdb_corpus_destroy(sdb_corpus*);
/* rows: host memory (pinned preferred), row-major n x dim of the corpus dtype, in scan order. */
sdb_status sdb_corpus_append(sdb_corpus*, const void* rows, uint64_t n);
/* same, rows already in device memory of this context's device */
sdb_status sdb_corpus_append_device(sdb_corpus*, const void* d_rows, uint64_t n);
/* synthetic rows generated in HBM by the counter-based generator shared with the oracle
 * (element (r, c) = gen(seed, (first_row + r) * dim + c)); bench/test input only. */
sdb_status sdb_corpus_append_synthetic(sdb_corpus*, uint64_t seed, uint64_t first_row, uint64_t n);
/* rows the reference would skip (field missing / non-numeric / dimension mismatch:
 * extract_vector, knn_topk.rs:274-288; residual WHERE filter, planner/select.rs:1642-1652).
 * skip[i] != 0 excludes row i.  May be called again to change the mask. */
sdb_status sdb_corpus_set_skip(sdb_corpus*, const uint8_t* skip, uint64_t n);
/* Tombstones: the rows (scan positions) are excluded from every later search, as if the reference's TableScan no
 * longer yielded them (a DELETE, or the old version of an UPDATE whose new version is appended at the end of the
 * column).  Works on a finalized corpus without re-finalizing (skip mask + NaN screening norm + zeroed int8 row) and
 * before finalize (skip mask only).  Must not race with searches.  Row numbers of the remaining rows do not change;
 * the caller compacts (new corpus) when the tombstones pile up, or when the table version moved (KnnTopK has no
 * persistent state of its own: the cached column is keyed by (ns, db, table, field, table version), SURVEY 8f-1). */
sdb_status sdb_corpus_remove(sdb_corpus*, const uint64_t* row_ids, uint64_t n);
/* builds per-row exact f64 magnitudes, f32 screening norms, the bf16 screen copy and the special-row
 * list.  Must be called after the last append and before searching. */
sdb_status sdb_corpus_finalize(sdb_corpus*);
uint64_t sdb_corpus_rows(const sdb_corpus*);
/* copies rows [first_row, first_row + n) of the device-resident master copy back to host memory (n x dim of the
 * corpus dtype): lets a harness check results against exactly the bytes the kernels read */
sdb_status sdb_corpus_read_rows(sdb_corpus*, uint64_t first_row, uint64_t n, void* out);
/* order p of Distance::Minkowski(p) (catalog/schema/index.rs:247-284; fnc/util/math/vector.rs:163-174); default 3.
 * MINKOWSKI goes through pow(): CUDA's libm here, the platform libm in the reference -- each call agrees to within an
 * ulp or two, so Minkowski distances are equal to ~1e-14 relative rather than bit for bit (every other metric is
 * bit-exact).  Integer orders 1 .. 8 are screened (f32 Lp screen + exact re-rank), every other order is ranked by the
 * exact kernel; the order may change after finalize, but not while a batch of the corpus is in flight (between a submit
 * and its wait): the kernels of that batch read the order when they run.
 * The screen, schedule and exact settings below apply to the batches submitted after the call: a batch in flight keeps
 * the screen, schedule and exact mode it was submitted with, its repairs at wait time included. */
sdb_status sdb_corpus_set_minkowski_order(sdb_corpus*, double order);
sdb_status sdb_corpus_set_screen(sdb_corpus*, sdb_screen);
/* schedule of the tensor-core screens (results are identical; tuning / A-B only).  streaming = 1 (default): a scored
 * sample seeds the thresholds, then ONE launch streams the rest of the corpus while refiner warps raise the thresholds
 * inside the kernel.  streaming = 0: the multi-pass schedule (a launch + a selection kernel per geometric pass). */
sdb_status sdb_corpus_set_schedule(sdb_corpus*, int streaming);
/* exact = 1 (default): results are proven identical to the reference (queries whose proof fails are re-run by the exact
 * kernel).  exact = 0: opt-in approximate mode -- the exactly re-ranked best candidates of the screen are returned
 * without the proof / fallback (used by the index builder, where near-duplicate clusters would otherwise send every
 * query to the exact kernel). */
sdb_status sdb_corpus_set_exact(sdb_corpus*, int exact);
/* queries: nq x dim f64 (the reference's query is Vec<Number>; Number::Float values).
 * out_rows / out_dist: nq x k, nearest first, ties by scan order; out_count[q] <= k.
 * cancel_flag (nullable) is polled between kernel phases.  */
sdb_status sdb_knn_bruteforce(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k, uint64_t* out_rows,
                              double* out_dist, uint32_t* out_count, const volatile int* cancel_flag);
/* device-resident variant: d_queries / d_out_* are device pointers; results are complete when the
 * call returns.  row_base is added to every returned row (global id of a row-sharded corpus). */
sdb_status sdb_knn_bruteforce_device(sdb_corpus*, const double* d_queries, uint32_t nq, uint32_t k,
                                     uint64_t row_base, uint64_t* d_out_rows, double* d_out_dist,
                                     uint32_t* d_out_count);
sdb_status sdb_knn_last_stats(const sdb_corpus*, sdb_knn_stats* out);

/* ---- asynchronous batches.  submit enqueues a whole batch (query preparation, screen, exact re-rank, proof, result
 * copy) on the context's stream WITHOUT any host synchronisation and returns a ticket; wait blocks until that batch is
 * complete (and, for the rare query whose proof failed, runs the exact kernel).  Up to 4 batches may be in flight per
 * corpus, so the host can prepare / transfer batch i+1 while batch i computes -- the shape in which concurrent
 * SurrealQL queries arrive at KnnTopK::execute (one operator instance per query, exec/operators/knn_topk.rs:166).
 * Buffers handed to submit must stay valid until the matching wait returns.  Host variant: `queries` and `out_*` are
 * host buffers (pinned for overlap); the H2D copy runs on a separate copy stream.  Tickets complete in any order. */
sdb_status sdb_knn_submit(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k, uint64_t* out_rows,
                          double* out_dist, uint32_t* out_count, uint32_t* ticket);
sdb_status sdb_knn_submit_device(sdb_corpus*, const double* d_queries, uint32_t nq, uint32_t k, uint64_t row_base,
                                 uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count, uint32_t* ticket);
sdb_status sdb_knn_wait(sdb_corpus*, uint32_t ticket);

/* ---- filtered brute force: `WHERE emb <|k|> $q AND cond`, the condition applied before ranking, per statement, with
 * no change to the corpus (a filtered call is a search: the screen copies, the skip mask and the special rows stay as
 * sdb_corpus_finalize left them, so one finalized column serves any number of predicates).
 * filters: n_filters bitmaps of W = ceil(sdb_corpus_rows / 32) uint32 words each; bit r = bit r % 32 of word r / 32
 * (the sdb_hop_filter convention).  No word past W - 1 of a bitmap is read.
 * query_filter: ALWAYS host memory, nq indices < n_filters (checked, and copied before the call returns); NULL = every
 * query uses filter 0.
 * Query q ranks exactly the rows whose bit is set in its filter and that are neither skipped (sdb_corpus_set_skip) nor
 * removed (sdb_corpus_remove): a set bit never brings a skipped or removed row back.  The result equals the unfiltered
 * call's after set_skip(skip | ~filter) + finalize -- same rows, same order, bit-identical distances, same counts
 * (out_count[q] < k when fewer rows pass, 0 when none does).  Everything else is as in the unfiltered calls: every
 * metric, F32 and F64, k <= 4096, cancellation, sdb_knn_last_stats, up to 4 tickets in flight (filtered and unfiltered
 * mixed), completion through sdb_knn_wait.  SDB_EINVAL: n_filters == 0 with nq > 0, filters == NULL, or an index >=
 * n_filters.
 * A query whose bitmap has at most 4096 set bits (COSINE, EUCLIDEAN, MANHATTAN, CHEBYSHEV, PEARSON, MINKOWSKI of
 * an integer order 1 .. 8, HAMMING and JACCARD on the count path; k <= 256) skips the screen
 * (its passing rows are ranked directly; results are
 * the same); sdb_knn_last_stats then reports screen_used = SDB_SCREEN_NONE_EXACT and n_passes = 0 for a batch of such
 * queries only.
 * Host variants: `filters` is host memory, staged per batch on the copy stream (submit: `queries`, `filters` and the
 * outputs stay valid until the wait returns).  Device variants: d_filters is device memory, read in place (submit: it
 * stays valid and unchanged until the wait returns).
 * sdb_knn_submit_filtered_device is the asynchronous device variant (row_base as in sdb_knn_submit_device).  The
 * direct / screened split needs each bitmap's set bits on the host, so before it returns the call counts them on the
 * device and waits for that count alone: one short host wait for a kernel that reads the bitmaps once, on a stream
 * that carries no batch, never for the batches already in flight. */
sdb_status sdb_knn_bruteforce_filtered(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k,
                                       const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                       uint64_t* out_rows, double* out_dist, uint32_t* out_count,
                                       const volatile int* cancel_flag);
sdb_status sdb_knn_bruteforce_filtered_device(sdb_corpus*, const double* d_queries, uint32_t nq, uint32_t k,
                                              const uint32_t* d_filters, uint32_t n_filters,
                                              const uint32_t* query_filter, uint64_t row_base, uint64_t* d_out_rows,
                                              double* d_out_dist, uint32_t* d_out_count);
sdb_status sdb_knn_submit_filtered(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k,
                                   const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                   uint64_t* out_rows, double* out_dist, uint32_t* out_count, uint32_t* ticket);
sdb_status sdb_knn_submit_filtered_device(sdb_corpus*, const double* d_queries, uint32_t nq, uint32_t k,
                                          const uint32_t* d_filters, uint32_t n_filters, const uint32_t* query_filter,
                                          uint64_t row_base, uint64_t* d_out_rows, double* d_out_dist,
                                          uint32_t* d_out_count, uint32_t* ticket);

/* ---- multi-GPU brute force (SURVEY 8e): the corpus is row-sharded, every shard searches its rows, ONE NCCL
 * all-gather moves the per-shard top-k blocks and a merge kernel on every rank produces the global top-k by
 * (distance, global row).  NCCL lives inside the library (bound at run time with dlopen, so single-GPU users need
 * none); everything is enqueued on the context's stream without host synchronisation.
 *   one process per GPU : rank 0 calls sdb_comm_unique_id and hands the 128 bytes to the other ranks out of band;
 *                         every rank calls sdb_comm_init_rank on its context (collective).
 *   one process, N GPUs : sdb_ctx_create_multi creates the N contexts and their communicator (ncclCommInitAll);
 *                         sdb_knn_sharded_multi drives all shards from the calling thread.
 * A corpus becomes a shard by sdb_corpus_set_row_base(first global row).  sdb_knn_sharded_* are COLLECTIVE: every
 * rank must call them with the same queries, nq and k, in the same order.  Exactness across ranks: each block carries
 * the number of queries its rank must still repair on the host (failed proof, special queries); every rank sees every
 * header after the all-gather, so all ranks agree on whether a repair round (local exact re-runs, second all-gather
 * and merge) is needed -- no extra collective. */
#define SDB_COMM_ID_BYTES 128
sdb_status sdb_comm_unique_id(uint8_t* id128);
sdb_status sdb_comm_init_rank(sdb_ctx*, int nranks, int rank, const uint8_t* id128);
int sdb_comm_size(const sdb_ctx*);
int sdb_comm_rank(const sdb_ctx*);
sdb_status sdb_ctx_create_multi(const int* devices, int ndev, sdb_ctx** out /* [ndev] */);
sdb_status sdb_corpus_set_row_base(sdb_corpus*, uint64_t first_global_row);
sdb_status sdb_knn_sharded_submit(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k, uint64_t* out_rows,
                                  double* out_dist, uint32_t* out_count, uint32_t* ticket);
sdb_status sdb_knn_sharded_submit_device(sdb_corpus*, const double* d_queries, uint32_t nq, uint32_t k,
                                         uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                                         uint32_t* ticket);
sdb_status sdb_knn_sharded_wait(sdb_corpus*, uint32_t ticket);
/* one process, N GPUs: shards[i] lives on the i-th context of sdb_ctx_create_multi; queries / out_* are host buffers */
sdb_status sdb_knn_sharded_multi(sdb_corpus* const* shards, int n_shards, const double* queries, uint32_t nq, uint32_t k,
                                 uint64_t* out_rows, double* out_dist, uint32_t* out_count);
/* Filtered brute force on a row-sharded column: `WHERE emb <|k|> $q AND cond` when the column spans several GPUs.
 * The bitmaps cover the GLOBAL rows: n_filters bitmaps of W = ceil(n_rows_total / 32) uint32 words each, bit r = bit
 * r % 32 of word r / 32 (the sdb_hop_filter convention), query_filter as in sdb_knn_bruteforce_filtered (host memory,
 * NULL = filter 0).  Collective like the calls above: every rank passes the same queries, bitmaps and query_filter.
 * Each shard reads only its span of each bitmap (words row_base / 32 .. (row_base + rows) / 32 + 1, the host variants
 * copy just that span) and shifts it to its own rows on the device; any row_base works, aligned or not.  Query q
 * returns exactly what sdb_knn_bruteforce_filtered returns on the unsharded column with the same bitmaps: the same
 * global rows in the same order, bit-identical distances, the same counts.  Completion through sdb_knn_sharded_wait;
 * filtered and unfiltered sharded tickets mix, up to 4 in flight.  Refusals: those of sdb_knn_bruteforce_filtered,
 * and SDB_EINVAL when row_base + sdb_corpus_rows > n_rows_total; the column keeps answering after one.  Device
 * variant: d_filters is device memory, read in place until the wait returns; before it returns the call counts the
 * slice's set bits on the device and waits for that count alone (see sdb_knn_submit_filtered_device). */
sdb_status sdb_knn_sharded_submit_filtered(sdb_corpus*, const double* queries, uint32_t nq, uint32_t k,
                                           const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                           uint64_t n_rows_total, uint64_t* out_rows, double* out_dist,
                                           uint32_t* out_count, uint32_t* ticket);
sdb_status sdb_knn_sharded_submit_filtered_device(sdb_corpus*, const double* d_queries, uint32_t nq, uint32_t k,
                                                  const uint32_t* d_filters, uint32_t n_filters,
                                                  const uint32_t* query_filter, uint64_t n_rows_total,
                                                  uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                                                  uint32_t* ticket);
/* one process, N GPUs: every shard slices the same host bitmaps */
sdb_status sdb_knn_sharded_multi_filtered(sdb_corpus* const* shards, int n_shards, const double* queries, uint32_t nq,
                                          uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                          const uint32_t* query_filter, uint64_t n_rows_total, uint64_t* out_rows,
                                          double* out_dist, uint32_t* out_count);
/* ---- projected scalar vector functions over a whole column (SURVEY 8f-4): replaces a per-row evaluation of
 *      vector::distance::* / vector::similarity::* / vector::dot / vector::magnitude (fnc/vector.rs:25-143,
 *      fnc/util/math/vector.rs:61-314) in `SELECT vector::similarity::cosine(emb, $q) FROM t`.
 * fn: an sdb_metric id (= what Distance::compute returns for it: COSINE -> cosine DISTANCE, PEARSON -> the
 * similarity, JACCARD -> the similarity, MINKOWSKI with the corpus' order) or one of sdb_vector_fn.  out: host, one f64 per row in scan order,
 * bit-identical to the reference's sequential f64 arithmetic; skipped rows get NaN.  query: host, dim doubles
 * (ignored for SDB_FN_MAGNITUDE). */
typedef enum { SDB_FN_SIMILARITY_COSINE = 16, SDB_FN_DOT = 17, SDB_FN_MAGNITUDE = 18 } sdb_vector_fn;
sdb_status sdb_corpus_project(sdb_corpus*, const double* query, int fn, double* out);
/* ---- ORDER BY a projected vector function: replaces Compute + SortTopK (exec/operators/sort/topk.rs) in
 *      `SELECT id, vector::similarity::cosine(emb, $q) AS score FROM t ORDER BY score DESC LIMIT k` on a cached column.
 * fn: as in sdb_corpus_project (an sdb_metric id or an sdb_vector_fn); each row's value is exactly what
 * sdb_corpus_project returns for that row (MINKOWSKI: the same pow() caveat).  SDB_FN_MAGNITUDE ignores the queries,
 * which may then be NULL.  Query q returns the k rows SortTopK keeps over the rows its filter passes (filters,
 * n_filters, query_filter exactly as in sdb_knn_bruteforce_filtered; filters == NULL: every row) that are neither
 * skipped nor removed: ordered by Number::cmp of the value (-0.0 == 0.0, otherwise total_cmp, so NaNs by sign and
 * payload), reversed as a whole for SDB_ORDER_DESC, then by ascending scan position.  out_value is the computed f64
 * (a -0.0 stays -0.0); out_count[q] = min(k, ranked rows).  k <= 4096 (SDB_EUNSUPPORTED beyond); k = 0 gives zero
 * counts.  Above k = 1000 the reference sorts with an unstable sort instead of its top-k heap, so rows of equal value
 * may come back in any order there: scan order is one valid answer.
 * Routing: fn = the corpus metric with SDB_ORDER_ASC is the KNN ranking and takes the KNN path unchanged (the results
 * equal sdb_knn_bruteforce[_filtered] byte for byte); SDB_FN_SIMILARITY_COSINE DESC on a COSINE corpus is screened
 * like KNN (k <= 256) and proven with the similarity's bound, vector::similarity::pearson DESC on a PEARSON corpus
 * on the same screens with the query's centred copy un-negated (k <= 256), SDB_FN_DOT in either direction on a COSINE
 * or EUCLIDEAN corpus on the bf16 tensor-core screen (maximum / minimum inner product, k <= 256: the screens score the
 * dot with q for DESC and with -q for ASC, never on the int8 copy, with the F32 stream as the ladder's last rung),
 * SDB_COSINE / SDB_FN_SIMILARITY_COSINE / SDB_EUCLIDEAN in the other orders on a COSINE or EUCLIDEAN corpus with its
 * bf16 copy (cosine distance DESC and similarity ASC on either; cosine distance ASC and similarity DESC on EUCLIDEAN;
 * euclidean ASC on COSINE; euclidean DESC, farthest first, on either; k <= 256) on the screens in the view of the
 * ranked function: the cosine score towards q or -q (the COSINE corpus' int8 copy included) or the euclidean score
 * with the other metric's per-row norm and special rows, which finalize keeps beside the corpus' own (past 1024 such
 * rows those views take the exact kernel), HAMMING / JACCARD DESC on their own corpus on the count path (k <= 256,
 * exact counts); every other (fn, order) is ranked by the exact kernel.
 * Refusals: an unknown fn or order, or nq > 0 with NULL queries for a function that takes a query: SDB_EINVAL.
 * Tickets share the corpus' four slots with KNN tickets; sdb_knn_wait completes them; cancellation and
 * sdb_knn_last_stats work as for KNN.  Row-sharded columns: sdb_corpus_order_sharded_* below. */
/* order: an sdb_order value, passed as int (like fn) so that any other value can be refused without first being
 * converted to the enum */
typedef enum { SDB_ORDER_ASC = 0, SDB_ORDER_DESC = 1 } sdb_order;
sdb_status sdb_corpus_order_topk(sdb_corpus*, const double* queries, uint32_t nq, int fn, int order, uint32_t k,
                                 const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                 uint64_t* out_rows, double* out_value, uint32_t* out_count);
/* device queries, bitmaps and outputs (query_filter stays host memory); row_base is added to every returned row */
sdb_status sdb_corpus_order_topk_device(sdb_corpus*, const double* d_queries, uint32_t nq, int fn, int order,
                                        uint32_t k, const uint32_t* d_filters, uint32_t n_filters,
                                        const uint32_t* query_filter, uint64_t row_base, uint64_t* d_out_rows,
                                        double* d_out_value, uint32_t* d_out_count);
/* asynchronous variants (buffers valid until sdb_knn_wait returns, as for sdb_knn_submit[_filtered][_device]) */
sdb_status sdb_corpus_order_submit(sdb_corpus*, const double* queries, uint32_t nq, int fn, int order,
                                   uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                   const uint32_t* query_filter, uint64_t* out_rows, double* out_value,
                                   uint32_t* out_count, uint32_t* ticket);
sdb_status sdb_corpus_order_submit_device(sdb_corpus*, const double* d_queries, uint32_t nq, int fn, int order,
                                          uint32_t k, const uint32_t* d_filters, uint32_t n_filters,
                                          const uint32_t* query_filter, uint64_t row_base, uint64_t* d_out_rows,
                                          double* d_out_value, uint32_t* d_out_count, uint32_t* ticket);

/* ORDER BY on a row-sharded column: the collective counterpart of sdb_corpus_order_submit[_device], like
 * sdb_knn_sharded_submit[_filtered][_device].  Every shard ranks its rows by (fn, order) on its own route (screens,
 * count path or exact kernel, as sdb_corpus_order_topk would on that shard) and returns its top-k by (value, global
 * row); the blocks are exchanged as for KNN and merged in the ranking's direction, so query q returns exactly what
 * sdb_corpus_order_topk returns on the unsharded column: the same global rows in the same order (above k = 1000, rows
 * of equal value in one valid order, as there), bit-identical values, the same counts.  filters == NULL: unfiltered
 * (n_rows_total ignored); otherwise the bitmaps cover the GLOBAL rows exactly as in sdb_knn_sharded_submit_filtered.
 * COLLECTIVE: every rank passes the same queries, fn, order, k, bitmaps and query_filter, in the same order of calls.
 * For SDB_MINKOWSKI every shard must also hold the same order (sdb_corpus_set_minkowski_order); the library cannot
 * check either without another collective.  Completion through sdb_knn_sharded_wait; order and KNN sharded tickets
 * share the four slots and mix.  Refusals: those of sdb_corpus_order_topk (unknown fn or order, NULL queries for a
 * function that takes one: SDB_EINVAL; k > 4096: SDB_EUNSUPPORTED) and SDB_EINVAL when filters are given and
 * row_base + sdb_corpus_rows > n_rows_total; no ticket stays claimed and the column keeps answering after one. */
sdb_status sdb_corpus_order_sharded_submit(sdb_corpus*, const double* queries, uint32_t nq, int fn, int order,
                                           uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                           const uint32_t* query_filter, uint64_t n_rows_total, uint64_t* out_rows,
                                           double* out_value, uint32_t* out_count, uint32_t* ticket);
/* device queries, bitmaps and outputs (query_filter stays host memory) */
sdb_status sdb_corpus_order_sharded_submit_device(sdb_corpus*, const double* d_queries, uint32_t nq, int fn,
                                                  int order, uint32_t k, const uint32_t* d_filters,
                                                  uint32_t n_filters, const uint32_t* query_filter,
                                                  uint64_t n_rows_total, uint64_t* d_out_rows, double* d_out_value,
                                                  uint32_t* d_out_count, uint32_t* ticket);
/* one process, N GPUs (like sdb_knn_sharded_multi[_filtered]); host buffers, blocking */
sdb_status sdb_corpus_order_sharded_multi(sdb_corpus* const* shards, int n_shards, const double* queries, uint32_t nq,
                                          int fn, int order, uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                          const uint32_t* query_filter, uint64_t n_rows_total, uint64_t* out_rows,
                                          double* out_value, uint32_t* out_count);

/* merges `n_lists` per-shard result lists (each nq x k; list l's entry j of query q is valid iff
 * j < d_counts[l*stride_counts + q]) into the global top-k by (distance, row); all pointers are device
 * pointers.  stride_* = distance in ELEMENTS between consecutive lists (0 = dense: nq*k, nq*k, nq), so the
 * lists can sit inside the per-rank blocks of ONE NCCL all-gather buffer.  This is the merge step after
 * the all-gather of per-shard candidates. */
sdb_status sdb_topk_merge_device(sdb_ctx*, uint32_t n_lists, uint32_t nq, uint32_t k, const uint64_t* d_rows,
                                 const double* d_dist, const uint32_t* d_counts, uint64_t stride_rows,
                                 uint64_t stride_dist, uint64_t stride_counts, uint64_t* d_out_rows,
                                 double* d_out_dist, uint32_t* d_out_count);
/* sdb_topk_merge_device for an ORDER BY ranking: the lists are in (value, row) order for `order` (an sdb_order value:
 * Number::cmp of the value, reversed as a whole for SDB_ORDER_DESC, then ascending row) and so is the merged list;
 * values are carried through unchanged (a -0.0 stays -0.0).  SDB_ORDER_ASC merges exactly as sdb_topk_merge_device.
 * k <= 4096 (SDB_EUNSUPPORTED beyond); more than 32 lists share the sorter's limit. */
sdb_status sdb_order_merge_device(sdb_ctx*, uint32_t n_lists, uint32_t nq, uint32_t k, int order, const uint64_t* d_rows,
                                  const double* d_value, const uint32_t* d_counts, uint64_t stride_rows,
                                  uint64_t stride_value, uint64_t stride_counts, uint64_t* d_out_rows,
                                  double* d_out_value, uint32_t* d_out_count);

/* ---- HNSW search: replaces Hnsw::knn_search (idx/trees/hnsw/mod.rs:459-482) called from
 *      HnswIndex::search_graph (idx/trees/hnsw/index.rs:341-364) ------------------------------- */
/* vectors: n_elems x dim f32 (element id = row).  Layer l adjacency is CSR over element ids;
 * row_ptr[l] has n_elems+1 entries; neighbours keep the stored order (graph.rs:104-125).
 * Every sdb_metric is served, with the reference's typed arithmetic of the index's vector type
 * (idx/trees/vector.rs:206-451): all loaders build the per-element state COSINE (types other than F32: the norm, 8
 * bytes per element), PEARSON (mean, sum of squared deviations: 16 bytes per element) and JACCARD (sorted distinct keys:
 * (key bytes * dim + 4) bytes per element, keys of 8 bytes for F64 / I64 and 4 bytes otherwise) need; SDB_ENOMEM if it
 * does not fit.  MINKOWSKI uses order 3 until sdb_hnsw_set_minkowski_order.  PEARSON and JACCARD are similarities that
 * the walk ranks as distances (smaller first), as the reference does -- except F64 JACCARD, which the reference computes
 * as 1 - similarity (vector.rs:316-327).  sdb_hnsw_load is sdb_hnsw_load_typed with SDB_VT_F32. */
sdb_status sdb_hnsw_load(sdb_ctx*, uint32_t dim, sdb_metric, uint64_t n_elems, const float* vectors,
                         uint32_t n_layers, const uint64_t* const* row_ptr, const uint32_t* const* col_idx,
                         int64_t entry_point, sdb_hnsw** out);
/* Any vector type: vectors holds n_elems x dim elements of it.  The integer types compute with wrapping `+ - * abs`,
 * as the reference's release build does (I16 COSINE's dot product wraps in i16).  SDB_EINVAL for an unknown type;
 * SDB_EUNSUPPORTED for I16 PEARSON with dim > 32767 (the reference panics: the mean's divisor does not fit i16). */
sdb_status sdb_hnsw_load_typed(sdb_ctx*, uint32_t dim, sdb_metric, sdb_vector_type, uint64_t n_elems, const void* vectors,
                               uint32_t n_layers, const uint64_t* const* row_ptr, const uint32_t* const* col_idx,
                               int64_t entry_point, sdb_hnsw** out);
/* Device-resident variants for index construction (SURVEY 8f-2): vectors and per-layer CSR arrays are DEVICE pointers
 * that the handle BORROWS (nothing is copied; the caller keeps them alive and unchanged while the handle exists), and
 * the search takes device queries / writes device results.  The incremental builder uses the walk kernel itself as the
 * insertion search (Hnsw::insert -> HnswLayer::search_multi with efc, hnsw/mod.rs:297-377, hnsw/layer.rs:342-387).
 * sdb_hnsw_load_device is sdb_hnsw_load_device_typed with SDB_VT_F32. */
sdb_status sdb_hnsw_load_device(sdb_ctx*, uint32_t dim, sdb_metric, uint64_t n_elems, const float* d_vectors,
                                uint32_t n_layers, const uint64_t* const* d_row_ptr, const uint32_t* const* d_col_idx,
                                int64_t entry_point, sdb_hnsw** out);
/* Any vector type: d_vectors holds n_elems x dim elements of it.  Refusals as sdb_hnsw_load_typed. */
sdb_status sdb_hnsw_load_device_typed(sdb_ctx*, uint32_t dim, sdb_metric, sdb_vector_type, uint64_t n_elems,
                                      const void* d_vectors, uint32_t n_layers, const uint64_t* const* d_row_ptr,
                                      const uint32_t* const* d_col_idx, int64_t entry_point, sdb_hnsw** out);
/* Swaps the adjacency of a handle from sdb_hnsw_load_device[_typed] (the new arrays are borrowed the same way; the old
 * ones are no longer read once this returns) and keeps the elements' metric state (cosine norms, Pearson moments,
 * Jaccard keys), which depends on the vectors only.  The builder re-points one handle at the growing graph after every
 * insertion batch, or at layers [l .. top] to search from layer l.  SDB_EINVAL on a handle that owns its arrays. */
sdb_status sdb_hnsw_set_layers_device(sdb_hnsw*, uint32_t n_layers, const uint64_t* const* d_row_ptr,
                                      const uint32_t* const* d_col_idx, int64_t entry_point);
sdb_status sdb_hnsw_search_device(sdb_hnsw*, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                  uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count);
void sdb_hnsw_destroy(sdb_hnsw*);
/* Filtered search: replaces Hnsw::knn_search_with_filter (hnsw/mod.rs:488-515; HnswLayer::search_single_with_filter /
 * search_with_filter / add_if_truthy, hnsw/layer.rs:111-149,226-306) when the WHERE condition has been evaluated
 * ahead of time into a predicate mask: truthy[e] != 0 iff HnswTruthyDocumentFilter::check_any_doc_truthy
 * (hnsw/filter.rs:52-136) holds for element e (host, n_elems bytes).  The descent through the upper layers is
 * unfiltered, as in the reference.  SDB_EOVERFLOW = the filter is too selective for the on-chip candidate window
 * (the caller keeps the CPU path for that query). */
sdb_status sdb_hnsw_search_filtered(sdb_hnsw*, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                    const uint8_t* truthy, uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                                    uint64_t* out_counters);
/* Filtered search of any selectivity, one bitmap per query: `WHERE cond AND emb <|k,ef|> $q` for a batch of statements
 * with different conditions.  Query q is exactly Hnsw::knn_search_with_filter with truthy[e] = bit e of its bitmap --
 * same ids, f64 distances and both counters as the reference, for any selectivity, none and all included.  The descent
 * through the upper layers is unfiltered.
 * filters: n_filters bitmaps of W = ceil(n_elems / 32) uint32 words each; bit e = bit e % 32 of word e / 32 (the
 * sdb_hop_filter convention); bits past n_elems in the last word are ignored.
 * query_filter: ALWAYS host memory, nq indices < n_filters (checked, and copied before the call returns); NULL = every
 * query uses filter 0.
 * These calls never return SDB_EOVERFLOW.  A query that outgrows the on-chip candidate window or the visited table is
 * walked again by the spill tier: its candidate queue in device memory (a heap of 16 bytes per element) with an exact
 * visited set (4 bytes per element), in a pool of such slots sized to the free device memory; queries wait for a slot
 * and none fails for capacity.  SDB_ENOMEM only when not even one slot fits.  The other queries of the batch are not
 * affected.  SDB_EINVAL: n_filters == 0 with nq > 0, filters == NULL with nq > 0, or an index >= n_filters.  Every
 * metric and vector type, ef <= 4096, the Minkowski order, SDB_ECANCELLED and the handle's lock as in sdb_hnsw_search.
 * Pending documents: clear their elements' bits (add_if_truthy ignores such elements, as for the byte mask above).
 * Host variant: queries, filters and the outputs are host memory.  Device variant: d_queries, d_filters and the
 * outputs are device memory (d_out_counters nullable). */
sdb_status sdb_hnsw_search_filtered_batch(sdb_hnsw*, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                          const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                          uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                                          uint64_t* out_counters);
sdb_status sdb_hnsw_search_filtered_batch_device(sdb_hnsw*, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                                 const uint32_t* d_filters, uint32_t n_filters,
                                                 const uint32_t* query_filter, uint64_t* d_out_elems,
                                                 double* d_out_dist, uint32_t* d_out_count, uint64_t* d_out_counters);
/* how many queries of the handle's last sdb_hnsw_search_filtered_batch[_device] call the spill tier finished; after
 * sdb_hnsw_wait(t) on a filtered ticket, t's */
uint32_t sdb_hnsw_last_spilled(const sdb_hnsw*);

/* Asynchronous HNSW search: submit queues a whole batch without a host synchronisation and returns a ticket;
 * sdb_hnsw_wait(ticket) completes it.  Up to 4 tickets per handle are in flight (a fifth submit: SDB_EOVERFLOW, and the
 * handle keeps answering); they complete in any order, filtered and unfiltered mixed, and blocking searches on the
 * handle may run between them.  After the wait returns SDB_OK a ticket's outputs are byte for byte those of the
 * matching blocking call on the same handle (ids, f64 distances, counts, both counters):
 *   sdb_hnsw_submit                      = sdb_hnsw_search (all_docs_pending NULL) or sdb_hnsw_search_pending,
 *   sdb_hnsw_submit_device               = sdb_hnsw_search_device (d_out_counters nullable),
 *   sdb_hnsw_submit_filtered[_device]    = sdb_hnsw_search_filtered_batch[_device].
 * Submit refuses what the blocking call refuses before it walks (SDB_EINVAL, SDB_EUNSUPPORTED), and returns
 * SDB_ECANCELLED, with no ticket, when the context's cancel flag is up.  The wait returns what the blocking call finds
 * after its walk: SDB_EOVERFLOW (unfiltered visited table), the spill tier's SDB_ENOMEM / SDB_EUNSUPPORTED, and
 * SDB_ECANCELLED when the flag went up while the ticket was in flight (outputs undefined; the spill tier does not run).
 * The wait releases the ticket whatever it returns; an unknown or completed ticket is SDB_EINVAL.  nq, k or ef = 0 get
 * a ticket whose wait leaves zero counts.  sdb_hnsw_last_spilled after the wait of a filtered ticket reports its spill.
 * Buffers: query_filter (host) is checked and copied before submit returns; queries, filters, all_docs_pending and the
 * outputs stay valid (d_filters also unchanged) until the wait returns.  Pinned host buffers overlap with the walk;
 * pageable ones work, with host copies the driver makes synchronous.  The Minkowski order is the one at submit.
 * While a ticket is in flight sdb_hnsw_set_layers_device returns SDB_EINVAL (the spill tier at the wait reads the
 * layers the ticket was submitted against); sdb_hnsw_destroy waits for the tickets' work and frees their buffers.
 * Submit holds the handle's lock only while it queues; the wait releases it while it waits for the device.  Tickets
 * alternate the context's two streams, each with its own visited tables, so one batch's walk fills the SMs another's
 * tail and spill tier leave idle. */
sdb_status sdb_hnsw_submit(sdb_hnsw*, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                           const uint8_t* all_docs_pending /* nullable */, uint64_t* out_elems, double* out_dist,
                           uint32_t* out_count, uint64_t* out_counters /* nullable */, uint32_t* ticket);
sdb_status sdb_hnsw_submit_device(sdb_hnsw*, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                  uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count,
                                  uint64_t* d_out_counters /* nullable */, uint32_t* ticket);
sdb_status sdb_hnsw_submit_filtered(sdb_hnsw*, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                    const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                    uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                                    uint64_t* out_counters, uint32_t* ticket);
sdb_status sdb_hnsw_submit_filtered_device(sdb_hnsw*, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                           const uint32_t* d_filters, uint32_t n_filters,
                                           const uint32_t* query_filter /* host */, uint64_t* d_out_elems,
                                           double* d_out_dist, uint32_t* d_out_count, uint64_t* d_out_counters,
                                           uint32_t* ticket);
sdb_status sdb_hnsw_wait(sdb_hnsw*, uint32_t ticket);

/* Search while pending updates exist: Hnsw::knn_search(.., pending_docs = Some(bitmap)) (hnsw/mod.rs:459-482).
 * all_docs_pending[e] != 0 iff EVERY document of element e is in the pending bitmap that
 * HnswIndex::search_pendings (hnsw/index.rs:372-420) returned (are_all_docs_in_pending, hnsw/layer.rs:320-339),
 * evaluated by the caller per element (host, n_elems bytes).  Such an element still enters the result window but is
 * never expanded (layer.rs:209), in every layer.  The filtered search needs no extra entry point: add_if_truthy
 * ignores those elements (layer.rs:287-296), i.e. the caller clears their bits in the `truthy` mask. */
sdb_status sdb_hnsw_search_pending(sdb_hnsw*, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                   const uint8_t* all_docs_pending, uint64_t* out_elems, double* out_dist,
                                   uint32_t* out_count, uint64_t* out_counters);

/* Distance::calculate for VectorType::F32 vectors (idx/trees/vector.rs:243-289,659-672) applied to vectors that are
 * not part of the graph: the new_vectors of pending updates, which HnswIndex::search_pendings ranks by brute force
 * (hnsw/index.rs:398-404).  query: dim floats, vectors: n x dim floats, out: n doubles (all host memory).  Same
 * arithmetic as the walk kernel (f32 8-lane accumulation, f64 finish). */
sdb_status sdb_vec_distance_f32(sdb_ctx*, sdb_metric, uint32_t dim, const float* query, const float* vectors, uint64_t n,
                                double* out);
/* The same for an index of any metric and vector type: Distance::calculate(&query, &vector) (hnsw/index.rs:407) with
 * the index's metric, vector type and Minkowski order, i.e. what search_pendings needs.  JACCARD is asymmetric: query
 * first, as there.  query: dim elements, vectors: n x dim elements, both of the index's vector type; out: n doubles
 * (all host memory).  MINKOWSKI goes through pow(), CUDA's libm (within an ulp or two of the platform libm per call);
 * every other metric is bit-exact. */
sdb_status sdb_hnsw_distance(sdb_hnsw*, const void* query, const void* vectors, uint64_t n, double* out);
/* order p of Distance::Minkowski(p) for a MINKOWSKI index (default 3; NaN -> SDB_EINVAL).  Waits for running searches
 * on the handle; the next search uses the new order. */
sdb_status sdb_hnsw_set_minkowski_order(sdb_hnsw*, double order);

/* ---- staging: the reference's persisted HNSW state -> device (SURVEY 8a row a14).  These replace the per-key
 *      decode loops of HnswLayer::load (idx/trees/hnsw/layer.rs:526-540, UndirectedGraph::load_node
 *      idx/trees/graph.rs:117-126) and HnswElements::get_vector (hnsw/elements.rs:95-128, Vector::from(
 *      SerializedVector) idx/trees/vector.rs:93-103).  The caller range-scans the KV store and hands over the raw
 *      VALUE bytes, concatenated: value i occupies blob[off[i] .. off[i+1]).  Blobs may be pageable or pinned host
 *      memory.  *n_bad (nullable) counts values that failed validation (bad header, length != dim, target id out
 *      of range, value not representable in the output type, edge to an unknown element); those values are skipped.
 * He values: revisioned SerializedVector {F64,F32,I64,I32,I16}; elem_ids[i] = destination row (NULL: row i).
 * d_out_rows: DEVICE buffer n_rows x dim of out_dtype (SDB_F32 / SDB_F64); d_present (device, nullable) gets 1 per
 * decoded row. */
sdb_status sdb_stage_decode_vectors(sdb_ctx*, const uint8_t* blob, const uint64_t* off, const uint64_t* elem_ids,
                                    uint64_t n, uint32_t dim, sdb_dtype out_dtype, uint64_t n_rows, void* d_out_rows,
                                    uint8_t* d_present, uint64_t* n_bad);
/* Hn values of ONE layer (BE u16 count + BE u64 neighbour ids), node_ids[i] = the key's node id.  Output: CSR over
 * element ids 0..n_elems-1 in stored neighbour order, first occurrence kept (DynamicSet::insert); host arrays owned
 * by the library (sdb_free). */
sdb_status sdb_stage_decode_nodes(sdb_ctx*, const uint8_t* blob, const uint64_t* off, const uint64_t* node_ids,
                                  uint64_t n, uint64_t n_elems, uint64_t** out_row_ptr, uint32_t** out_col_idx,
                                  uint64_t* n_bad);
/* Both of the above fused with sdb_hnsw_load: raw He values + per-layer Hn values in, device-resident index out
 * (no host-side CSR is ever materialised).  entry_point / n_layers come from the Hs state (hnsw/mod.rs:61-72).
 * An F32 index: a He value of another variant is refused with SDB_EUNSUPPORTED (use sdb_hnsw_load_staged_typed). */
sdb_status sdb_hnsw_load_staged(sdb_ctx*, uint32_t dim, sdb_metric, uint64_t n_elems, const uint8_t* vec_blob,
                                const uint64_t* vec_off, const uint64_t* vec_ids, uint64_t n_vec, uint32_t n_layers,
                                const uint8_t* const* node_blob, const uint64_t* const* node_off,
                                const uint64_t* const* node_ids, const uint64_t* n_nodes, int64_t entry_point,
                                sdb_hnsw** out, uint64_t* n_bad);
/* The same for an index of any vector type.  He values are decoded natively (an I64 above 2^53 keeps its value); a
 * value whose variant is not the index's type is counted in *n_bad and skipped, like any malformed value.  Refusals
 * as sdb_hnsw_load_typed. */
sdb_status sdb_hnsw_load_staged_typed(sdb_ctx*, uint32_t dim, sdb_metric, sdb_vector_type, uint64_t n_elems,
                                      const uint8_t* vec_blob, const uint64_t* vec_off, const uint64_t* vec_ids,
                                      uint64_t n_vec, uint32_t n_layers, const uint8_t* const* node_blob,
                                      const uint64_t* const* node_off, const uint64_t* const* node_ids,
                                      const uint64_t* n_nodes, int64_t entry_point, sdb_hnsw** out, uint64_t* n_bad);
/* queries nq x dim elements of the index's vector type (float for sdb_hnsw_load / _device / _staged); out nq x k
 * (element id, f64 distance) ascending; out_counters (nullable) nq x 2 = {distance evaluations, expanded nodes} per
 * query.  The same holds for the queries of _search_device, _search_filtered and _search_pending. */
sdb_status sdb_hnsw_search(sdb_hnsw*, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                           uint64_t* out_elems, double* out_dist, uint32_t* out_count, uint64_t* out_counters);

/* Exact kNN over the elements of an index, in its own arithmetic (TestCollection::knn, idx/trees/hnsw/mod.rs:1186-1197):
 * for every query, d = Distance::calculate(element, query) -- the walk's argument order and distance code, so d equals
 * what sdb_hnsw_search reports for the pair -- and the k smallest ordered by (total-order key of d, element id), the
 * order of KnnResultBuilder.  d_members (device, distinct element ids, any order): the candidates, n_members of them;
 * NULL = every element.  d_queries: nq x dim elements of the index's vector type (device); d_out_elems / d_out_dist
 * nq x k, d_out_count nq = min(k, candidates) (device).  1 <= k <= 256, else SDB_EINVAL; a member id >= n_elems is
 * SDB_EINVAL.  -0.0 is reported as 0.0, as by the walk.  Used for the GPU builder's candidate lists and for ground-truth
 * recall. */
sdb_status sdb_hnsw_knn_exact_device(sdb_hnsw*, const void* d_queries, uint32_t nq, uint32_t k, const uint32_t* d_members,
                                     uint64_t n_members, uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count);
/* Heuristic::select, standard variant (idx/trees/hnsw/heuristic.rs:61-81,201-216), for any metric and vector type, on
 * the handle's vectors, element state and Minkowski order, with the walk's distance code: a selection made from a given
 * candidate list equals the reference's.  Elements d_elem_ids[i] (device; NULL: row0 + i), i < n; d_cand n x kc
 * element ids (device), d_cand_cnt valid entries per row; the element itself may appear and is skipped.  If at most
 * m_max candidates other than the element remain, all are taken.  Otherwise candidates are visited in order and e is
 * accepted iff e_dist > r_dist holds for no accepted r, r_dist = calculate(r, e) (elements.rs:133-140), until m_max are
 * accepted.  presorted != 0: the list is visited as given, e_dist = calculate(e, element), the distance an insertion
 * search or sdb_hnsw_knn_exact_device ranked it by; presorted = 0 (build_priority_list, layer.rs:389-405): e_dist =
 * calculate(element, e) and the list is visited by e_dist, equal distances in list order.  d_out: n x m_max element
 * ids, d_out_cnt accepted count (device).  Candidate ids must be < n_elems. */
sdb_status sdb_hnsw_select_device(sdb_hnsw*, const uint32_t* d_elem_ids, uint64_t row0, uint64_t n, const uint64_t* d_cand,
                                  const uint32_t* d_cand_cnt, uint32_t kc, uint32_t m_max, int presorted, uint32_t* d_out,
                                  uint32_t* d_out_cnt);

/* Index-construction helper (SURVEY 8f-2, "next" row): Heuristic::select, standard variant
 * (idx/trees/hnsw/heuristic.rs:61-81,201-216), applied in parallel to pre-ranked candidate lists.  F32 COSINE and
 * EUCLIDEAN only (SDB_EUNSUPPORTED otherwise), in its own f32 arithmetic (fused multiply-adds, squared euclidean), not
 * the walk's: the F32 cosine / euclidean GPU builder keeps it so that its graphs do not change.  Every other metric and
 * type: sdb_hnsw_select_device.
 * d_vectors: n x dim f32 (device) of the layer's members; d_cand: n x kc candidate member indices, nearest first
 * (e.g. the rows written by sdb_knn_bruteforce_device; the element itself is skipped), d_cand_cnt: valid entries per
 * row.  For every element: if it has <= m_max candidates all are taken, otherwise candidates are visited nearest-first
 * and e is accepted iff no already accepted r is closer to e than the element is (e_dist > dist(e,r) rejects), until
 * m_max are accepted.  presorted = 0: the candidates are first ordered by their distance to the element
 * (build_priority_list, layer.rs:389-405 -- the re-selection of an over-full node), equal distances in list order; a
 * NaN distance (a zero row under cosine, a NaN or infinite element) comes after every number, NaNs in list order.  A
 * NaN distance never rejects and is never rejected.  d_out: n x m_max member indices, d_out_cnt: accepted count.  All
 * pointers are device pointers.  dim + kc > 7264 (more than 227 KB of shared memory per block): SDB_EUNSUPPORTED. */
sdb_status sdb_hnsw_select_neighbors(sdb_ctx*, const float* d_vectors, uint32_t dim, sdb_metric, uint64_t row0, uint64_t n,
                                     const uint64_t* d_cand, const uint32_t* d_cand_cnt, uint32_t kc, uint32_t m_max,
                                     int presorted, uint32_t* d_out, uint32_t* d_out_cnt);

/* the same selection for an explicit list of elements (d_elem_ids[i] = row of element i in d_vectors): the re-selection
 * of over-full neighbours after a batch of insertions (hnsw/layer.rs:362-378) touches scattered elements */
sdb_status sdb_hnsw_select_neighbors_ids(sdb_ctx*, const float* d_vectors, uint32_t dim, sdb_metric,
                                         const uint32_t* d_elem_ids, uint64_t n, const uint64_t* d_cand,
                                         const uint32_t* d_cand_cnt, uint32_t kc, uint32_t m_max, int presorted,
                                         uint32_t* d_out, uint32_t* d_out_cnt);

/* ---- graph expansion: replaces GraphEdgeScan::execute (exec/operators/scan/graph.rs:168-283)
 *      driven by LookupPart (exec/parts/lookup.rs:139-170) and the +collect recursion
 *      (exec/operators/recursion/collect.rs:74-143) -------------------------------------------- */
sdb_status sdb_graph_load_csr(sdb_ctx*, uint64_t n_rows, const uint64_t* row_ptr, const uint32_t* col_idx,
                              sdb_graph** out);
/* Row-sharded adjacency (SURVEY 8e, "one exchange per hop"): this rank holds rows [row_lo, row_hi) of the
 * n_rows_total-row CSR -- row_ptr has row_hi - row_lo + 1 entries rebased to row_ptr[0] = 0, col_idx the matching
 * slice.  sdb_graph_expand / _device / sdb_graph_collect on shard handles are COLLECTIVE over the context's
 * communicator (sdb_comm_init_rank / sdb_ctx_create_multi): every rank passes the same frontier and receives the
 * complete result, identical -- order and duplicates included -- to the unsharded call.  Per hop every rank expands
 * the sources it owns into their positions of the global output (positions = prefix sum of the all-reduced degree
 * array) and one all-reduce assembles the next frontier; +collect de-duplicates the assembled level on every rank.
 * One thread (or process) per rank: the calls synchronise with the host between hops. */
sdb_status sdb_graph_load_csr_shard(sdb_ctx*, uint64_t n_rows_total, uint64_t row_lo, uint64_t row_hi,
                                    const uint64_t* row_ptr, const uint32_t* col_idx, sdb_graph** out);
void sdb_graph_destroy(sdb_graph*);
/* applies hops[0..n_hops) in order to the frontier (multiset semantics: duplicates kept, frontier
 * order preserved, per-source limit honoured; 0 = no limit).  *out_ids is library-owned host
 * memory (free with sdb_free). */
sdb_status sdb_graph_expand(sdb_graph* const* hops, uint32_t n_hops, const uint32_t* frontier, uint64_t n_frontier,
                            uint32_t per_source_limit, uint32_t** out_ids, uint64_t* out_n);
/* device-resident variant: d_frontier and *d_out_ids are device pointers; *d_out_ids is library-owned (sdb_device_free) */
sdb_status sdb_graph_expand_device(sdb_graph* const* hops, uint32_t n_hops, const uint32_t* d_frontier, uint64_t n_frontier,
                                   uint32_t per_source_limit, uint32_t** d_out_ids, uint64_t* out_n);
void sdb_device_free(sdb_ctx*, void* d_ptr);
/* +collect BFS: first-seen dedup, emits from min_depth, start only marked seen when inclusive. */
sdb_status sdb_graph_collect(sdb_graph*, const uint32_t* start, uint64_t n_start, uint32_t min_depth,
                             uint32_t max_depth, int inclusive, uint32_t** out_ids, uint64_t* out_n);

/* ---- WHERE-filtered hops: `->(edge WHERE c1)->(node WHERE c2)`, which the reference plans as GraphScanOutput::FullEdge
 *      followed by a Filter (exec/planner/source.rs, plan_lookup_with_input).  The caller evaluates each condition into a
 *      bitmap (bit i = bit i % 32 of word i / 32):
 *        edge_bits    one bit per CSR position p (ceil(n_edges / 32) words): the edge record behind p satisfies the
 *                     hop's edge condition.  A `<->` CSR holds each edge record at two positions per endpoint; set both.
 *        target_bits  one bit per node id (ceil(n_rows / 32) words): node v satisfies the target condition.  Needs every
 *                     target id below n_rows (SDB_EINVAL otherwise).
 *      Position p passes iff (edge_bits == NULL || bit p) && (target_bits == NULL || bit col_idx[p]).  The result is the
 *      unfiltered call's, order and duplicates included, with the failing positions removed; per_source_limit = n > 0
 *      keeps each source's first n PASSING positions.  A NULL filter array, or a hop whose two bitmaps are NULL, runs
 *      that hop unfiltered.  Shard handles are refused (SDB_EUNSUPPORTED). */
typedef struct {
  const uint32_t* edge_bits;
  const uint32_t* target_bits;
} sdb_hop_filter;
/* filters: n_hops entries or NULL; the bitmaps are host memory, copied for this call */
sdb_status sdb_graph_expand_filtered(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                     const uint32_t* frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                     uint32_t** out_ids, uint64_t* out_n);
/* device-resident variant: the bitmaps (the filters array itself is host memory), d_frontier and *d_out_ids are device
 * pointers; *d_out_ids is library-owned (sdb_device_free) */
sdb_status sdb_graph_expand_filtered_device(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                            const uint32_t* d_frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                            uint32_t** d_out_ids, uint64_t* out_n);
/* +collect whose every BFS level is the filtered hop (host bitmaps); the start set itself is not filtered */
sdb_status sdb_graph_collect_filtered(sdb_graph*, const sdb_hop_filter* filter, const uint32_t* start, uint64_t n_start,
                                      uint32_t min_depth, uint32_t max_depth, int inclusive, uint32_t** out_ids,
                                      uint64_t* out_n);

/* ---- batches of documents: LookupPart::evaluate_batch (exec/parts/lookup.rs:96-112) and the per-row +collect
 *      (exec/operators/recursion/collect.rs:74-143) over a ValueBatch of rows, in one call.  Document d is the segment
 *      frontier[doc_off[d] .. doc_off[d + 1]) (the record ids of one row's value; an array value is flattened).  doc_off
 *      has n_docs + 1 entries: doc_off[0] == 0, non-decreasing, doc_off[n_docs] == n_frontier, n_docs < 2^32; anything
 *      else is SDB_EINVAL.  Empty documents and n_docs == 0 are valid.  The result is every document's result
 *      concatenated; out_doc_off (n_docs + 1 entries, the caller's buffer) marks where each one starts and ends.
 *      filters / filter: NULL (unfiltered) or as in the filtered calls above.  Unfiltered calls on shard handles are
 *      collective like the flat ones (every rank receives the complete output and identical offsets); filters on shard
 *      handles are refused (SDB_EUNSUPPORTED).  Cancellation is polled once per hop / level. */
/* Segment d of the output is exactly sdb_graph_expand[_filtered] on document d: same order, same duplicates, the limit
 * per source and per hop.  So the concatenated output is the flat call's on the whole frontier, byte for byte.  Host
 * frontier, offsets, bitmaps and result (*out_ids: sdb_free; NULL when empty). */
sdb_status sdb_graph_expand_batch(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                  const uint32_t* frontier, uint64_t n_frontier, const uint64_t* doc_off, uint64_t n_docs,
                                  uint32_t per_source_limit, uint32_t** out_ids, uint64_t* out_doc_off, uint64_t* out_n);
/* device-resident variant: d_frontier, d_doc_off, the bitmaps (the filters array itself is host memory), *d_out_ids and
 * d_out_doc_off are device memory; *d_out_ids is library-owned (sdb_device_free).  d_doc_off is checked on the device,
 * and the verdict is read back before the first hop (one 4-byte copy). */
sdb_status sdb_graph_expand_batch_device(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                         const uint32_t* d_frontier, uint64_t n_frontier, const uint64_t* d_doc_off,
                                         uint64_t n_docs, uint32_t per_source_limit, uint32_t** d_out_ids,
                                         uint64_t* d_out_doc_off, uint64_t* out_n);
/* Segment d of the output is exactly sdb_graph_collect[_filtered] on document d's start ids: its own first-seen set,
 * in level order (with inclusive its start ids first).  The de-duplication state is sized by the (document, node)
 * pairs the call visits, not by n_docs x n_rows.  The documents of a level are expanded together; a run of documents
 * whose level (before de-duplication) would exceed 2^32 ids, or, on an unsharded handle, does not fit on the device,
 * is served as two halves, down to single documents.  So SDB_EOVERFLOW means the whole result or one document's level
 * exceeds the limit, as for the single-document call, and SDB_ENOMEM that one document does not fit.  Host memory.
 * On shard handles every rank splits alike (level sizes are global), but an allocation failure is per rank: a rank
 * that returns SDB_ENOMEM or SDB_ECUDA leaves its peers in a collective, and the communicator is not usable after it. */
sdb_status sdb_graph_collect_batch(sdb_graph*, const sdb_hop_filter* filter, const uint32_t* start, uint64_t n_start,
                                   const uint64_t* doc_off, uint64_t n_docs, uint32_t min_depth, uint32_t max_depth,
                                   int inclusive, uint32_t** out_ids, uint64_t* out_doc_off, uint64_t* out_n);
/* Diagnostics of the last sdb_graph_collect_batch on this handle (for measurement, not for control flow): the pair
 * table's peak device bytes (the transient of a growth included), how many times it grew, how many level passes were
 * repeated because the level overflowed it, and how many runs of documents were split in two.  Any output may be NULL. */
void sdb_graph_last_collect_table(const sdb_graph*, uint64_t* peak_bytes, uint32_t* grows, uint32_t* repeated_passes,
                                  uint32_t* splits);
void sdb_free(void*);

#ifdef __cplusplus
}
#endif
#endif
