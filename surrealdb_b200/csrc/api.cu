// api.cu -- the extern "C" boundary (include/sdbgpu.h): contexts, corpus lifecycle, brute-force KNN driver.
#include <cmath>

#include <algorithm>
#include <chrono>

#include "internal.cuh"

namespace sdb {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}


// schedule ratio of the LEGACY multi-pass schedule (f32 SIMT screen; tensor-core screens when streaming refinement is
// switched off): every pass looks at (R-1) x the rows seen so far
static uint32_t pass_ratio(uint32_t nq) { return nq >= 512 ? 4u : PASS_RATIO; }

static std::vector<PassDesc> build_passes(uint64_t n_rows, uint32_t cand_cap, uint32_t nq) {
  std::vector<PassDesc> v;
  const uint64_t PASS_RATIO = pass_ratio(nq);  // shadows the compile-time default
  const uint64_t T = (n_rows + TILE_ROWS - 1) / TILE_ROWS;
  if (T == 0) return v;
  const uint64_t max0 = cand_cap / TILE_ROWS;  // pass 0 appends every row it sees
  uint64_t stride = 1;
  while ((T + stride - 1) / stride > max0) stride *= PASS_RATIO;
  PassDesc p0{(uint32_t)stride, 0u, (uint32_t)((T + stride - 1) / stride), 0u};
  v.push_back(p0);
  for (uint64_t s = stride / PASS_RATIO; s >= 1; s /= PASS_RATIO) {
    const uint64_t M = (T + s - 1) / s;
    PassDesc p{(uint32_t)s, (uint32_t)PASS_RATIO, (uint32_t)(M - (M + PASS_RATIO - 1) / PASS_RATIO), 0u};
    v.push_back(p);
    if (s == 1) break;
  }
  return v;
}

static uint32_t gcd_u32(uint32_t a, uint32_t b) {
  while (b) {
    const uint32_t t = a % b;
    a = b;
    b = t;
  }
  return a;
}
// streaming schedule: a PROBE launch scores a few tiles spread over the corpus and keeps only chunk maxima (seed of the
// thresholds), then ONE streaming launch covers every tile, visiting them in a golden-ratio stride order so that any
// stretch of the launch samples the whole corpus (sorted / clustered corpora do not fool the early thresholds).
// Corpora that fit the candidate lists entirely are scored in one pass-0 launch instead.
static void build_stream_passes(uint64_t n_rows, uint32_t cand_cap, uint32_t k, PassDesc* probe, PassDesc* main) {
  const uint64_t T = (n_rows + TILE_ROWS - 1) / TILE_ROWS;
  const uint64_t max0 = cand_cap / TILE_ROWS;
  *probe = PassDesc{1u, 0u, 0u, 0u};
  *main = PassDesc{1u, 0u, 0u, 0u};
  if (T == 0) return;
  if (T <= max0) {  // *probe doubles as the single pass-0 launch: main stays empty
    probe->count = (uint32_t)T;
    return;
  }
  const uint64_t P = k <= 32 ? 16 : PROBE_TILES_MAX;  // 8 chunk maxima per tile: 128 / 512 values >= 4 k / 2 k
  const uint64_t stride = T / P;                       // T > max0 >= 16; for P = 64 and T < 64 every tile is probed
  if (stride == 0) *probe = PassDesc{1u, 0u, (uint32_t)T, 0u};
  else *probe = PassDesc{(uint32_t)stride, 0u, (uint32_t)P, 0u};
  const uint32_t cnt = (uint32_t)T;
  uint32_t perm = 0;
  if (cnt >= 8) {
    perm = (uint32_t)(cnt * 0.6180339887498949) | 1u;
    while (gcd_u32(perm, cnt) != 1) perm += 2;
    if (perm >= cnt) perm = 0;
  }
  *main = PassDesc{1u, 0u, cnt, perm};
}

// The plan of a batch of nq queries ranked by `rank`, k results each, under the screen and tensor-core schedule asked
// for (the corpus' settings, or those a debug batch names).
// The precision ladder, cheapest first.  The candidate set of a query is "every row whose screened score is within the
// screen's error margin of the k-th best", so its size adapts to the data (a handful on spread-out data, a whole
// cluster on tightly packed data); a rung fails for a query only when that set overflows the list.  When that happens
// to more than a handful of queries the batch is re-screened with a tighter screen / longer lists instead of paying
// one exact pass over the corpus per failed query; the rung that worked is remembered per corpus, k and view.
static Plan plan_batch(const Corpus* c, const Ranking& rank, uint32_t k, uint32_t nq, sdb_screen screen,
                       bool stream_refine) {
  Plan p;
  const Family f = family(c);
  const bool screened = screened_ranking(c, rank), counted = screened && count_ranked(c, k, screen);
  p.rank = rank;
  p.v = view_of(c, rank);
  p.stream_refine = stream_refine;
  p.exact = c->exact;
  // direct regime: the re-rank and cand_final serve every family but Exact (Count: when the count path would rank the
  // batch), k <= 256
  p.direct_ok =
      k > 0 && k <= 256 && screened && (f == Family::Dot || f == Family::Centred || f == Family::Lp || counted);
  if (nq == 0 || k == 0) return p;  // Route::Empty: nothing to search
  // vector::dot and the cross views were ranked by the exact kernel, which reports a cancel raised while a batch is in
  // flight (it polls before every query); on the screens they still report it, from the wait
  p.cancel_at_wait = dot_ranking(c, rank) || cross_ranking(c, rank);
  // MANHATTAN / CHEBYSHEV: a single query streams the rows once either way, and the exact kernel does it at the higher
  // HBM rate (DESIGN.md section 5): AUTO ranks it there; an explicit SIMT_F32 request is kept.  MINKOWSKI's exact
  // kernel is bound by its f64 pow() calls, not by HBM, and the screen is faster for a single query too (section 5).
  // HAMMING likewise: AUTO ranks one query with the exact kernel; JACCARD's exact kernel is O(D^2) per row, so the
  // count path takes a single query too.
  p.single_exact = screen == SDB_SCREEN_AUTO &&
                   (c->metric == SDB_MANHATTAN || c->metric == SDB_CHEBYSHEV || c->metric == SDB_HAMMING);
  const bool int8_ok = c->d_i8 && screen_tc_available();  // (COSINE and Centred corpora hold an int8 copy)
  sdb_screen scr = screen;
  if (scr == SDB_SCREEN_AUTO)
    scr = !screen_tc_available() ? SDB_SCREEN_SIMT_F32
                                 : (int8_ok && c->max_rel_qerr <= 0.02f ? SDB_SCREEN_TC_INT8 : SDB_SCREEN_TC_BF16);
  if (scr == SDB_SCREEN_TC_INT8 && !int8_ok) scr = SDB_SCREEN_TC_BF16;
  // the int8 copy holds x / |x| and its integer threshold compare takes no per-row scale: only the cosine score on the
  // own screening norm runs on it (towards q or -q, whose int8 copy is the negation of q's); dot batches and the
  // other views start on bf16
  if (scr == SDB_SCREEN_TC_INT8 && (p.v.sc != Score::Cosine || p.v.cross)) scr = SDB_SCREEN_TC_BF16;
  // (Lp corpora hold no bf16 copy: the f32 Lp screen, screen_lp.cu, is their only screen, for f32 and f64 rows)
  if (scr == SDB_SCREEN_TC_BF16 && (!screen_tc_available() || !c->d_bf16)) scr = SDB_SCREEN_SIMT_F32;
  // the SIMT screen streams f32 rows: an f64 Dot corpus is screened on the tensor cores or not at all, and so is a
  // Centred one of either type (the SIMT screen would need the centred rows)
  if ((f == Family::Centred || (f == Family::Dot && c->dtype == SDB_F64)) && scr == SDB_SCREEN_SIMT_F32)
    scr = SDB_SCREEN_NONE_EXACT;
  // (Count: the count path, enqueue_counted, or the exact kernel)
  if (c->special_overflow || k > 256 || f == Family::Count || f == Family::Exact) scr = SDB_SCREEN_NONE_EXACT;
  // a view on the cross state whose special list overflowed
  if (p.v.cross && c->xspecial_overflow) scr = SDB_SCREEN_NONE_EXACT;
  // a ranking the screens do not serve (screened_ranking): the exact kernel
  if (!screened) scr = SDB_SCREEN_NONE_EXACT;
  auto push = [&](sdb_screen s, uint32_t cap) { p.ladder[p.n_ladder++] = Rung{s, cap}; };
  if (scr == SDB_SCREEN_TC_INT8) {
    push(SDB_SCREEN_TC_INT8, 4096), push(SDB_SCREEN_TC_INT8, 16384);
    push(SDB_SCREEN_TC_BF16, 4096), push(SDB_SCREEN_TC_BF16, 16384);
  } else if (scr == SDB_SCREEN_TC_BF16) {
    push(SDB_SCREEN_TC_BF16, 4096), push(SDB_SCREEN_TC_BF16, 16384);
  } else if (scr == SDB_SCREEN_SIMT_F32 && f == Family::Lp) {
    push(SDB_SCREEN_SIMT_F32, 4096), push(SDB_SCREEN_SIMT_F32, 16384);
  } else if (scr == SDB_SCREEN_SIMT_F32) {
    push(SDB_SCREEN_SIMT_F32, 4096);
  }
  // the f32 stream (error bound ~500x tighter than bf16) as the last rung before the exact kernel -- only ever used
  // for the few queries of a batch that every tensor-core rung failed to prove (finish_local), never for a whole batch
  if (p.n_ladder && p.ladder[p.n_ladder - 1].scr != SDB_SCREEN_SIMT_F32 && c->dtype == SDB_F32 && f == Family::Dot)
    push(SDB_SCREEN_SIMT_F32, 4096);
  p.route = counted ? Plan::Route::Counted : p.n_ladder ? Plan::Route::Screened : Plan::Route::Exact;
  // the whole batch: its first-choice screen and the rungs it may be re-screened on (the f32 stream behind tensor-core
  // rungs is for single queries; an all-SIMT ladder re-screens whole batches)
  const uint32_t n = p.rungs(nq);
  const bool f32_tail =
      n > 1 && p.ladder[n - 1].scr == SDB_SCREEN_SIMT_F32 && p.ladder[n - 2].scr != SDB_SCREEN_SIMT_F32;
  p.n_batch_rungs = f32_tail ? n - 1 : n;
  p.key = RungKey{n ? p.ladder[0].scr : SDB_SCREEN_NONE_EXACT, k, view_key(p.v)};
  return p;
}

static cudaError_t drain(Ctx* ctx) {  // both batch streams idle
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  const cudaError_t e2 = cudaStreamSynchronize(ctx->stream2);
  return e != cudaSuccess ? e : e2;
}

// ---- one batch = enqueue (no host synchronisation) + finish (event wait, ladder, exact fallbacks) ----------------
static sdb_status ticket_prepare(Corpus* c, Ticket& t, uint32_t nq) {
  if (!t.ev_begin) {
    SDB_CUDA(cudaEventCreate(&t.ev_begin));
    SDB_CUDA(cudaEventCreate(&t.ev_screen0));
    SDB_CUDA(cudaEventCreate(&t.ev_screen1));
    SDB_CUDA(cudaEventCreate(&t.ev_end));
    SDB_CUDA(cudaEventCreateWithFlags(&t.ev_h2d, cudaEventDisableTiming));
    SDB_CUDA(cudaEventCreateWithFlags(&t.ev_out, cudaEventDisableTiming));
    SDB_CUDA(cudaEventCreateWithFlags(&t.ev_main, cudaEventDisableTiming));
  }
  if (t.h_cap < nq) {
    t.h_cap = 0;
    const uint32_t cap = (nq + 1023) / 1024 * 1024;
    SDB_CUDA(t.h_flags.reserve(2 * (size_t)cap + 8));
    t.h_qflags = t.h_flags + cap;
    t.h_stat = t.h_qflags + cap;
    t.h_cap = cap;
  }
  return SDB_OK;
}

bool trace_enabled() {
  static const bool on = getenv("SDB_TRACE") != nullptr;
  return on;
}
void trace_mark(Ctx* ctx, Ticket& t, const char* name, cudaStream_t st) {
  if (!trace_enabled()) return;
  if (!ctx->trace_epoch) {
    cudaEventCreate(&ctx->trace_epoch);
    cudaEventRecord(ctx->trace_epoch, st);
    cudaEventSynchronize(ctx->trace_epoch);
    ctx->trace_host0 = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  }
  cudaEvent_t e;
  if (cudaEventCreate(&e) != cudaSuccess) return;
  cudaEventRecord(e, st);
  t.trace.emplace_back(name, e);
}
void trace_host(Ctx* ctx, uint32_t ticket, const char* name) {
  if (!trace_enabled() || !ctx->trace_epoch) return;
  const double now = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  fprintf(stderr, "TRACE dev%d ticket%u host %-12s %10.3f\n", ctx->device, ticket, name, (now - ctx->trace_host0) * 1e3);
}
void trace_dump(Ctx* ctx, Ticket& t) {
  if (!trace_enabled()) return;
  for (auto& m : t.trace) {
    float ms = 0.f;
    cudaEventSynchronize(m.second);
    cudaEventElapsedTime(&ms, ctx->trace_epoch, m.second);
    fprintf(stderr, "TRACE dev%d ticket%u set%d %-12s %10.3f\n", ctx->device, t.id, t.set, m.first, ms);
    cudaEventDestroy(m.second);
  }
  t.trace.clear();
}

// ScreenTap (test-only): what a stage-A selection is about to gather -- main list and private sub-lists, before capping
static sdb_status tap_gathered(const Scratch& s, ScreenTap* tap, uint32_t nq, uint32_t n_slots, cudaStream_t st) {
  std::vector<uint32_t> cnt(nq), sub((size_t)nq * n_slots);
  SDB_CUDA(cudaMemcpyAsync(cnt.data(), s.d_cand_cnt, sizeof(uint32_t) * nq, cudaMemcpyDeviceToHost, st));
  if (n_slots)
    SDB_CUDA(cudaMemcpyAsync(sub.data(), s.d_sub_cnt, sizeof(uint32_t) * sub.size(), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  std::vector<uint32_t>& g = tap->gathered;
  g.resize(nq, 0u);
  for (uint32_t q = 0; q < nq; q++) {
    uint64_t n = cnt[q];
    for (uint32_t j = 0; j < n_slots; j++) n += std::min(sub[(size_t)q * n_slots + j], s.sub_cap);
    g[q] = std::max(g[q], (uint32_t)std::min<uint64_t>(n, 0xFFFFFFFFu));
  }
  return SDB_OK;
}
// ScreenTap: the candidate lists as they stand (cnt: their counts, optional)
static sdb_status tap_list(const Scratch& s, uint32_t nq, std::vector<Cand>* list, std::vector<uint32_t>* cnt,
                           cudaStream_t st) {
  list->resize((size_t)nq * s.sc_cap);
  SDB_CUDA(cudaMemcpyAsync(list->data(), s.d_cand, sizeof(Cand) * list->size(), cudaMemcpyDeviceToHost, st));
  if (cnt) {
    cnt->resize(nq);
    SDB_CUDA(cudaMemcpyAsync(cnt->data(), s.d_cand_cnt, sizeof(uint32_t) * nq, cudaMemcpyDeviceToHost, st));
  }
  SDB_CUDA(cudaStreamSynchronize(st));
  return SDB_OK;
}

// ---- direct regime of filtered batches: the queries whose filter passes at most DIRECT_MAX_ROWS rows ------------------
// mixed batches run permuted (screened queries first, then the direct ones): gather of the queries, scatter of the results
__global__ void gather_queries_kernel(const double* __restrict__ src, const uint32_t* __restrict__ perm, uint32_t dim,
                                      double* __restrict__ dst) {
  const uint32_t i = blockIdx.x;
  const double* s = src + (size_t)perm[i] * dim;
  for (uint32_t j = threadIdx.x; j < dim; j += blockDim.x) dst[(size_t)i * dim + j] = s[j];
}
__global__ void scatter_results_kernel(const uint32_t* __restrict__ perm, uint32_t k, const uint64_t* __restrict__ rows,
                                       const double* __restrict__ dist, const uint32_t* __restrict__ cnt,
                                       uint64_t* __restrict__ out_rows, double* __restrict__ out_dist,
                                       uint32_t* __restrict__ out_cnt) {
  const uint32_t i = blockIdx.x, d = perm[i];
  const uint32_t n = cnt[i] < k ? cnt[i] : k;
  for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
    out_rows[(size_t)d * k + j] = rows[(size_t)i * k + j];
    out_dist[(size_t)d * k + j] = dist[(size_t)i * k + j];
  }
  if (threadIdx.x == 0) out_cnt[d] = cnt[i];
}
static sdb_status scatter_results(Corpus* c, Ticket& t) {
  if (!t.permuted || !t.nq) return SDB_OK;
  scatter_results_kernel<<<t.nq, 128, 0, t.stream>>>(t.d_perm, t.k, t.d_out_rows, t.d_out_dist, t.d_out_count,
                                                     t.d_fin_rows, t.d_fin_dist, t.d_fin_count);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// One run of the enqueue functions: a whole batch, the screened head or the direct tail of a mixed one, or the failed
// queries of a per-query repair.  The ticket holds what every run of the batch shares: plan, stream, scratch set, k,
// row_base, events and cancel flag.
struct Run {
  const double* d_queries;
  uint32_t nq;
  uint64_t* d_out_rows; double* d_out_dist; uint32_t* d_out_count;
  FiltArg filt;
  uint32_t rung;
  ScreenTap* tap;      // test-only (see ScreenTap)
  uint32_t *h_flags, *h_qflags;  // pinned: where the run's per-query flags go
  uint32_t* h_stat;              // pinned: where its counters go (nullptr: nowhere)
};
// what a run decided: the screen it used and its screen launches
struct Enqueued {
  int screen = SDB_SCREEN_NONE_EXACT;
  uint32_t n_passes = 0;
};

static sdb_status copy_flags(const Scratch& s, const Run& r, cudaStream_t st) {
  SDB_CUDA(cudaMemcpyAsync(r.h_flags, s.d_flags, sizeof(uint32_t) * r.nq, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaMemcpyAsync(r.h_qflags, s.d_qflags, sizeof(uint32_t) * r.nq, cudaMemcpyDeviceToHost, st));
  if (r.h_stat) SDB_CUDA(cudaMemcpyAsync(r.h_stat, s.d_stat, sizeof(uint32_t) * 4, cudaMemcpyDeviceToHost, st));
  return SDB_OK;
}

// direct queries: no screen.  Each list holds exactly the query's passing rows, so tau stays -inf and cand_final's
// proof holds trivially; the exact re-rank and cand_final order them as any candidate list.
static sdb_status enqueue_direct(Corpus* c, Ticket& t, const Run& r) {
  cudaStream_t st = t.stream;
  Scratch& s = c->sets[t.set];
  const View& v = t.plan.v;
  SDB_TRY(scratch_for(c, s, r.nq, DIRECT_MAX_ROWS));
  SDB_TRY(prep_queries(c, s, r.d_queries, r.nq, st, v));
  SDB_TRY(cand_begin(c, s, r.nq, SDB_SCREEN_NONE_EXACT, st, v, t.plan.exact));
  SDB_TRY(cand_direct(c, s, r.filt, r.nq, st));
  SDB_TRY(cand_rerank(c, s, r.filt, r.nq, st, false, v));
  SDB_TRY(cand_final(c, s, r.filt, r.nq, t.k, t.row_base, r.d_out_rows, r.d_out_dist, r.d_out_count, st, v));
  return copy_flags(s, r, st);
}

static sdb_status enqueue_screened(Corpus* c, Ticket& t, const Run& r, Enqueued* e);
// a whole batch: its last t.n_direct queries are direct, the others screened
static sdb_status enqueue_batch(Corpus* c, Ticket& t, const Run& r, Enqueued* e) {
  const uint32_t nd = t.n_direct;
  if (nd == 0) return enqueue_screened(c, t, r, e);
  cudaStream_t st = t.stream;
  if (nd == r.nq) {  // every query is direct: no screen at all
    *e = Enqueued();
    SDB_CUDA(cudaEventRecord(t.ev_begin, st));
    SDB_CUDA(cudaEventRecord(t.ev_screen0, st));
    SDB_CUDA(cudaEventRecord(t.ev_screen1, st));
    SDB_TRY(enqueue_direct(c, t, r));
    SDB_CUDA(cudaEventRecord(t.ev_end, st));
    return SDB_OK;
  }
  // mixed (permuted) batch: the screened head, then the direct tail behind it on the same stream and scratch set
  Scratch& s = c->sets[t.set];
  SDB_TRY(scratch_for(c, s, r.nq, DIRECT_MAX_ROWS));  // sized for both, so that the tail does not reallocate
  const uint32_t ns = r.nq - nd;
  Run head = r;
  head.nq = ns;
  SDB_TRY(enqueue_screened(c, t, head, e));
  SDB_CUDA(t.d_stat_scr.reserve(4));  // (the block header of a sharded batch adds both parts' flagged queries)
  SDB_CUDA(cudaMemcpyAsync(t.d_stat_scr, s.d_stat, sizeof(uint32_t) * 4, cudaMemcpyDeviceToDevice, st));
  Run tail = r;
  tail.d_queries += (size_t)ns * c->dim;
  tail.nq = nd;
  tail.d_out_rows += (size_t)ns * t.k;
  tail.d_out_dist += (size_t)ns * t.k;
  tail.d_out_count += ns;
  tail.filt.qf += ns;
  tail.h_flags += ns;
  tail.h_qflags += ns;
  tail.h_stat = nullptr;  // (the batch's counters are the head's)
  SDB_TRY(enqueue_direct(c, t, tail));
  SDB_CUDA(cudaEventRecord(t.ev_end, st));
  return SDB_OK;
}

// HAMMING / JACCARD (count_ranked): exact counts of every row in one launch, ranked per row range; each query's list
// is the union of its ranges' best k with their exact distances, so cand_final orders it with tau = -inf and nothing
// is left to prove or repair.  Reported as one SIMT_F32 pass.
static sdb_status enqueue_counted(Corpus* c, Ticket& t, const Run& r, Enqueued* e) {
  Ctx* ctx = c->ctx;
  cudaStream_t st = t.stream;
  Scratch& s = c->sets[t.set];
  const uint32_t nq = r.nq, k = t.k;
  e->screen = SDB_SCREEN_SIMT_F32;
  e->n_passes = 1;
  SDB_CUDA(cudaEventRecord(t.ev_begin, st));
  trace_mark(ctx, t, "begin", st);
  const View& v = t.plan.v;
  SDB_TRY(scratch_for(c, s, nq, std::max(4096u, count_ranges(c, nq, k) * k)));
  SDB_TRY(prep_queries(c, s, r.d_queries, nq, st, v));
  SDB_TRY(cand_begin(c, s, nq, SDB_SCREEN_NONE_EXACT, st, v, t.plan.exact));
  if (c->last_main && c->last_main != t.ev_main) SDB_CUDA(cudaStreamWaitEvent(st, c->last_main, 0));
  SDB_CUDA(cudaEventRecord(t.ev_screen0, st));
  if ((t.cancel && *t.cancel) || ctx_cancelled(ctx)) {
    cudaStreamSynchronize(st);
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  SDB_TRY(count_pass(c, s, r.filt, nq, k, st, v.desc));
  SDB_CUDA(cudaEventRecord(t.ev_main, st));
  c->last_main = t.ev_main;
  SDB_CUDA(cudaEventRecord(t.ev_screen1, st));
  trace_mark(ctx, t, "counted", st);
  SDB_TRY(cand_final(c, s, r.filt, nq, k, t.row_base, r.d_out_rows, r.d_out_dist, r.d_out_count, st, v));
  SDB_TRY(copy_flags(s, r, st));
  SDB_CUDA(cudaEventRecord(t.ev_end, st));
  trace_mark(ctx, t, "end", st);
  return SDB_OK;
}

static sdb_status enqueue_screened(Corpus* c, Ticket& t, const Run& r, Enqueued* e) {
  Ctx* ctx = c->ctx;
  cudaStream_t st = t.stream;
  Scratch& s = c->sets[t.set];
  const uint32_t nq = r.nq, k = t.k;
  const Plan& plan = t.plan;
  const View& v = plan.v;
  if (plan.counted(nq)) return enqueue_counted(c, t, r, e);
  const uint32_t n_rungs = plan.rungs(nq);
  e->n_passes = 0;
  SDB_CUDA(cudaEventRecord(t.ev_begin, st));
  trace_mark(ctx, t, "begin", st);
  if (n_rungs == 0) {  // exact-only: the exact kernel needs the prepared queries (f64 copy, |q|, flags)
    e->screen = SDB_SCREEN_NONE_EXACT;
    SDB_TRY(scratch_for(c, s, nq, 4096));
    SDB_TRY(prep_queries(c, s, r.d_queries, nq, st, v));
    SDB_CUDA(cudaEventRecord(t.ev_screen0, st));
    SDB_CUDA(cudaEventRecord(t.ev_screen1, st));
    SDB_CUDA(cudaMemsetAsync(r.d_out_count, 0, sizeof(uint32_t) * nq, st));
    SDB_CUDA(cudaMemcpyAsync(r.h_qflags, s.d_qflags, sizeof(uint32_t) * nq, cudaMemcpyDeviceToHost, st));
    for (uint32_t q = 0; q < nq; q++) r.h_flags[q] = 2u;  // every query takes the exact kernel
    const uint32_t stat[4] = {nq, 0u, 0u, 0u};
    if (r.h_stat) std::copy(stat, stat + 4, r.h_stat);
    SDB_CUDA(cudaEventRecord(t.ev_end, st));
    return SDB_OK;
  }
  const Rung rg = plan.ladder[std::min(r.rung, n_rungs - 1)];
  const sdb_screen rs = rg.scr;
  e->screen = (int)rs;
  const bool tc = rs == SDB_SCREEN_TC_INT8 || rs == SDB_SCREEN_TC_BF16;
  const bool int8 = rs == SDB_SCREEN_TC_INT8;
  SDB_TRY(scratch_for(c, s, nq, rg.cap));
  const uint32_t cap = s.sc_cap;
  SDB_TRY(prep_queries(c, s, r.d_queries, nq, st, v));
  SDB_TRY(cand_begin(c, s, nq, (int)rs, st, v, plan.exact));
  // Screens are persistent one-CTA-per-SM kernels: two of them in flight on different streams would split the SMs,
  // run in two waves and starve the refiners of the CTAs that are not resident yet.  So the screen of this batch waits
  // for the end of the previous batch's screen -- only the TAIL of the previous batch overlaps with it.
  if (c->last_main && c->last_main != t.ev_main) SDB_CUDA(cudaStreamWaitEvent(st, c->last_main, 0));
  SDB_CUDA(cudaEventRecord(t.ev_screen0, st));  // after the wait: screen_ms is this batch's screen, not the queueing
  trace_mark(ctx, t, "screen0", st);
  if (tc && plan.stream_refine) {
    PassDesc p0, pm;
    build_stream_passes(c->n, cap, k, &p0, &pm);
    if (p0.count && !pm.count) {  // the whole corpus fits the lists: score everything once
      SDB_TRY(screen_tc_pass(c, s, r.filt, nq, k, p0, int8, 0, st, v));
      SDB_CUDA(cudaEventRecord(t.ev_main, st));
      c->last_main = t.ev_main;
      if (r.tap) SDB_TRY(tap_gathered(s, r.tap, nq, 0u, st));
      SDB_TRY(cand_select(c, s, nq, k, int8, 0u, st));
      e->n_passes++;
    } else if (pm.count) {
      SDB_TRY(screen_tc_pass(c, s, r.filt, nq, k, p0, int8, 3, st, v));  // probe: chunk maxima of a few tiles
      SDB_TRY(cand_seed_from_probe(c, s, nq, k, p0.count, st));       // thresholds + histogram geometry
      trace_mark(ctx, t, "seeded", st);
      SDB_TRY(screen_tc_pass(c, s, r.filt, nq, k, pm, int8, 2, st, v));  // the streaming launch over every tile
      trace_mark(ctx, t, "main_end", st);
      SDB_CUDA(cudaEventRecord(t.ev_main, st));
      c->last_main = t.ev_main;
      if (r.tap) SDB_TRY(tap_gathered(s, r.tap, nq, s.last_slots, st));
      SDB_TRY(cand_select(c, s, nq, k, int8, s.last_slots, st));
      e->n_passes += 2;
    }
  } else {
    const std::vector<PassDesc> passes = build_passes(c->n, cap, nq);
    bool first_pass = true;
    for (const PassDesc& p : passes) {
      if ((t.cancel && *t.cancel) || ctx_cancelled(ctx)) {
        cudaStreamSynchronize(st);
        set_error("query cancelled");
        return SDB_ECANCELLED;
      }
      if (tc) SDB_TRY(screen_tc_pass(c, s, r.filt, nq, k, p, int8, first_pass ? 0 : 1, st, v));
      else if (family(c) == Family::Lp) SDB_TRY(screen_lp_pass(c, s, r.filt, nq, p, st));
      else SDB_TRY(screen_simt_pass(c, s, r.filt, nq, p, st, v));
      if (r.tap) SDB_TRY(tap_gathered(s, r.tap, nq, tc ? s.last_slots : 0u, st));
      SDB_TRY(cand_select(c, s, nq, k, int8, tc ? s.last_slots : 0u, st));
      first_pass = false;
      e->n_passes++;
    }
    SDB_CUDA(cudaEventRecord(t.ev_main, st));
    c->last_main = t.ev_main;
  }
  if (r.tap) SDB_TRY(tap_list(s, nq, &r.tap->list_a, &r.tap->cnt_a, st));
  SDB_CUDA(cudaEventRecord(t.ev_screen1, st));
  trace_mark(ctx, t, "selected", st);
  // stage B: the coarse screens' candidates are re-scored in f32 and narrowed before the (FP64-bound) exact re-rank
  bool refined = false;
  if (tc && plan.exact) {
    SDB_TRY(cand_refine(c, s, nq, st, v));
    if (r.tap) SDB_TRY(tap_list(s, nq, &r.tap->list_r, nullptr, st));
    SDB_TRY(cand_select(c, s, nq, k, false, 0u, st, 1));
    refined = true;
    trace_mark(ctx, t, "refined", st);
  }
  if (r.filt.bits) SDB_TRY(cand_add_specials(c, s, r.filt, nq, st, v));  // each query re-ranks its passing special rows
  SDB_TRY(cand_rerank(c, s, r.filt, nq, st, refined, v));
  trace_mark(ctx, t, "reranked", st);
  SDB_TRY(cand_final(c, s, r.filt, nq, k, t.row_base, r.d_out_rows, r.d_out_dist, r.d_out_count, st, v));
  trace_mark(ctx, t, "final", st);
  SDB_TRY(copy_flags(s, r, st));
  SDB_CUDA(cudaEventRecord(t.ev_end, st));
  trace_mark(ctx, t, "end", st);
  return SDB_OK;
}

// the whole batch at its rung, with what it decided recorded on the ticket
static sdb_status enqueue_ticket(Corpus* c, Ticket& t) {
  const Run r{t.d_queries, t.nq, t.d_out_rows, t.d_out_dist, t.d_out_count, t.filt, t.rung, nullptr,
              t.h_flags, t.h_qflags, t.h_stat};
  Enqueued e;
  SDB_TRY(enqueue_batch(c, t, r, &e));
  t.screen = e.screen;
  t.n_passes = e.n_passes;
  return SDB_OK;
}

static sdb_status copy_out(Corpus* c, Ticket& t) {  // host-buffer entry points: device result -> caller's buffers
  cudaStream_t st = t.stream;
  if (!t.h_out_count) return SDB_OK;
  if (t.k) {
    SDB_CUDA(cudaMemcpyAsync(t.h_out_rows, t.d_fin_rows, sizeof(uint64_t) * (size_t)t.nq * t.k, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaMemcpyAsync(t.h_out_dist, t.d_fin_dist, sizeof(double) * (size_t)t.nq * t.k, cudaMemcpyDeviceToHost, st));
  }
  SDB_CUDA(cudaMemcpyAsync(t.h_out_count, t.d_fin_count, sizeof(uint32_t) * t.nq, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaEventRecord(t.ev_out, st));  // wait() blocks on THIS batch's copies, not on whatever was queued behind it
  return SDB_OK;
}

// rungs the batch's screened queries may climb, which a mixed batch screens on their own (those of the whole batch when
// every query is direct).  0: the batch ran no screen whose counters stay on the device -- exact-only, counted, empty,
// or a mixed batch whose one screened query took the exact kernel -- and the host holds its counters.
static uint32_t screened_rungs(const Ticket& t) {
  return t.plan.rungs(t.n_direct < t.nq ? t.nq - t.n_direct : t.nq);
}

// local (this shard's) part of the completion: ladder re-runs and exact fallbacks.  *repaired = the device result
// changed after the batch's own kernels had produced it.
static sdb_status finish_local(Corpus* c, Ticket& t, uint32_t* n_fallback, bool* repaired) {
  Ctx* ctx = c->ctx;
  cudaStream_t st = t.stream;
  const Plan& p = t.plan;
  const uint32_t nq = t.nq, k = t.k, n_rungs = screened_rungs(t);
  *repaired = false;
  *n_fallback = 0;
  SDB_CUDA(cudaEventSynchronize(t.ev_end));
  if (p.cancel_at_wait && ((t.cancel && *t.cancel) || ctx_cancelled(ctx))) {
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  if (t.screen != SDB_SCREEN_NONE_EXACT && p.exact) {
    while (t.rung + 1 < p.n_batch_rungs) {  // many failures: the whole batch moves up one rung (and stays there)
      uint32_t n_fail = 0;
      for (uint32_t q = 0; q < nq; q++) n_fail += (t.h_flags[q] & 2u) ? 1u : 0u;
      if (n_fail <= 2 + nq / 64) break;
      SDB_CUDA(drain(ctx));  // later batches in flight share scratch sets and the ladder state: drain them first
      t.rung++;
      SDB_TRY(enqueue_ticket(c, t));
      SDB_CUDA(cudaEventSynchronize(t.ev_end));
      *repaired = true;
    }
  }
  if (n_rungs) c->remembered = {p.key, t.rung};
  // ---- what the batch's rung could not prove ----
  std::vector<uint32_t> fails, exacts;
  for (uint32_t q = 0; q < nq; q++) {
    if (t.h_qflags[q] & 1u) exacts.push_back(q);  // zero / non-finite query norm: ranked by the exact kernel
    else if ((t.h_flags[q] & 2u) && (p.exact || t.screen == SDB_SCREEN_NONE_EXACT)) fails.push_back(q);
  }
  if (fails.empty() && exacts.empty()) return SDB_OK;
  SDB_CUDA(drain(ctx));  // the repair below shares scratch (and the exact kernel's keys) with every batch in flight
  // A few failures: only THOSE queries climb the remaining rungs, as a small batch of their own (a bf16 pass over the
  // corpus costs about as much for 60 queries as for 1, and far less than one sequential-f64 pass per query); the f32
  // stream is the last rung.  Whatever is still unproven after that goes to the exact kernel.
  if (!fails.empty() && t.screen != SDB_SCREEN_NONE_EXACT && p.exact && k) {
    for (uint32_t rung = t.rung + 1; rung < n_rungs && !fails.empty(); rung++) {
      if ((t.cancel && *t.cancel) || ctx_cancelled(ctx)) break;
      const uint32_t nf = (uint32_t)fails.size();
      const size_t need_q = (size_t)nf * c->dim, need_o = (size_t)nf * k;
      cudaError_t e = c->d_rp_q.reserve(need_q);
      if (e == cudaSuccess) e = c->rp.reserve(need_o, nf);
      if (e != cudaSuccess) {
        set_error("repair buffers: %s", cudaGetErrorString(e));
        return SDB_ENOMEM;
      }
      for (uint32_t i = 0; i < nf; i++)
        cudaMemcpyAsync(c->d_rp_q + (size_t)i * c->dim, t.d_queries + (size_t)fails[i] * c->dim, sizeof(double) * c->dim, cudaMemcpyDeviceToDevice, st);
      std::vector<uint32_t> rp_qf;  // filtered batch: each gathered query keeps its own filter
      FiltArg filt = t.filt;
      if (t.filt.bits) {
        rp_qf.resize(nf);
        for (uint32_t i = 0; i < nf; i++) rp_qf[i] = t.h_qf[fails[i]];
        e = c->d_rp_qf.reserve(nf);
        if (e == cudaSuccess) e = cudaMemcpyAsync(c->d_rp_qf, rp_qf.data(), sizeof(uint32_t) * nf, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) {
          set_error("repair filter indices: %s", cudaGetErrorString(e));
          return SDB_ECUDA;
        }
        filt.qf = c->d_rp_qf;
      }
      // the failed queries are screened ones (a direct query's proof cannot fail); their flags go to the batch's first
      // entries, which were read above
      const Run rp{c->d_rp_q, nf, c->rp.rows, c->rp.dist, c->rp.count, filt, rung, nullptr, t.h_flags, t.h_qflags,
                   nullptr};
      Enqueued ignored;
      SDB_TRY(enqueue_screened(c, t, rp, &ignored));
      SDB_CUDA(cudaEventSynchronize(t.ev_end));
      std::vector<uint32_t> still;
      for (uint32_t i = 0; i < nf; i++) {
        const uint32_t q = fails[i];
        if ((t.h_flags[i] & 2u) || (t.h_qflags[i] & 1u)) {
          still.push_back(q);
          continue;
        }
        cudaMemcpyAsync(t.d_out_rows + (size_t)q * k, c->rp.rows + (size_t)i * k, sizeof(uint64_t) * k, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(t.d_out_dist + (size_t)q * k, c->rp.dist + (size_t)i * k, sizeof(double) * k, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(t.d_out_count + q, c->rp.count + i, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st);
        t.n_repaired++;
      }
      SDB_CUDA(cudaStreamSynchronize(st));
      fails.swap(still);
      *repaired = true;
    }
  }
  // ---- exact kernel: special queries and whatever no screen could prove ----
  exacts.insert(exacts.end(), fails.begin(), fails.end());
  for (uint32_t q : exacts) {
    if ((t.cancel && *t.cancel) || ctx_cancelled(ctx)) {
      cudaStreamSynchronize(st);
      set_error("query cancelled");
      return SDB_ECANCELLED;
    }
    SDB_TRY(prep_fallback_query(c, t.d_queries + (size_t)q * c->dim, st));
    const uint32_t* q_filter = t.filt.bits ? t.filt.bits + (size_t)t.h_qf[q] * t.filt.words : nullptr;
    SDB_TRY(exact_query(c, c->d_fb_q, c->d_fb_qmag, c->d_fb_qflags, k, t.row_base, t.d_out_rows + (size_t)q * k,
                        t.d_out_dist + (size_t)q * k, t.d_out_count + q, st, q_filter, t.filt.words, p.rank));
    (*n_fallback)++;
    *repaired = true;
  }
  if (*repaired) {
    SDB_TRY(scatter_results(c, t));  // a permuted batch: the repaired results to the caller's positions
    SDB_CUDA(cudaStreamSynchronize(st));
  }
  return SDB_OK;
}

static sdb_status finish_stats(Corpus* c, Ticket& t, uint32_t n_fallback) {
  sdb_knn_stats stt{};
  SDB_CUDA(cudaEventElapsedTime(&stt.screen_ms, t.ev_screen0, t.ev_screen1));
  SDB_CUDA(cudaEventElapsedTime(&stt.total_ms, t.ev_begin, t.ev_end));
  stt.screen_used = (uint32_t)t.screen;
  stt.n_passes = t.n_passes;
  stt.n_fallback = n_fallback;
  stt.n_repaired = t.n_repaired;
  stt.n_special_rows = c->n_special;
  stt.n_candidates = t.h_stat[2];  // largest candidate set of the batch
  stt.n_reranked = t.h_stat[1];
  stt.n_survivors = t.h_stat[3];
  stt.kernel_launches = c->ctx->launches - t.launches0;
  c->stats = stt;
  trace_host(c->ctx, t.id, "waited");
  trace_dump(c->ctx, t);
  return SDB_OK;
}

static Ticket* find_ticket(Corpus* c, uint32_t id) {
  for (Ticket& t : c->tickets)
    if (t.busy && t.id == id) return &t;
  return nullptr;
}
Ticket* claim_ticket(Corpus* c) {
  for (Ticket& t : c->tickets)
    if (!t.busy) return &t;
  set_error("too many batches in flight (%d): call the matching wait first", N_TICKETS);
  return nullptr;
}
static void release_ticket(Ticket& t) {
  t.busy = false;
  t.h_out_rows = nullptr;
  t.h_out_dist = nullptr;
  t.h_out_count = nullptr;
}

// filtered batch (submit_locked, sdb_debug_screen_batch_filtered), on a ticket whose plan is set: the per query filter
// index on the host (exact fallbacks, repairs), the direct / screened split (query indices in batch order) and
// FiltArg::mask_hits
static void plan_filtered(const Corpus* c, Ticket& t, uint32_t nq, const uint32_t* d_filters,
                          const uint32_t* query_filter, const uint64_t* filter_rows, std::vector<uint32_t>* scr,
                          std::vector<uint32_t>* dir) {
  t.h_qf.assign(nq, 0u);
  if (query_filter) std::copy(query_filter, query_filter + nq, t.h_qf.begin());
  t.filt.bits = d_filters;
  t.filt.words = (uint32_t)((c->n + 31) / 32);
  // direct regime: a query whose filter passes at most DIRECT_MAX_ROWS rows (filter_rows: set bits, an upper bound
  // of the rows it passes) skips the screen, where the plan allows it
  const bool direct_ok = filter_rows && t.plan.direct_ok;
  for (uint32_t q = 0; q < nq; q++) {
    const uint64_t rows_q = filter_rows ? filter_rows[t.h_qf[q]] : ~0ull;
    if (direct_ok && rows_q <= DIRECT_MAX_ROWS) dir->push_back(q);
    else {
      scr->push_back(q);
      if (rows_q < c->n / MASK_HITS_DIV) t.filt.mask_hits = 1;  // a selective filter among the screened queries
    }
  }
  t.n_direct = (uint32_t)dir->size();
}

// the batch itself, on a ticket that submit_call has prepared and whose inputs it has staged
static sdb_status submit_locked(Corpus* c, Ticket* t, const double* d_queries, uint32_t nq, uint32_t k, uint64_t row_base,
                                uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                                const volatile int* cancel, const uint32_t* d_filters, const uint32_t* query_filter,
                                const uint64_t* filter_rows, const Ranking& rank) {
  if (!c->finalized) {
    set_error("corpus not finalized (call sdb_corpus_finalize after the last append)");
    return SDB_EINVAL;
  }
  if ((cancel && *cancel) || ctx_cancelled(c->ctx)) {  // the poll of knn_topk.rs:186 before any work is queued
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  {  // slot parity picks the stream and the scratch set: consecutive batches overlap (screen of i+1 || tail of i)
    t->set = (int)(t - c->tickets) & 1;
    t->stream = t->set ? c->ctx->stream2 : c->ctx->stream;
    if (t->wait_h2d) SDB_CUDA(cudaStreamWaitEvent(t->stream, t->ev_h2d, 0));
    t->wait_h2d = false;
  }
  t->id = c->next_ticket++;
  if (c->next_ticket == 0) c->next_ticket = 1;
  t->d_queries = d_queries;
  t->nq = nq;
  t->k = k;
  t->row_base = row_base;
  t->d_fin_rows = t->d_out_rows = d_out_rows;
  t->d_fin_dist = t->d_out_dist = d_out_dist;
  t->d_fin_count = t->d_out_count = d_out_count;
  t->filt = FiltArg();
  t->n_direct = 0;
  t->permuted = false;
  t->plan = plan_batch(c, rank, k, nq, c->screen, c->stream_refine);
  const Plan& p = t->plan;
  if (d_filters) {
    std::vector<uint32_t> scr, dir;
    plan_filtered(c, *t, nq, d_filters, query_filter, filter_rows, &scr, &dir);
    if (!dir.empty() && !scr.empty()) {  // mixed: run permuted, screened queries first (see Ticket::permuted)
      std::vector<uint32_t> perm(scr);
      perm.insert(perm.end(), dir.begin(), dir.end());
      std::vector<uint32_t> qf(nq);
      for (uint32_t i = 0; i < nq; i++) qf[i] = t->h_qf[perm[i]];
      t->h_qf.swap(qf);
      SDB_CUDA(t->d_perm.reserve(nq));
      SDB_CUDA(t->d_pq.reserve((size_t)nq * c->dim));
      SDB_CUDA(t->pres.reserve((size_t)nq * k, nq));
      SDB_CUDA(cudaMemcpyAsync(t->d_perm, perm.data(), sizeof(uint32_t) * nq, cudaMemcpyHostToDevice, t->stream));
      gather_queries_kernel<<<nq, 128, 0, t->stream>>>(d_queries, t->d_perm, c->dim, t->d_pq);
      count_launch(c->ctx);
      SDB_CUDA(cudaGetLastError());
      t->permuted = true;
      t->d_queries = t->d_pq;
      t->d_out_rows = t->pres.rows;
      t->d_out_dist = t->pres.dist;
      t->d_out_count = t->pres.count;
    }
    SDB_CUDA(t->d_qf.reserve(nq ? nq : 1));
    if (nq) SDB_CUDA(cudaMemcpyAsync(t->d_qf, t->h_qf.data(), sizeof(uint32_t) * nq, cudaMemcpyHostToDevice, t->stream));
    t->filt.qf = t->d_qf;
  }
  t->cancel = cancel;
  t->launches0 = c->ctx->launches;
  t->n_repaired = 0;
  t->rung = c->remembered.key == p.key && c->remembered.rung < p.n_batch_rungs ? c->remembered.rung : 0;
  if (p.route == Plan::Route::Empty) {  // nothing to search: counts are zero
    cudaStream_t st = t->stream;
    SDB_CUDA(cudaEventRecord(t->ev_begin, st));
    SDB_CUDA(cudaEventRecord(t->ev_screen0, st));
    SDB_CUDA(cudaEventRecord(t->ev_screen1, st));
    if (nq) SDB_CUDA(cudaMemsetAsync(d_out_count, 0, sizeof(uint32_t) * nq, st));
    for (uint32_t q = 0; q < nq; q++) t->h_flags[q] = t->h_qflags[q] = 0;
    t->h_stat[0] = t->h_stat[1] = t->h_stat[2] = t->h_stat[3] = 0;
    t->screen = SDB_SCREEN_NONE_EXACT;
    t->n_passes = 0;
    SDB_CUDA(cudaEventRecord(t->ev_end, st));
    t->busy = true;
    return SDB_OK;
  }
  sdb_status rc = enqueue_ticket(c, *t);
  if (rc == SDB_OK) rc = scatter_results(c, *t);
  if (rc == SDB_OK) t->busy = true;
  trace_host(c->ctx, t->id, "submitted");
  return rc;
}

static sdb_status wait_locked(Corpus* c, Ticket* t) {
  uint32_t n_fb = 0;
  bool repaired = false;
  sdb_status rc = finish_local(c, *t, &n_fb, &repaired);
  if (rc == SDB_OK && t->h_out_count) {
    if (repaired) rc = copy_out(c, *t);  // the copies enqueued at submit time predate the repair
    if (rc == SDB_OK && cudaEventSynchronize(t->ev_out) != cudaSuccess) {
      set_error("sdb_knn_wait: %s", cudaGetErrorString(cudaGetLastError()));
      rc = SDB_ECUDA;
    }
  }
  if (rc == SDB_OK) rc = finish_stats(c, *t, n_fb);
  release_ticket(*t);
  return rc;
}

// ---- hooks for comm.cu (sharded search).  The caller holds c->mu. ---------------------------------------------------
void knn_trace_mark(Corpus* c, uint32_t ticket, const char* name) {
  Ticket* t = find_ticket(c, ticket);
  if (t) trace_mark(c->ctx, *t, name, t->stream);
}
cudaStream_t knn_ticket_stream(Corpus* c, uint32_t ticket) {
  Ticket* t = find_ticket(c, ticket);
  return t ? t->stream : c->ctx->stream;
}
sdb_status knn_finish_for_shard(Corpus* c, uint32_t ticket, bool* repaired) {
  Ticket* t = find_ticket(c, ticket);
  if (!t) return SDB_EINVAL;
  uint32_t n_fb = 0;
  SDB_TRY(finish_local(c, *t, &n_fb, repaired));
  return finish_stats(c, *t, n_fb);
}
sdb_status knn_release_ticket(Corpus* c, uint32_t ticket) {
  Ticket* t = find_ticket(c, ticket);
  if (!t) return SDB_EINVAL;
  release_ticket(*t);
  return SDB_OK;
}
// a permuted batch's counters: queries flagged by both sub-batches, the rest as the direct sub-batch left them
__global__ void sum_flagged_kernel(const uint32_t* __restrict__ direct, const uint32_t* __restrict__ screened,
                                   uint32_t* __restrict__ out) {
  if (threadIdx.x < 4) out[threadIdx.x] = direct[threadIdx.x] + (threadIdx.x == 0 ? screened[0] : 0u);
}
// the 16-byte block header of a sharded batch, enqueued on its stream: [0] = queries this shard must still repair on
// the host (failed proof, special queries), [1..3] the batch's other counters (d_stat)
sdb_status knn_shard_header(Corpus* c, uint32_t ticket, void* d_hdr) {
  Ticket* t = find_ticket(c, ticket);
  if (!t) return SDB_EINVAL;
  cudaStream_t st = t->stream;
  if (screened_rungs(*t) == 0) {  // the counters the host holds
    SDB_CUDA(cudaMemcpyAsync(d_hdr, t->h_stat, 16, cudaMemcpyHostToDevice, st));
  } else if (t->permuted) {
    sum_flagged_kernel<<<1, 32, 0, st>>>(c->sets[t->set].d_stat, t->d_stat_scr, (uint32_t*)d_hdr);
    count_launch(c->ctx);
    SDB_CUDA(cudaGetLastError());
  } else {
    SDB_CUDA(cudaMemcpyAsync(d_hdr, c->sets[t->set].d_stat, 16, cudaMemcpyDeviceToDevice, st));
  }
  return SDB_OK;
}

// ---- global top-k merge of per-shard lists (after the NCCL all-gather) -----------------------------
// Both merges order the entries by (order_key(value, DESC), global row): DESC = false is KNN's (distance, row) order and
// the ascending ORDER BY ranking, DESC = true the descending one (sdb_corpus_order_sharded_*).  Each list must already
// be in that order.  Padding and exhausted lists take key ~0 and row ~0: order_key never yields ~0 for DESC, and for
// ASC the row still sets the sentinel apart from the all-ones NaN.  The value carried through is the one the shard
// returned, so -0.0 stays -0.0.
template <bool DESC>
__global__ void __launch_bounds__(1024) topk_merge_kernel(uint32_t n_lists, uint32_t nq, uint32_t k,
                                                          const uint64_t* __restrict__ rows,
                                                          const double* __restrict__ dist,
                                                          const uint32_t* __restrict__ counts, uint64_t st_rows,
                                                          uint64_t st_dist, uint64_t st_cnt,
                                                          uint64_t* __restrict__ out_rows, double* __restrict__ out_dist,
                                                          uint32_t* __restrict__ out_count) {
  extern __shared__ uint64_t s_mem[];
  const uint32_t q = blockIdx.x;
  const uint32_t total = n_lists * k;
  uint32_t p2 = 1;
  while (p2 < total) p2 <<= 1;
  uint64_t* s_key = s_mem;
  uint64_t* s_row = s_mem + p2;
  double* s_d = reinterpret_cast<double*>(s_mem + 2 * p2);
  __shared__ uint32_t s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
    uint64_t key = ~0ull, row = ~0ull;
    double d = 0.0;
    if (i < total) {
      const uint32_t l = i / k, j = i % k;
      if (j < counts[(size_t)l * st_cnt + q]) {
        const size_t o = (size_t)q * k + j;
        d = dist[(size_t)l * st_dist + o];
        key = order_key(d, DESC);
        row = rows[(size_t)l * st_rows + o];
        atomicAdd(&s_n, 1u);
      }
    }
    s_key[i] = key;
    s_row[i] = row;
    s_d[i] = d;
  }
  __syncthreads();
  for (uint32_t kk = 2; kk <= p2; kk <<= 1)
    for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const uint64_t ka = s_key[i], kb = s_key[ixj], ra = s_row[i], rb = s_row[ixj];
          const bool a_gt_b = ka > kb || (ka == kb && ra > rb);
          const bool up = ((i & kk) == 0);
          if (up ? a_gt_b : !a_gt_b) {
            s_key[i] = kb; s_key[ixj] = ka;
            s_row[i] = rb; s_row[ixj] = ra;
            const double da = s_d[i];
            s_d[i] = s_d[ixj];
            s_d[ixj] = da;
          }
        }
      }
      __syncthreads();
    }
  const uint32_t n_out = s_n < k ? s_n : k;
  for (uint32_t i = threadIdx.x; i < n_out; i += blockDim.x) {
    out_rows[(size_t)q * k + i] = s_row[i];
    out_dist[(size_t)q * k + i] = s_d[i];
  }
  if (threadIdx.x == 0) out_count[q] = n_out;
}


// <= 32 lists: one warp per query, lane l walks list l (each list is already in (order key, row) order).  Every step
// takes the warp-wide minimum head.  No shared memory and 128-thread blocks, so the merge runs beside the resident screen
// of the next batch (the sorter above needs 24 bytes of shared memory per entry and up to 1024 threads).
template <bool DESC>
__global__ void __launch_bounds__(128) topk_kway_merge_kernel(uint32_t n_lists, uint32_t nq, uint32_t k,
                                                              const uint64_t* __restrict__ rows,
                                                              const double* __restrict__ dist,
                                                              const uint32_t* __restrict__ counts, uint64_t st_rows,
                                                              uint64_t st_dist, uint64_t st_cnt,
                                                              uint64_t* __restrict__ out_rows, double* __restrict__ out_dist,
                                                              uint32_t* __restrict__ out_count) {
  const uint32_t q = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (q >= nq) return;
  uint32_t cnt = 0, pos = 0;
  const uint64_t* lr = nullptr;
  const double* ld = nullptr;
  if (lane < n_lists) {
    cnt = counts[(size_t)lane * st_cnt + q];
    if (cnt > k) cnt = k;
    lr = rows + (size_t)lane * st_rows + (size_t)q * k;
    ld = dist + (size_t)lane * st_dist + (size_t)q * k;
  }
  uint64_t key = ~0ull, row = ~0ull;
  double d = 0.0;
  if (pos < cnt) {
    d = ld[0];
    key = order_key(d, DESC);
    row = lr[0];
  }
  uint32_t n_out = 0;
  for (; n_out < k; n_out++) {
    uint64_t bk = key, br = row;
    uint32_t bl = lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t ok = __shfl_xor_sync(0xffffffffu, bk, o), orow = __shfl_xor_sync(0xffffffffu, br, o);
      const uint32_t ol = __shfl_xor_sync(0xffffffffu, bl, o);
      if (ok < bk || (ok == bk && (orow < br || (orow == br && ol < bl)))) {
        bk = ok;
        br = orow;
        bl = ol;
      }
    }
    if (bk == ~0ull && br == ~0ull) break;  // every list exhausted
    if (lane == bl) {
      out_rows[(size_t)q * k + n_out] = row;
      out_dist[(size_t)q * k + n_out] = d;
      pos++;
      if (pos < cnt) {
        d = ld[pos];
        key = order_key(d, DESC);
        row = lr[pos];
      } else {
        key = ~0ull;
        row = ~0ull;
      }
    }
  }
  if (lane == 0) out_count[q] = n_out;
}

sdb_status topk_merge_launch(Ctx* ctx, uint32_t n_lists, uint32_t nq, uint32_t k, const uint64_t* d_rows,
                             const double* d_dist, const uint32_t* d_counts, uint64_t stride_rows, uint64_t stride_dist,
                             uint64_t stride_counts, uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                             bool desc, cudaStream_t st) {
  if (!stride_rows) stride_rows = (uint64_t)nq * k;
  if (!stride_dist) stride_dist = (uint64_t)nq * k;
  if (!stride_counts) stride_counts = nq;
  if (n_lists <= 32) {
    auto kway = desc ? topk_kway_merge_kernel<true> : topk_kway_merge_kernel<false>;
    kway<<<(nq + 3) / 4, 128, 0, st>>>(n_lists, nq, k, d_rows, d_dist, d_counts, stride_rows, stride_dist, stride_counts,
                                       d_out_rows, d_out_dist, d_out_count);
    count_launch(ctx);
    SDB_CUDA(cudaGetLastError());
    return SDB_OK;
  }
  uint32_t p2 = 1;
  while (p2 < n_lists * k) p2 <<= 1;
  const size_t smem = (size_t)p2 * 24;
  if (smem > 200 * 1024) {
    set_error("merge of %u lists x k=%u exceeds the shared-memory sorter", n_lists, k);
    return SDB_EUNSUPPORTED;
  }
  const uint32_t threads = p2 >= 1024 ? 1024 : (p2 < 64 ? 64 : p2);
  auto sorter = desc ? topk_merge_kernel<true> : topk_merge_kernel<false>;
  sorter<<<nq, threads, smem, st>>>(n_lists, nq, k, d_rows, d_dist, d_counts, stride_rows, stride_dist, stride_counts,
                                    d_out_rows, d_out_dist, d_out_count);
  count_launch(ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

}  // namespace sdb

using namespace sdb;

extern "C" {

const char* sdb_last_error(void) { return g_err; }
const char* sdb_version(void) { return "sdbgpu 0.1.0 (sm_90a)"; }

sdb_status sdb_ctx_create(int device, sdb_ctx** out) {
  if (!out) return SDB_EINVAL;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device available (%s); this library has no CPU fallback", cudaGetErrorString(e));
    return SDB_ECUDA;
  }
  if (device < 0 || device >= n) {
    set_error("device %d out of range (0..%d)", device, n - 1);
    return SDB_EINVAL;
  }
  cudaDeviceProp prop;
  SDB_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; this library ships sm_90a code only", device, prop.major, prop.minor);
    return SDB_ECUDA;
  }
  SDB_CUDA(cudaSetDevice(device));
  sdb_ctx* c = new sdb_ctx();
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  {
    int least = 0, greatest = 0;
    if (cudaDeviceGetStreamPriorityRange(&least, &greatest) == cudaSuccess) c->prio_high = greatest;
  }
  SDB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  SDB_CUDA(cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking));
  SDB_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  {
    SDB_CUDA(c->h_cancel.reserve(1, nullptr, cudaHostAllocMapped));
    *c->h_cancel = 0;
    SDB_CUDA(c->d_cancel.reserve(1));
    SDB_CUDA(cudaMemset(c->d_cancel, 0, sizeof(int)));
    SDB_CUDA(cudaStreamCreateWithFlags(&c->cancel_stream, cudaStreamNonBlocking));
  }
  // dynamic shared-memory limits are per device: set them for THIS device now (not behind a process-wide flag)
  SDB_TRY(screen_tc_init_device(c));
  SDB_TRY(candidates_init_device());
  SDB_TRY(exact_init_device());
  SDB_CUDA(cudaFuncSetAttribute(topk_merge_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  SDB_CUDA(cudaFuncSetAttribute(topk_merge_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  {  // keep stream-ordered allocations cached in the pool instead of returning them to the OS at every sync
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
  }
  *out = c;
  return SDB_OK;
}
void sdb_ctx_destroy(sdb_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  comm_destroy(c);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->stream2) cudaStreamDestroy(c->stream2);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->cancel_stream) cudaStreamDestroy(c->cancel_stream);
  delete c;
}
static void push_cancel_word(sdb_ctx* c) {  // any host thread; its own stream, so it overtakes running kernels
  if (!c->d_cancel || !c->cancel_stream) return;
  if (cudaSetDevice(c->device) != cudaSuccess) return;
  cudaMemcpyAsync(c->d_cancel, (const void*)c->h_cancel.get(), sizeof(int), cudaMemcpyHostToDevice, c->cancel_stream);
  cudaStreamSynchronize(c->cancel_stream);
}
void sdb_ctx_cancel(sdb_ctx* c) {
  if (!c || !c->h_cancel) return;
  *c->h_cancel = 1;
  push_cancel_word(c);
}
void sdb_ctx_cancel_reset(sdb_ctx* c) {
  if (!c || !c->h_cancel) return;
  *c->h_cancel = 0;
  push_cancel_word(c);
}
uint64_t sdb_ctx_kernel_launches(const sdb_ctx* c) { return c ? c->launches : 0; }
void* sdb_ctx_stream(const sdb_ctx* c) { return c ? (void*)c->stream : nullptr; }
void* sdb_pinned_alloc(size_t bytes) {
  PinnedBuf<uint8_t> p;
  if (p.reserve(bytes) != cudaSuccess) {
    set_error("cudaHostAlloc(%zu) failed", bytes);
    return nullptr;
  }
  return p.release();
}
void sdb_pinned_free(void* p) {
  if (p) PinnedBuf<uint8_t>::free_released(p);
}
void sdb_free(void* p) { free(p); }

sdb_status sdb_corpus_create(sdb_ctx* ctx, uint32_t dim, sdb_dtype dt, sdb_metric m, uint64_t cap, sdb_corpus** out) {
  if (!ctx || !out || dim == 0 || dim > 65535 || cap == 0 || cap >= 0xFFFFFFF0ull) {
    set_error("sdb_corpus_create: bad argument (dim 1..65535, 0 < capacity < 2^32)");
    return SDB_EINVAL;
  }
  // The buffers of each metric's family (Family, internal.cuh): COSINE / EUCLIDEAN the screen copies, PEARSON also
  // the moments, JACCARD the count path's first-occurrence state; the Lp screen and HAMMING's count path read the rows.
  // MINKOWSKI goes through pow(), which CUDA's libm and Rust's (the platform libm) implement separately: within 1 ulp of
  // each other per term, so its distances are compared with a 1e-12 relative tolerance instead of bit equality with the
  // CPU oracle (tests/test_gpu_knn.py).
  const bool screenable = m == SDB_COSINE || m == SDB_EUCLIDEAN;
  if ((int)m < 0 || (int)m > (int)SDB_PEARSON) {
    set_error("unknown metric %d", (int)m);
    return SDB_EINVAL;
  }
  if (dt != SDB_F32 && dt != SDB_F64) return SDB_EINVAL;
  SDB_CUDA(cudaSetDevice(ctx->device));
  sdb_corpus* c = new sdb_corpus();
  c->ctx = ctx;
  c->dim = dim;
  c->dim_pad = (dim + 63) / 64 * 64;
  c->dim_pad8 = (dim + 127) / 128 * 128;
  c->dtype = dt;
  c->metric = m;
  c->cap = cap;
  const size_t esz = dt == SDB_F32 ? 4 : 8;
  const uint64_t cap_pad = (cap + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
  cudaError_t e = c->d_rows.reserve(esz * cap * dim);
  if (e == cudaSuccess) e = c->d_mag.reserve(cap);
  if (e == cudaSuccess) e = c->d_snorm.reserve(cap_pad);
  if (e == cudaSuccess && dt == SDB_F32 && screenable) e = c->d_bf16.reserve(cap_pad * c->dim_pad);
  if (e == cudaSuccess && dt == SDB_F32 && m == SDB_COSINE) e = c->d_i8.reserve((size_t)cap_pad * c->dim_pad8);
  if (e != cudaSuccess) {
    set_error("corpus allocation failed: %s", cudaGetErrorString(e));
    sdb_corpus_destroy(c);
    return SDB_ENOMEM;
  }
  // f64 rows get the same screen copies (3 more bytes per element beside their 8), but only when they fit: an f64
  // corpus without them is still served, by the exact kernel alone, as before they existed
  if (dt == SDB_F64 && screenable) {
    cudaError_t e2 = c->d_bf16.reserve(cap_pad * c->dim_pad);
    if (e2 == cudaSuccess && m == SDB_COSINE) e2 = c->d_i8.reserve((size_t)cap_pad * c->dim_pad8);
    if (e2 != cudaSuccess) {
      c->d_bf16.reset();
      c->d_i8.reset();
    }
  }
  // PEARSON (f32 and f64 rows): the cosine screens run on the centred rows, which takes the bf16 and int8 copies and
  // 16 bytes of moments per row -- again only when they fit
  if (m == SDB_PEARSON) {
    cudaError_t e2 = c->d_bf16.reserve(cap_pad * c->dim_pad);
    if (e2 == cudaSuccess) e2 = c->d_i8.reserve((size_t)cap_pad * c->dim_pad8);
    if (e2 == cudaSuccess) e2 = c->d_mom.reserve(cap);
    if (e2 != cudaSuccess) {
      c->d_bf16.reset();
      c->d_i8.reset();
      c->d_mom.reset();
    }
  }
  // JACCARD: the count path's first-occurrence bitmask (one bit per element) and distinct-value count per row, 4 bytes
  // per 32 elements plus 4 per row -- only when they fit; without them the exact kernel ranks the corpus
  if (m == SDB_JACCARD) {
    cudaError_t e2 = c->d_jfirst.reserve((size_t)cap * ((dim + 31) / 32));
    if (e2 == cudaSuccess) e2 = c->d_jux.reserve(cap);
    if (e2 != cudaSuccess) {
      c->d_jfirst.reset();
      c->d_jux.reset();
    }
  }
  *out = c;
  return SDB_OK;
}
void sdb_corpus_destroy(sdb_corpus* c) {
  if (!c) return;
  cudaSetDevice(c->ctx->device);
  drain(c->ctx);
  comm_corpus_released(c);
  for (Ticket& t : c->tickets) {
    cudaEvent_t evs[] = {t.ev_begin, t.ev_screen0, t.ev_screen1, t.ev_end, t.ev_h2d, t.ev_out, t.ev_main};
    for (cudaEvent_t e : evs)
      if (e) cudaEventDestroy(e);
  }
  delete c;
}
uint64_t sdb_corpus_rows(const sdb_corpus* c) { return c ? c->n : 0; }

static sdb_status append_common(sdb_corpus* c, const void* src, uint64_t n, cudaMemcpyKind kind) {
  if (!c || (!src && n)) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (c->n + n > c->cap) {
    set_error("append of %llu rows exceeds capacity %llu", (unsigned long long)n, (unsigned long long)c->cap);
    return SDB_EOVERFLOW;
  }
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  const size_t esz = c->dtype == SDB_F32 ? 4 : 8;
  SDB_CUDA(cudaMemcpyAsync((char*)c->d_rows.get() + esz * c->n * c->dim, src, esz * n * c->dim, kind, c->ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  c->n += n;
  c->finalized = false;
  return SDB_OK;
}
sdb_status sdb_corpus_append(sdb_corpus* c, const void* rows, uint64_t n) {
  return append_common(c, rows, n, cudaMemcpyHostToDevice);
}
sdb_status sdb_corpus_append_device(sdb_corpus* c, const void* d_rows, uint64_t n) {
  return append_common(c, d_rows, n, cudaMemcpyDeviceToDevice);
}
sdb_status sdb_corpus_append_synthetic(sdb_corpus* c, uint64_t seed, uint64_t first_row, uint64_t n) {
  if (!c) return SDB_EINVAL;
  if (c->dtype != SDB_F32) {
    set_error("synthetic rows are f32");
    return SDB_EUNSUPPORTED;
  }
  std::lock_guard<std::mutex> g(c->mu);
  if (c->n + n > c->cap) return SDB_EOVERFLOW;
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  SDB_TRY(gen_fill_f32(c->ctx, (float*)c->d_rows.get() + c->n * c->dim, seed, first_row * c->dim, n * c->dim, c->ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  c->n += n;
  c->finalized = false;
  return SDB_OK;
}
sdb_status sdb_corpus_set_skip(sdb_corpus* c, const uint8_t* skip, uint64_t n) {
  if (!c || n > c->cap) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  if (!skip) {
    c->d_skip.reset();
  } else {
    SDB_CUDA(c->d_skip.reserve(c->cap));
    SDB_CUDA(cudaMemsetAsync(c->d_skip, 0, c->cap, c->ctx->stream));
    SDB_CUDA(cudaMemcpyAsync(c->d_skip, skip, n, cudaMemcpyHostToDevice, c->ctx->stream));
  }
  SDB_TRY(corpus_reapply_tombstones(c, c->ctx->stream));  // rows removed earlier stay removed
  SDB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  c->finalized = false;
  return SDB_OK;
}
sdb_status sdb_corpus_remove(sdb_corpus* c, const uint64_t* row_ids, uint64_t n) {
  if (!c || (n && !row_ids)) return SDB_EINVAL;
  if (n == 0) return SDB_OK;
  std::lock_guard<std::mutex> g(c->mu);
  for (uint64_t i = 0; i < n; i++)
    if (row_ids[i] >= c->n) {
      set_error("sdb_corpus_remove: row %llu outside the corpus (%llu rows)", (unsigned long long)row_ids[i],
                (unsigned long long)c->n);
      return SDB_EINVAL;
    }
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  SDB_CUDA(drain(c->ctx));  // no batch may be in flight while rows disappear
  SDB_TRY(corpus_remove_device(c, row_ids, n));
  c->n_removed += n;
  return SDB_OK;
}
sdb_status sdb_corpus_finalize(sdb_corpus* c) {
  if (!c) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  return corpus_finalize_device(c);
}
sdb_status sdb_corpus_set_screen(sdb_corpus* c, sdb_screen s) {
  if (!c || (int)s < 0 || (int)s > 4) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  c->screen = s;
  return SDB_OK;
}
sdb_status sdb_corpus_read_rows(sdb_corpus* c, uint64_t first_row, uint64_t n, void* out) {
  if (!c || (!out && n)) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (first_row > c->n || n > c->n - first_row) {
    set_error("sdb_corpus_read_rows: rows %llu..%llu outside the corpus (%llu rows)", (unsigned long long)first_row,
              (unsigned long long)(first_row + n), (unsigned long long)c->n);
    return SDB_EINVAL;
  }
  if (n == 0) return SDB_OK;
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  const size_t esz = c->dtype == SDB_F32 ? 4 : 8;
  SDB_CUDA(cudaMemcpyAsync(out, (const char*)c->d_rows.get() + esz * first_row * c->dim, esz * n * c->dim,
                           cudaMemcpyDeviceToHost, c->ctx->copy_stream));
  SDB_CUDA(cudaStreamSynchronize(c->ctx->copy_stream));
  return SDB_OK;
}
sdb_status sdb_corpus_set_minkowski_order(sdb_corpus* c, double order) {
  if (!c || !(order == order)) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  c->minkowski_p = order;
  return SDB_OK;
}
sdb_status sdb_corpus_set_schedule(sdb_corpus* c, int streaming) {
  if (!c) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  c->stream_refine = streaming != 0;
  return SDB_OK;
}
sdb_status sdb_corpus_set_exact(sdb_corpus* c, int exact) {
  if (!c) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  c->exact = exact != 0;
  return SDB_OK;
}
sdb_status sdb_knn_last_stats(const sdb_corpus* c, sdb_knn_stats* out) {
  if (!c || !out) return SDB_EINVAL;
  *out = c->stats;
  return SDB_OK;
}

// ---- staging of a batch's inputs -----------------------------------------------------------------------------------
// per filter used by the batch, on the host, as far as the two decisions need it, over the bits [first, first + n_rows)
// of bitmaps of `words` words (a shard's rows of global bitmaps; unsharded calls: 0 and the corpus' rows): the exact
// number of set bits while it is at most DIRECT_MAX_ROWS (direct regime; the count stops at the first bit beyond, after
// ~T / 32 / density words, and all-zero words cost one compare), else an estimate from 4096 evenly spaced words, which
// only decides FiltArg::mask_hits (a speed switch; either value gives the same results)
static std::vector<uint64_t> count_filter_rows_host(const uint32_t* filters, uint64_t words, uint64_t first,
                                                    uint64_t n_rows, uint32_t n_filters, const uint32_t* query_filter,
                                                    uint32_t nq) {
  const uint64_t w0 = first / 32, w1 = (first + n_rows + 31) / 32;  // the words holding the range
  const uint32_t end = (uint32_t)((first + n_rows) & 31u);
  const uint32_t m0 = ~0u << (first & 31u), m1 = end ? ~0u >> (32u - end) : ~0u;  // its bits in the first / last word
  std::vector<uint64_t> cnt(n_filters, ~0ull);
  for (uint32_t q = 0; q < nq; q++) {
    const uint32_t f = query_filter ? query_filter[q] : 0u;
    if (cnt[f] != ~0ull) continue;
    const uint32_t* b = filters + (size_t)f * words;
    uint64_t n = 0;
    for (uint64_t w = w0; w < w1 && n <= DIRECT_MAX_ROWS; w++) {
      const uint32_t v = b[w] & (w == w0 ? m0 : ~0u) & (w == w1 - 1 ? m1 : ~0u);
      if (v) n += (uint64_t)__builtin_popcount(v);
    }
    if (n > DIRECT_MAX_ROWS) {
      const uint64_t samples = std::min<uint64_t>(w1 - w0, 4096), step = (w1 - w0) / samples;
      uint64_t s = 0;
      for (uint64_t i = 0; i < samples; i++) s += (uint64_t)__builtin_popcount(b[w0 + i * step]);
      n = std::max<uint64_t>(DIRECT_MAX_ROWS + 1, s * step);  // estimate, never below the direct bound
    }
    cnt[f] = n;
  }
  return cnt;
}
__global__ void count_filter_rows_kernel(const uint32_t* __restrict__ bits, uint64_t words,
                                         unsigned long long* __restrict__ cnt) {
  const uint32_t* b = bits + (size_t)blockIdx.y * words;
  unsigned long long n = 0;
  for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < words; w += (uint64_t)gridDim.x * blockDim.x)
    n += (unsigned long long)__popc(__ldg(b + w));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31u) == 0 && n) atomicAdd(cnt + blockIdx.y, n);
}
// A shard's part of global bitmaps (sharded filtered calls): bits [row_base, row_base + n) of each as a local bitmap of
// ceil(n / 32) words, bit r = the shard's row r.  src: word row_base / 32 of filter 0's bitmap, filters `pitch` words
// apart, `avail` words of each readable from there; shift = row_base % 32.  The bits past the shard's last row belong
// to the next shard's rows and are cleared: the screens' padding rows must never pass.  cnt (nullable, zeroed): set
// bits per filter.
__global__ void slice_filter_rows_kernel(const uint32_t* __restrict__ src, uint64_t pitch, uint64_t avail,
                                         uint32_t shift, uint64_t n, uint32_t n_filters, uint32_t* __restrict__ dst,
                                         unsigned long long* __restrict__ cnt) {
  const uint64_t words = (n + 31) / 32;
  const uint32_t tail = (uint32_t)(n & 31u);
  for (uint32_t f = blockIdx.y; f < n_filters; f += gridDim.y) {
    const uint32_t* s = src + (size_t)f * pitch;
    unsigned long long c = 0;
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < words; w += (uint64_t)gridDim.x * blockDim.x) {
      const uint32_t lo = __ldg(s + w), hi = w + 1 < avail ? __ldg(s + w + 1) : 0u;
      uint32_t v = __funnelshift_r(lo, hi, shift);
      if (tail && w == words - 1) v &= (1u << tail) - 1u;
      dst[(size_t)f * words + w] = v;
      c += (unsigned long long)__popc(v);
    }
    if (cnt) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if ((threadIdx.x & 31u) == 0 && c) atomicAdd(cnt + f, c);
    }
  }
}

}  // extern "C"
namespace sdb {

sdb_status check_filters(uint32_t nq, const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter) {
  if (nq && (n_filters == 0 || !filters)) {
    set_error("filtered KNN: %s", n_filters == 0 ? "no filter given (n_filters == 0)" : "filters is NULL");
    return SDB_EINVAL;
  }
  if (query_filter)
    for (uint32_t q = 0; q < nq; q++)
      if (query_filter[q] >= n_filters) {
        set_error("filtered KNN: query %u uses filter %u of %u", q, query_filter[q], n_filters);
        return SDB_EINVAL;
      }
  return SDB_OK;
}

// The bitmaps of a filtered batch as its kernels read them (*bits: ceil(c->n / 32) words per filter, bit r = the
// corpus' row r) and the set bits of each for plan_filtered (*rows), enqueued on the copy stream, which carries no batch.
//   unsharded call: host bitmaps are copied whole into the slot's d_in_filt; device bitmaps are read in place
//   sharded call: only the shard's span of each global bitmap is read, words row_base / 32 .. (row_base + n) / 32 + 1
//     (host bitmaps: one strided copy into d_in_span), and slice_filter_rows_kernel shifts it into d_in_filt
// Host bitmaps are counted on the host.  Device bitmaps are counted on the device, and the host waits for that count
// alone -- an event on the copy stream, never a batch stream, so a batch in flight keeps running.  The caller records
// ev_h2d on the copy stream afterwards; the batch's stream waits for it.
static sdb_status stage_filters(Corpus* c, Ticket& t, const RowFilters& rf, bool host, uint32_t nq,
                                const uint32_t** bits, std::vector<uint64_t>* rows) {
  cudaStream_t cs = c->ctx->copy_stream;
  const uint32_t nf = rf.n_filters;
  const bool sharded = rf.n_rows_total != 0;
  const uint64_t words = (c->n + 31) / 32;
  const uint64_t W = sharded ? (rf.n_rows_total + 31) / 32 : words;  // words of each bitmap the caller holds
  const uint64_t first = sharded ? c->row_base : 0;
  *bits = rf.bits;
  if (host || sharded) {
    SDB_CUDA(t.d_in_filt.reserve(std::max<size_t>(1, (size_t)nf * words)));
    *bits = t.d_in_filt;
  }
  rows->assign(nf, 0);
  if (!words || !nf || !c->finalized) return SDB_OK;  // (submit_locked refuses a corpus that is not finalized)
  if (host && !sharded) {
    SDB_CUDA(cudaMemcpyAsync(t.d_in_filt, rf.bits, sizeof(uint32_t) * nf * words, cudaMemcpyHostToDevice, cs));
    *rows = count_filter_rows_host(rf.bits, W, first, c->n, nf, rf.query_filter, nq);  // while the copy runs
    return SDB_OK;
  }
  unsigned long long* d_cnt = nullptr;
  if (!host) {
    SDB_CUDA(t.d_fcnt.reserve(nf));
    SDB_CUDA(t.h_fcnt.reserve(nf));
    SDB_CUDA(cudaMemsetAsync(t.d_fcnt, 0, sizeof(unsigned long long) * nf, cs));
    d_cnt = t.d_fcnt;
  }
  const uint32_t gx = (uint32_t)std::min<uint64_t>((words + 255) / 256, 64);
  if (sharded) {
    const uint64_t w0 = first / 32, span = std::min(words + 1, W - w0);  // (the last row's word is below W)
    const uint32_t* src = rf.bits + w0;
    uint64_t pitch = W;
    if (host) {  // per rank and batch about 1 / R of the bytes an unsharded filtered call moves
      SDB_CUDA(t.d_in_span.reserve((size_t)nf * span));
      SDB_CUDA(cudaMemcpy2DAsync(t.d_in_span, sizeof(uint32_t) * span, src, sizeof(uint32_t) * W,
                                 sizeof(uint32_t) * span, nf, cudaMemcpyHostToDevice, cs));
      src = t.d_in_span;
      pitch = span;
    }
    slice_filter_rows_kernel<<<dim3(gx, std::min(nf, 65535u)), 256, 0, cs>>>(src, pitch, span, (uint32_t)(first & 31u),
                                                                           c->n, nf, t.d_in_filt, d_cnt);
  } else {
    count_filter_rows_kernel<<<dim3(gx, nf), 256, 0, cs>>>(rf.bits, words, d_cnt);
  }
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  if (host) {
    *rows = count_filter_rows_host(rf.bits, W, first, c->n, nf, rf.query_filter, nq);  // while the slice runs
    return SDB_OK;
  }
  SDB_CUDA(cudaMemcpyAsync(t.h_fcnt, t.d_fcnt, sizeof(unsigned long long) * nf, cudaMemcpyDeviceToHost, cs));
  SDB_CUDA(cudaEventRecord(t.ev_h2d, cs));
  SDB_CUDA(cudaEventSynchronize(t.ev_h2d));
  for (uint32_t f = 0; f < nf; f++) (*rows)[f] = t.h_fcnt[f];
  return SDB_OK;
}

sdb_status submit_call(Corpus* c, Ticket* t, uint32_t nq, uint32_t k, const KnnCall& call) {
  SDB_TRY(ticket_prepare(c, *t, nq ? nq : 1));
  // host inputs travel on the copy stream, so the transfer of batch i+1 overlaps the kernels of batch i
  cudaStream_t cs = c->ctx->copy_stream;
  const double* d_queries = call.queries;
  const bool zero_q = !call.queries && nq;  // an SDB_FN_MAGNITUDE ranking without queries: it reads zero vectors
  if (call.host_in || zero_q) {
    SDB_CUDA(t->d_in_q.reserve(std::max<size_t>(1, (size_t)nq * c->dim)));
    if (call.queries)
      SDB_CUDA(cudaMemcpyAsync(t->d_in_q, call.queries, sizeof(double) * (size_t)nq * c->dim, cudaMemcpyHostToDevice, cs));
    else
      SDB_CUDA(cudaMemsetAsync(t->d_in_q, 0, sizeof(double) * (size_t)nq * c->dim, cs));
    d_queries = t->d_in_q;
  }
  const uint32_t* bits = nullptr;
  std::vector<uint64_t> rows_per_filter;
  if (call.rf.bits) SDB_TRY(stage_filters(c, *t, call.rf, call.host_in, nq, &bits, &rows_per_filter));
  t->wait_h2d = call.host_in || zero_q || call.rf.bits;
  if (t->wait_h2d) SDB_CUDA(cudaEventRecord(t->ev_h2d, cs));
  uint64_t* d_rows = call.out_rows;
  double* d_dist = call.out_dist;
  uint32_t* d_count = call.out_count;
  if (call.host_out) {
    SDB_CUDA(t->res.reserve((size_t)nq * (k ? k : 1), nq));
    d_rows = t->res.rows;
    d_dist = t->res.dist;
    d_count = t->res.count;
  }
  SDB_TRY(submit_locked(c, t, d_queries, nq, k, call.row_base, d_rows, d_dist, d_count, call.cancel, bits,
                        call.rf.query_filter, call.rf.bits ? rows_per_filter.data() : nullptr, call.rank));
  if (!call.host_out) return SDB_OK;
  t->h_out_rows = call.out_rows;
  t->h_out_dist = call.out_dist;
  t->h_out_count = call.out_count;
  const sdb_status rc = copy_out(c, *t);
  if (rc != SDB_OK) {
    cudaStreamSynchronize(t->stream);
    release_ticket(*t);
  }
  return rc;
}

// the sdb_knn_{bruteforce,submit}* entry points after their own argument checks: one batch, then its wait (blocking
// calls: ticket == nullptr) or its ticket id
static sdb_status knn_call(Corpus* c, uint32_t nq, uint32_t k, const KnnCall& call, uint32_t* ticket) {
  std::lock_guard<std::mutex> g(c->mu);
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  Ticket* t = claim_ticket(c);
  if (!t) return SDB_EOVERFLOW;
  SDB_TRY(submit_call(c, t, nq, k, call));
  if (!ticket) return wait_locked(c, t);
  *ticket = t->id;
  return SDB_OK;
}
static KnnCall host_call(Corpus* c, const double* queries, const RowFilters& rf, uint64_t* out_rows, double* out_dist,
                         uint32_t* out_count, const volatile int* cancel) {
  return KnnCall{queries, true, rf, c->row_base, out_rows, out_dist, out_count, true, cancel};
}
static KnnCall device_call(const double* d_queries, const RowFilters& rf, uint64_t row_base, uint64_t* d_out_rows,
                           double* d_out_dist, uint32_t* d_out_count) {
  return KnnCall{d_queries, false, rf, row_base, d_out_rows, d_out_dist, d_out_count, false, nullptr};
}

// ---- ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k: the argument checks of sdb_corpus_order_* (unsharded and
// sharded alike)
static bool vector_fn_known(int fn) {
  return (fn >= (int)SDB_CHEBYSHEV && fn <= (int)SDB_PEARSON) || fn == SDB_FN_SIMILARITY_COSINE || fn == SDB_FN_DOT ||
         fn == SDB_FN_MAGNITUDE;
}
sdb_status order_args(Corpus* c, const double* queries, uint32_t nq, int fn, int order, uint32_t k,
                      const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter, const uint64_t* out_rows,
                      const double* out_value, const uint32_t* out_count, Ranking* rank) {
  if (!c) return SDB_EINVAL;
  if (!vector_fn_known(fn)) {
    set_error("sdb_corpus_order: unknown vector function %d", fn);
    return SDB_EINVAL;
  }
  if (order != SDB_ORDER_ASC && order != SDB_ORDER_DESC) {
    set_error("sdb_corpus_order: unknown order %d", order);
    return SDB_EINVAL;
  }
  if (nq && ((!queries && fn != SDB_FN_MAGNITUDE) || !out_count || (k && (!out_rows || !out_value)))) {
    set_error("sdb_corpus_order: NULL queries (only SDB_FN_MAGNITUDE takes none) or outputs");
    return SDB_EINVAL;
  }
  if (k > 4096) {
    set_error("sdb_corpus_order: k = %u exceeds 4096", k);
    return SDB_EUNSUPPORTED;
  }
  if (filters) SDB_TRY(check_filters(nq, filters, n_filters, query_filter));
  *rank = Ranking{fn, order == SDB_ORDER_DESC};
  return SDB_OK;
}

}  // namespace sdb
extern "C" {

// Host-only diagnostic (no GPU needed): the corpus tiles (TILE_ROWS rows each) a screened search visits, in order.
// Every row that is not visited can never become a candidate and the exactness proof would not know, so "every tile
// exactly once" is a safety property of the schedules; tests/test_schedule_cover.py checks it exhaustively on the CPU.
sdb_status sdb_debug_schedule(uint64_t n_rows, uint32_t cand_cap, uint32_t k, uint32_t nq, int streaming,
                              uint32_t* out_tiles, uint64_t cap_tiles, uint64_t* out_n, uint32_t* out_probe_tiles,
                              uint32_t cap_probe, uint32_t* out_n_probe) {
  if (!out_n || !out_n_probe || cand_cap < TILE_ROWS) return SDB_EINVAL;
  uint64_t n = 0;
  uint32_t np = 0;
  auto emit = [&](uint32_t tile) {
    if (out_tiles && n < cap_tiles) out_tiles[n] = tile;
    n++;
  };
  if (streaming) {
    PassDesc p0, pm;
    build_stream_passes(n_rows, cand_cap, k, &p0, &pm);
    if (p0.count && !pm.count) {
      for (uint32_t i = 0; i < p0.count; i++) emit(pass_tile(p0, i));  // pass 0 scores everything
    } else {
      for (uint32_t i = 0; i < p0.count; i++) {
        if (out_probe_tiles && np < cap_probe) out_probe_tiles[np] = pass_tile(p0, i);
        np++;
      }
      for (uint32_t i = 0; i < pm.count; i++) emit(pass_tile(pm, i));
    }
  } else {
    for (const PassDesc& p : build_passes(n_rows, cand_cap, nq))
      for (uint32_t i = 0; i < p.count; i++) emit(pass_tile(p, i));
  }
  *out_n = n;
  *out_n_probe = np;
  return SDB_OK;
}

// Test-only diagnostics of the screens (declared in the header's diagnostics block): the corpus' screen copies and one
// screened batch, so that tests can hold every intermediate of the proof against a plain reference.
void sdb_debug_live_allocations(uint64_t* count, uint64_t* bytes) {
  if (count) *count = g_live_bufs.load();
  if (bytes) *bytes = g_live_bytes.load();
}

sdb_status sdb_debug_corpus_state(sdb_corpus* c, float* out_f, uint32_t* out_u, int8_t* out_i8, uint16_t* out_bf16,
                                  float* out_snorm, uint32_t* out_special) {
  if (!c) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  // MINKOWSKI of every order, not only Family::Lp: finalize prepares its state for every order (it may change later)
  const bool lp = c->metric == SDB_MANHATTAN || c->metric == SDB_CHEBYSHEV || c->metric == SDB_MINKOWSKI;
  if (!c->finalized || (c->dtype != SDB_F32 && !c->d_bf16 && !lp) ||
      (c->metric == SDB_PEARSON && family(c) != Family::Centred) ||
      (out_i8 && !c->d_i8) || (out_bf16 && !c->d_bf16)) {
    set_error("sdb_debug_corpus_state: needs a finalized F32 corpus or a screened F64 / PEARSON one (int8 copy: "
              "cosine and pearson only)");
    return SDB_EINVAL;
  }
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  SDB_CUDA(drain(c->ctx));
  const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
  if (out_f) {
    out_f[0] = c->i8_scale;
    out_f[1] = c->max_rel_qerr;
    out_f[2] = c->bf16_rel_err;
    out_f[3] = c->max_norm;
  }
  if (out_u) {
    out_u[0] = c->n_special;
    out_u[1] = c->n_outliers;
    out_u[2] = c->dim_pad;
    out_u[3] = c->dim_pad8;
    out_u[4] = (uint32_t)n_pad;
  }
  cudaStream_t st = c->ctx->copy_stream;
  if (out_i8 && n_pad) SDB_CUDA(cudaMemcpyAsync(out_i8, c->d_i8, n_pad * c->dim_pad8, cudaMemcpyDeviceToHost, st));
  if (out_bf16 && n_pad)
    SDB_CUDA(cudaMemcpyAsync(out_bf16, c->d_bf16, 2 * n_pad * c->dim_pad, cudaMemcpyDeviceToHost, st));
  if (out_snorm && n_pad) SDB_CUDA(cudaMemcpyAsync(out_snorm, c->d_snorm, 4 * n_pad, cudaMemcpyDeviceToHost, st));
  if (out_special && c->n_special)
    SDB_CUDA(cudaMemcpyAsync(out_special, c->d_special, 4 * c->n_special, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  return SDB_OK;
}

sdb_status sdb_debug_screen_batch(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k, sdb_screen screen,
                                  int streaming, uint32_t cand_cap, int score_all, float* out_qf, double* out_qmag,
                                  uint32_t* out_qu, int8_t* out_q8, uint16_t* out_qbf16, uint32_t* out_a,
                                  uint32_t* out_b, uint32_t* out_rr) {
  return sdb_debug_screen_batch_filtered(c, queries, nq, k, screen, streaming, cand_cap, score_all, out_qf, out_qmag,
                                         out_qu, out_q8, out_qbf16, out_a, out_b, out_rr, nullptr, 0, nullptr, -1);
}

// sdb_debug_screen_batch_filtered with the ranking `rank` (sdb_debug_screen_batch_ranked; the others rank KNN's)
static sdb_status debug_screen_batch(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k, sdb_screen screen,
                                     int streaming, uint32_t cand_cap, int score_all, float* out_qf, double* out_qmag,
                                     uint32_t* out_qu, int8_t* out_q8, uint16_t* out_qbf16, uint32_t* out_a,
                                     uint32_t* out_b, uint32_t* out_rr, const uint32_t* filters, uint32_t n_filters,
                                     const uint32_t* query_filter, int mask_hits, const Ranking& rank) {
  const bool tc = screen == SDB_SCREEN_TC_INT8 || screen == SDB_SCREEN_TC_BF16;
  if (!c || !queries || !nq || !k || k > 256 || cand_cap < 4096 || (!tc && screen != SDB_SCREEN_SIMT_F32) ||
      mask_hits < -1 || mask_hits > 1) {
    set_error("sdb_debug_screen_batch: bad argument (1 <= k <= 256, cand_cap >= 4096, a TC_INT8 / TC_BF16 / SIMT_F32 "
              "screen, mask_hits -1, 0 or 1)");
    return SDB_EINVAL;
  }
  if (filters) SDB_TRY(check_filters(nq, filters, n_filters, query_filter));
  std::lock_guard<std::mutex> g(c->mu);
  const Plan p = plan_batch(c, rank, k, nq, screen, streaming != 0);
  const View& v = p.v;
  const bool int8 = screen == SDB_SCREEN_TC_INT8;
  // Dot: any screen on f32 rows, the tensor cores on f64 ones; Centred: the tensor cores; Lp: SIMT_F32 (the Lp screen)
  const Family f = family(c);
  const bool served = f == Family::Dot       ? c->dtype == SDB_F32 || (tc && c->d_bf16)
                      : f == Family::Centred ? tc
                      : f == Family::Lp      ? screen == SDB_SCREEN_SIMT_F32
                                             : false;
  if (!c->finalized || !served || (int8 && !c->d_i8) || c->special_overflow || !c->n ||
      (v.cross && c->xspecial_overflow)) {
    set_error("sdb_debug_screen_batch: needs a finalized, non-empty F32 cosine / euclidean corpus, an F64 one with "
              "screen copies and a tensor-core screen (int8: cosine), a PEARSON one with screen copies and a "
              "tensor-core screen, or a MANHATTAN / CHEBYSHEV / MINKOWSKI (integer order 1 .. 8) one with SIMT_F32");
    return SDB_EINVAL;
  }
  Ctx* ctx = c->ctx;
  SDB_CUDA(cudaSetDevice(ctx->device));
  SDB_CUDA(drain(ctx));
  Ticket* t = claim_ticket(c);
  if (!t) return SDB_EOVERFLOW;
  SDB_TRY(ticket_prepare(c, *t, nq));
  const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
  const uint32_t cap = score_all ? (uint32_t)std::max<uint64_t>(cand_cap, n_pad) : cand_cap;
  // the batch runs on set 0 and the first stream; exactly `cap` slots per query: drop the set so that scratch_for
  // allocates it at this size
  Scratch& s = c->sets[0];
  s.sc_nq = s.sc_cap = 0;
  SDB_TRY(scratch_for(c, s, nq, cap));
  cudaStream_t st = ctx->stream;
  t->set = 0;
  t->stream = st;
  // the batch's filter, classified as ticket submission classifies it
  t->filt = FiltArg();
  t->n_direct = 0;
  t->permuted = false;
  t->plan = p;
  if (filters) {
    const uint32_t* bits = nullptr;
    std::vector<uint64_t> rows_per_filter;
    SDB_TRY(stage_filters(c, *t, RowFilters{filters, n_filters, query_filter, 0}, true, nq, &bits, &rows_per_filter));
    SDB_CUDA(cudaEventRecord(t->ev_h2d, ctx->copy_stream));
    SDB_CUDA(cudaStreamWaitEvent(st, t->ev_h2d, 0));
    std::vector<uint32_t> scr, dir;
    plan_filtered(c, *t, nq, bits, query_filter, rows_per_filter.data(), &scr, &dir);
    if (!score_all && !scr.empty() && !dir.empty()) {
      t->filt = FiltArg();
      t->n_direct = 0;
      set_error("sdb_debug_screen_batch_filtered: a batch that mixes direct and screened queries has no readable lists");
      return SDB_EUNSUPPORTED;
    }
    if (mask_hits >= 0) t->filt.mask_hits = (uint32_t)mask_hits;
    SDB_CUDA(t->d_qf.reserve(nq));
    SDB_CUDA(cudaMemcpyAsync(t->d_qf, t->h_qf.data(), sizeof(uint32_t) * nq, cudaMemcpyHostToDevice, st));
    t->filt.qf = t->d_qf;
  }
  const bool direct = !score_all && t->n_direct == nq;
  if (!score_all && !direct && p.key.first != screen) {  // the plan's rung 0 is another screen
    set_error("sdb_debug_screen_batch: the corpus does not offer screen %d", (int)screen);
    return SDB_EINVAL;
  }
  DevBuf<double> d_q;
  ResultBufs out;
  ScreenTap tap;
  auto run = [&]() -> sdb_status {
    SDB_CUDA(d_q.reserve((size_t)nq * c->dim));
    SDB_CUDA(out.reserve((size_t)nq * k, nq));
    SDB_CUDA(cudaMemcpyAsync(d_q, queries, sizeof(double) * (size_t)nq * c->dim, cudaMemcpyHostToDevice, st));
    if (score_all) {  // one pass-0 launch over every tile (SIMT: tau stays -inf), nothing selected
      const PassDesc all{1u, 0u, (uint32_t)(n_pad / TILE_ROWS), 0u};
      SDB_TRY(prep_queries(c, s, d_q, nq, st, v));
      SDB_TRY(cand_begin(c, s, nq, (int)screen, st, v, p.exact));
      SDB_TRY(tc                ? screen_tc_pass(c, s, t->filt, nq, k, all, int8, 0, st, v)
              : f == Family::Lp ? screen_lp_pass(c, s, t->filt, nq, all, st)
                                : screen_simt_pass(c, s, t->filt, nq, all, st, v));
      SDB_TRY(tap_list(s, nq, &tap.list_a, &tap.cnt_a, st));
      tap.gathered = tap.cnt_a;
      return SDB_OK;
    }
    // the production sequence of one batch at rung 0 of `screen` (no ladder, no exact fallback)
    t->k = k;
    t->row_base = 0;
    t->cancel = nullptr;
    const Run r{d_q, nq, out.rows, out.dist, out.count, t->filt, 0u, &tap, t->h_flags, t->h_qflags, t->h_stat};
    Enqueued e;
    SDB_TRY(enqueue_batch(c, *t, r, &e));
    SDB_CUDA(cudaStreamSynchronize(st));
    if (direct) return tap_list(s, nq, &tap.list_a, &tap.cnt_a, st);  // no screen ran: the lists are the direct ones
    return SDB_OK;
  };
  sdb_status rc = run();
  if (rc == SDB_OK) {  // per-query figures and lists (columns documented in the header)
    auto rd = [&](void* dst, const void* src, size_t bytes) {
      if (rc == SDB_OK && cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) {
        set_error("sdb_debug_screen_batch: copy-out failed");
        rc = SDB_ECUDA;
      }
    };
    const size_t cap_sz = (size_t)nq * cap;
    std::vector<float> f[9];
    const float* srcf[9] = {s.d_tau, s.d_margin, s.d_bscale, s.d_beps, s.d_tau2, s.d_beps2,
                            c->d_i8 ? s.d_q8scale.get() : nullptr, c->d_i8 ? s.d_q8err.get() : nullptr, s.d_qbferr};
    for (int j = 0; j < 9; j++) {
      f[j].assign(nq, NAN);
      if (srcf[j]) rd(f[j].data(), srcf[j], sizeof(float) * nq);
    }
    std::vector<uint32_t> flags(nq), qflags(nq), cnt_b(nq);
    std::vector<Cand> list_b(score_all ? 0 : cap_sz);
    std::vector<uint32_t> rr;
    rd(flags.data(), s.d_flags, sizeof(uint32_t) * nq);
    rd(qflags.data(), s.d_qflags, sizeof(uint32_t) * nq);
    if (out_qmag) rd(out_qmag, s.d_qmag, sizeof(double) * nq);
    if (out_q8 && c->d_i8) rd(out_q8, s.d_q8, (size_t)nq * c->dim_pad8);
    if (out_qbf16) rd(out_qbf16, s.d_qbf16, 2 * (size_t)nq * c->dim_pad);
    if (!score_all) {
      rd(cnt_b.data(), s.d_cand_cnt, sizeof(uint32_t) * nq);
      rd(list_b.data(), s.d_cand, sizeof(Cand) * cap_sz);
      if (out_rr) {
        rr.resize((size_t)nq * s.rr_stride);
        rd(rr.data(), s.d_rr_row, sizeof(uint32_t) * rr.size());
      }
    }
    if (rc == SDB_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = SDB_ECUDA;
    if (rc == SDB_OK) {
      // (filtered: the passing special rows are in the stage-B list)
      const uint32_t n_special = score_all || filters ? 0u : view_n_special(c, v);
      auto bits = [](float v) {
        uint32_t u;
        memcpy(&u, &v, 4);
        return u;
      };
      for (uint32_t q = 0; q < nq; q++) {
        if (out_qf)
          for (int j = 0; j < 9; j++) out_qf[(size_t)q * 9 + j] = f[j][q];
        const uint32_t n_a = std::min(tap.cnt_a[q], cap), n_b = score_all ? 0u : std::min(cnt_b[q], cap);
        if (out_qu) {
          uint32_t* u = out_qu + (size_t)q * 6;
          u[0] = flags[q];
          u[1] = qflags[q];
          u[2] = tap.gathered.empty() ? 0u : tap.gathered[q];
          u[3] = n_a;
          u[4] = n_b;
          u[5] = score_all ? 0u : n_b + n_special;
        }
        for (uint32_t e = 0; e < cap; e++) {
          const size_t i = (size_t)q * cap + e;
          if (out_a) {
            const bool have = e < n_a;
            out_a[3 * i] = have ? tap.list_a[i].row : 0xFFFFFFFFu;
            out_a[3 * i + 1] = have ? bits(tap.list_a[i].score) : 0x7fc00000u;
            out_a[3 * i + 2] = have && !tap.list_r.empty() ? bits(tap.list_r[i].score) : 0x7fc00000u;
          }
          if (out_b) {
            const bool have = e < n_b;
            out_b[2 * i] = have ? list_b[i].row : 0xFFFFFFFFu;
            out_b[2 * i + 1] = have ? bits(list_b[i].score) : 0x7fc00000u;
          }
        }
        if (out_rr && !score_all)
          for (uint32_t e = 0; e < cap + SPECIAL_CAP; e++)
            out_rr[(size_t)q * (cap + SPECIAL_CAP) + e] = e < n_b + n_special ? rr[(size_t)q * s.rr_stride + e] : 0xFFFFFFFFu;
      }
    }
  }
  return rc;
}

sdb_status sdb_debug_screen_batch_filtered(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k,
                                           sdb_screen screen, int streaming, uint32_t cand_cap, int score_all,
                                           float* out_qf, double* out_qmag, uint32_t* out_qu, int8_t* out_q8,
                                           uint16_t* out_qbf16, uint32_t* out_a, uint32_t* out_b, uint32_t* out_rr,
                                           const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                           int mask_hits) {
  return debug_screen_batch(c, queries, nq, k, screen, streaming, cand_cap, score_all, out_qf, out_qmag, out_qu, out_q8,
                            out_qbf16, out_a, out_b, out_rr, filters, n_filters, query_filter, mask_hits, Ranking());
}

sdb_status sdb_debug_screen_batch_ranked(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k,
                                         sdb_screen screen, int streaming, uint32_t cand_cap, int score_all,
                                         float* out_qf, double* out_qmag, uint32_t* out_qu, int8_t* out_q8,
                                         uint16_t* out_qbf16, uint32_t* out_a, uint32_t* out_b, uint32_t* out_rr,
                                         const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                         int mask_hits, int fn, int order) {
  if (c && !screened_ranking(c, Ranking{fn, order == SDB_ORDER_DESC})) {
    set_error("sdb_debug_screen_batch_ranked: (fn %d, order %d) is not a ranking the screens serve on this corpus", fn,
              order);
    return SDB_EINVAL;
  }
  if (order != SDB_ORDER_ASC && order != SDB_ORDER_DESC) {
    set_error("sdb_debug_screen_batch_ranked: unknown order %d", order);
    return SDB_EINVAL;
  }
  return debug_screen_batch(c, queries, nq, k, screen, streaming, cand_cap, score_all, out_qf, out_qmag, out_qu, out_q8,
                            out_qbf16, out_a, out_b, out_rr, filters, n_filters, query_filter, mask_hits,
                            Ranking{fn, order == SDB_ORDER_DESC});
}

sdb_status sdb_knn_submit(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k, uint64_t* out_rows,
                          double* out_dist, uint32_t* out_count, uint32_t* ticket) {
  if (!c || !ticket || !nq || !queries || !out_count || (k && (!out_rows || !out_dist))) return SDB_EINVAL;
  return knn_call(c, nq, k, host_call(c, queries, RowFilters(), out_rows, out_dist, out_count, nullptr), ticket);
}

sdb_status sdb_knn_submit_device(sdb_corpus* c, const double* d_queries, uint32_t nq, uint32_t k, uint64_t row_base,
                                 uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count, uint32_t* ticket) {
  if (!c || !ticket || (nq && (!d_queries || !d_out_count || (k && (!d_out_rows || !d_out_dist))))) return SDB_EINVAL;
  return knn_call(c, nq, k, device_call(d_queries, RowFilters(), row_base, d_out_rows, d_out_dist, d_out_count), ticket);
}

sdb_status sdb_knn_wait(sdb_corpus* c, uint32_t ticket) {
  if (!c) return SDB_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  Ticket* t = find_ticket(c, ticket);
  if (!t) {
    set_error("sdb_knn_wait: unknown or already completed ticket %u", ticket);
    return SDB_EINVAL;
  }
  return wait_locked(c, t);
}

sdb_status sdb_knn_bruteforce_device(sdb_corpus* c, const double* d_queries, uint32_t nq, uint32_t k,
                                     uint64_t row_base, uint64_t* d_out_rows, double* d_out_dist,
                                     uint32_t* d_out_count) {
  if (!c || (nq && (!d_queries || !d_out_count || (k && (!d_out_rows || !d_out_dist))))) return SDB_EINVAL;
  if (nq == 0) return SDB_OK;
  return knn_call(c, nq, k, device_call(d_queries, RowFilters(), row_base, d_out_rows, d_out_dist, d_out_count), nullptr);
}

sdb_status sdb_knn_bruteforce(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k, uint64_t* out_rows,
                              double* out_dist, uint32_t* out_count, const volatile int* cancel_flag) {
  if (!c || (nq && (!queries || !out_count || (k && (!out_rows || !out_dist))))) return SDB_EINVAL;
  if (nq == 0) return SDB_OK;
  if (cancel_flag && *cancel_flag) {
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  return knn_call(c, nq, k, host_call(c, queries, RowFilters(), out_rows, out_dist, out_count, cancel_flag), nullptr);
}

// ---- filtered brute-force KNN: per-query row bitmaps (see the header) ----------------------------------------------
sdb_status sdb_knn_bruteforce_filtered(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k,
                                       const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                       uint64_t* out_rows, double* out_dist, uint32_t* out_count,
                                       const volatile int* cancel_flag) {
  if (!c || (nq && (!queries || !out_count || (k && (!out_rows || !out_dist))))) return SDB_EINVAL;
  SDB_TRY(check_filters(nq, filters, n_filters, query_filter));
  if (nq == 0) return SDB_OK;
  if (cancel_flag && *cancel_flag) {
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  const RowFilters rf{filters, n_filters, query_filter, 0};
  return knn_call(c, nq, k, host_call(c, queries, rf, out_rows, out_dist, out_count, cancel_flag), nullptr);
}

// device bitmaps are read in place: counted on the copy stream (stage_filters), then the batch
sdb_status sdb_knn_bruteforce_filtered_device(sdb_corpus* c, const double* d_queries, uint32_t nq, uint32_t k,
                                              const uint32_t* d_filters, uint32_t n_filters,
                                              const uint32_t* query_filter, uint64_t row_base, uint64_t* d_out_rows,
                                              double* d_out_dist, uint32_t* d_out_count) {
  if (!c || (nq && (!d_queries || !d_out_count || (k && (!d_out_rows || !d_out_dist))))) return SDB_EINVAL;
  SDB_TRY(check_filters(nq, d_filters, n_filters, query_filter));
  if (nq == 0) return SDB_OK;
  const RowFilters rf{d_filters, n_filters, query_filter, 0};
  return knn_call(c, nq, k, device_call(d_queries, rf, row_base, d_out_rows, d_out_dist, d_out_count), nullptr);
}

sdb_status sdb_knn_submit_filtered_device(sdb_corpus* c, const double* d_queries, uint32_t nq, uint32_t k,
                                          const uint32_t* d_filters, uint32_t n_filters, const uint32_t* query_filter,
                                          uint64_t row_base, uint64_t* d_out_rows, double* d_out_dist,
                                          uint32_t* d_out_count, uint32_t* ticket) {
  if (!c || !ticket || (nq && (!d_queries || !d_out_count || (k && (!d_out_rows || !d_out_dist))))) return SDB_EINVAL;
  SDB_TRY(check_filters(nq, d_filters, n_filters, query_filter));
  const RowFilters rf{d_filters, n_filters, query_filter, 0};
  return knn_call(c, nq, k, device_call(d_queries, rf, row_base, d_out_rows, d_out_dist, d_out_count), ticket);
}

sdb_status sdb_knn_submit_filtered(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k,
                                   const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                   uint64_t* out_rows, double* out_dist, uint32_t* out_count, uint32_t* ticket) {
  if (!c || !ticket || !nq || !queries || !out_count || (k && (!out_rows || !out_dist))) return SDB_EINVAL;
  SDB_TRY(check_filters(nq, filters, n_filters, query_filter));
  const RowFilters rf{filters, n_filters, query_filter, 0};
  return knn_call(c, nq, k, host_call(c, queries, rf, out_rows, out_dist, out_count, nullptr), ticket);
}

// ---- ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k: the brute-force driver with another ranking -----------------
sdb_status sdb_corpus_order_topk(sdb_corpus* c, const double* queries, uint32_t nq, int fn, int order, uint32_t k,
                                 const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                 uint64_t* out_rows, double* out_value, uint32_t* out_count) {
  Ranking rank;
  SDB_TRY(order_args(c, queries, nq, fn, order, k, filters, n_filters, query_filter, out_rows, out_value, out_count,
                     &rank));
  if (nq == 0) return SDB_OK;
  KnnCall call = host_call(c, queries, RowFilters{filters, n_filters, query_filter, 0}, out_rows, out_value, out_count,
                           nullptr);
  call.rank = rank;
  return knn_call(c, nq, k, call, nullptr);
}

sdb_status sdb_corpus_order_topk_device(sdb_corpus* c, const double* d_queries, uint32_t nq, int fn, int order,
                                        uint32_t k, const uint32_t* d_filters, uint32_t n_filters,
                                        const uint32_t* query_filter, uint64_t row_base, uint64_t* d_out_rows,
                                        double* d_out_value, uint32_t* d_out_count) {
  Ranking rank;
  SDB_TRY(order_args(c, d_queries, nq, fn, order, k, d_filters, n_filters, query_filter, d_out_rows, d_out_value,
                     d_out_count, &rank));
  if (nq == 0) return SDB_OK;
  KnnCall call = device_call(d_queries, RowFilters{d_filters, n_filters, query_filter, 0}, row_base, d_out_rows,
                             d_out_value, d_out_count);
  call.rank = rank;
  return knn_call(c, nq, k, call, nullptr);
}

sdb_status sdb_corpus_order_submit(sdb_corpus* c, const double* queries, uint32_t nq, int fn, int order,
                                   uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                   const uint32_t* query_filter, uint64_t* out_rows, double* out_value,
                                   uint32_t* out_count, uint32_t* ticket) {
  Ranking rank;
  if (!ticket || !nq) return SDB_EINVAL;
  SDB_TRY(order_args(c, queries, nq, fn, order, k, filters, n_filters, query_filter, out_rows, out_value, out_count,
                     &rank));
  KnnCall call = host_call(c, queries, RowFilters{filters, n_filters, query_filter, 0}, out_rows, out_value, out_count,
                           nullptr);
  call.rank = rank;
  return knn_call(c, nq, k, call, ticket);
}

sdb_status sdb_corpus_order_submit_device(sdb_corpus* c, const double* d_queries, uint32_t nq, int fn,
                                          int order, uint32_t k, const uint32_t* d_filters, uint32_t n_filters,
                                          const uint32_t* query_filter, uint64_t row_base, uint64_t* d_out_rows,
                                          double* d_out_value, uint32_t* d_out_count, uint32_t* ticket) {
  Ranking rank;
  if (!ticket) return SDB_EINVAL;
  SDB_TRY(order_args(c, d_queries, nq, fn, order, k, d_filters, n_filters, query_filter, d_out_rows, d_out_value,
                     d_out_count, &rank));
  KnnCall call = device_call(d_queries, RowFilters{d_filters, n_filters, query_filter, 0}, row_base, d_out_rows,
                             d_out_value, d_out_count);
  call.rank = rank;
  return knn_call(c, nq, k, call, ticket);
}

sdb_status sdb_corpus_project(sdb_corpus* c, const double* query, int fn, double* out) {
  const bool is_metric = fn == SDB_COSINE || fn == SDB_EUCLIDEAN || fn == SDB_MANHATTAN || fn == SDB_CHEBYSHEV ||
                         fn == SDB_HAMMING || fn == SDB_PEARSON || fn == SDB_MINKOWSKI || fn == SDB_JACCARD;
  if (!c || !out || (!query && fn != SDB_FN_MAGNITUDE)) return SDB_EINVAL;
  if (!is_metric && fn != SDB_FN_SIMILARITY_COSINE && fn != SDB_FN_DOT && fn != SDB_FN_MAGNITUDE) {
    set_error("vector function %d not implemented on the GPU path", fn);
    return SDB_EUNSUPPORTED;
  }
  std::lock_guard<std::mutex> g(c->mu);
  if (!c->finalized) {
    set_error("corpus not finalized (call sdb_corpus_finalize after the last append)");
    return SDB_EINVAL;
  }
  if (c->n == 0) return SDB_OK;
  SDB_CUDA(cudaSetDevice(c->ctx->device));
  SDB_CUDA(drain(c->ctx));  // borrows scratch set 0 for the prepared query
  cudaStream_t st = c->ctx->stream;
  Scratch& s = c->sets[0];
  auto run = [&]() -> sdb_status {  // the temporaries are released on every path, before the synchronisation below
    AsyncBuf<double> d_q, d_vals;
    SDB_CUDA(d_q.reserve(c->dim, st));
    SDB_CUDA(d_vals.reserve(c->n, st));
    if (query) SDB_CUDA(cudaMemcpyAsync(d_q, query, sizeof(double) * c->dim, cudaMemcpyHostToDevice, st));
    else SDB_CUDA(cudaMemsetAsync(d_q, 0, sizeof(double) * c->dim, st));
    SDB_TRY(scratch_for(c, s, 1, 4096));
    SDB_TRY(prep_queries(c, s, d_q, 1, st, view_of(c, Ranking())));
    SDB_TRY(exact_project(c, fn, s.d_q64, s.d_qmag, s.d_qflags, d_vals, st));
    SDB_CUDA(cudaMemcpyAsync(out, d_vals, sizeof(double) * c->n, cudaMemcpyDeviceToHost, st));
    return SDB_OK;
  };
  const sdb_status rc = run();
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == SDB_OK) {
    set_error("sdb_corpus_project: %s", cudaGetErrorString(cudaGetLastError()));
    return SDB_ECUDA;
  }
  return rc;
}

sdb_status sdb_topk_merge_device(sdb_ctx* ctx, uint32_t n_lists, uint32_t nq, uint32_t k, const uint64_t* d_rows,
                                 const double* d_dist, const uint32_t* d_counts, uint64_t stride_rows,
                                 uint64_t stride_dist, uint64_t stride_counts, uint64_t* d_out_rows,
                                 double* d_out_dist, uint32_t* d_out_count) {
  if (!ctx || !n_lists || !k || !d_rows || !d_dist || !d_counts || !d_out_rows || !d_out_dist || !d_out_count)
    return SDB_EINVAL;
  if (nq == 0) return SDB_OK;
  std::lock_guard<std::mutex> g(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  SDB_TRY(topk_merge_launch(ctx, n_lists, nq, k, d_rows, d_dist, d_counts, stride_rows, stride_dist, stride_counts,
                            d_out_rows, d_out_dist, d_out_count, false, ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SDB_OK;
}

sdb_status sdb_order_merge_device(sdb_ctx* ctx, uint32_t n_lists, uint32_t nq, uint32_t k, int order,
                                  const uint64_t* d_rows, const double* d_value, const uint32_t* d_counts,
                                  uint64_t stride_rows, uint64_t stride_value, uint64_t stride_counts,
                                  uint64_t* d_out_rows, double* d_out_value, uint32_t* d_out_count) {
  if (!ctx || !n_lists || !k || !d_rows || !d_value || !d_counts || !d_out_rows || !d_out_value || !d_out_count)
    return SDB_EINVAL;
  if (order != SDB_ORDER_ASC && order != SDB_ORDER_DESC) {
    set_error("sdb_order_merge_device: unknown order %d", order);
    return SDB_EINVAL;
  }
  if (k > 4096) {
    set_error("sdb_order_merge_device: k = %u exceeds 4096", k);
    return SDB_EUNSUPPORTED;
  }
  if (nq == 0) return SDB_OK;
  std::lock_guard<std::mutex> g(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  SDB_TRY(topk_merge_launch(ctx, n_lists, nq, k, d_rows, d_value, d_counts, stride_rows, stride_value, stride_counts,
                            d_out_rows, d_out_value, d_out_count, order == SDB_ORDER_DESC, ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SDB_OK;
}

}  // extern "C"
