// internal.cuh -- shared declarations of the sdbgpu library (not part of the ABI).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/sdbgpu.h"

namespace sdb {

void set_error(const char* fmt, ...);

#define SDB_CUDA(call)                                                                      \
  do {                                                                                      \
    cudaError_t e__ = (call);                                                               \
    if (e__ != cudaSuccess) {                                                               \
      ::sdb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return SDB_ECUDA;                                                                     \
    }                                                                                       \
  } while (0)
#define SDB_TRY(call)                  \
  do {                                 \
    sdb_status s__ = (call);           \
    if (s__ != SDB_OK) return s__;     \
  } while (0)

// ---- owned buffers --------------------------------------------------------------------------------
// Every device and pinned buffer of the library is held by a Buf: move-only, freed by its destructor (on the device
// that is current then: the destroy entry points select the owner's device first).  reserve() only grows, and frees the
// old buffer before it allocates the larger one, so the peak is the new size alone; a failed reserve leaves it empty.
// A Buf converts to T*, so kernel launches and copies take it like the raw pointer.
enum class Mem { Device, Async, Pinned };  // cudaMalloc / cudaMallocAsync on a stream / cudaHostAlloc
inline std::atomic<uint64_t> g_live_bufs{0}, g_live_bytes{0};  // sdb_debug_live_allocations
template <class T, Mem K>
class Buf {
 public:
  Buf() = default;
  Buf(Buf&& o) noexcept : p_(o.p_), n_(o.n_), st_(o.st_) { o.p_ = nullptr, o.n_ = 0; }
  Buf& operator=(Buf&& o) noexcept {
    if (this != &o) reset(), p_ = o.p_, n_ = o.n_, st_ = o.st_, o.p_ = nullptr, o.n_ = 0;
    return *this;
  }
  ~Buf() { reset(); }
  T* get() const { return p_; }
  operator T*() const { return p_; }
  size_t size() const { return n_; }  // elements
  // st: the stream of a Mem::Async buffer (it is freed there too); flags: cudaHostAlloc flags of a Mem::Pinned one
  cudaError_t reserve(size_t n, cudaStream_t st = nullptr, unsigned flags = cudaHostAllocDefault) {
    if (n <= n_) return cudaSuccess;
    reset();
    void* p = nullptr;
    const cudaError_t e = K == Mem::Device ? cudaMalloc(&p, sizeof(T) * n)
                          : K == Mem::Async ? cudaMallocAsync(&p, sizeof(T) * n, st)
                                            : cudaHostAlloc(&p, sizeof(T) * n, flags);
    if (e != cudaSuccess) {
      cudaGetLastError();  // reported through the return value: the next launch check must not see it
      return e;
    }
    p_ = (T*)p, n_ = n, st_ = st;
    g_live_bufs++, g_live_bytes += sizeof(T) * n;
    return cudaSuccess;
  }
  void reset() {
    if (p_) free_released((void*)p_, st_);
    drop();
  }
  T* release() {  // hands the buffer to the caller, who frees it with free_released
    T* p = p_;
    drop();
    return p;
  }
  static void free_released(void* p, cudaStream_t st = nullptr) {
    if (K == Mem::Device) cudaFree(p);
    else if (K == Mem::Async) cudaFreeAsync(p, st);
    else cudaFreeHost(p);
  }

 private:
  void drop() {
    if (p_) g_live_bufs--, g_live_bytes -= sizeof(T) * n_;
    p_ = nullptr, n_ = 0;
  }
  T* p_ = nullptr;
  size_t n_ = 0;
  cudaStream_t st_ = nullptr;
};
template <class T> using DevBuf = Buf<T, Mem::Device>;
template <class T> using AsyncBuf = Buf<T, Mem::Async>;
template <class T> using PinnedBuf = Buf<T, Mem::Pinned>;

// rows / distances / counts of a batch's results (nq queries, n_out = nq x k entries), grow-only
struct ResultBufs {
  DevBuf<uint64_t> rows;
  DevBuf<double> dist;
  DevBuf<uint32_t> count;
  cudaError_t reserve(size_t n_out, size_t nq) {
    cudaError_t e = rows.reserve(n_out);
    if (e == cudaSuccess) e = dist.reserve(n_out);
    if (e == cudaSuccess) e = count.reserve(nq);
    return e;
  }
};

constexpr int TILE_ROWS = 256;    // screening tile = 256 corpus rows (one wgmma N=256 MMA tile)
constexpr int PASS_RATIO = 8;     // default geometric threshold-refinement ratio (api.cu:pass_ratio picks per batch size)
constexpr int SPECIAL_CAP = 1024; // rows with zero / non-finite norm handled by exact ranking

// ---- ordered keys -------------------------------------------------------------------------------
// Number::cmp on Floats (val/number.rs:620-633): -0.0 == 0.0, otherwise f64::total_cmp.
// All bit manipulation is done on integers obtained through an opaque move: nvcc otherwise rewrites
// `bits(d) | signbit` into fneg(fabs(d)), implements it with a DADD, and the DADD canonicalises NaNs --
// which silently destroyed the sign/payload of NaN distances.
__host__ __device__ inline uint64_t f64_bits(double d) {
  uint64_t b;
#ifdef __CUDA_ARCH__
  asm volatile("mov.b64 %0, %1;" : "=l"(b) : "d"(d));
#else
  memcpy(&b, &d, 8);
#endif
  return b;
}
__host__ __device__ inline uint64_t dist_key(double d) {
  uint64_t b = f64_bits(d);
  if ((b << 1) == 0) b = 0;  // canonicalise -0.0
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
// the key of a value in a ranking's direction: dist_key ascending, its complement descending (the whole total order
// reversed, NaNs included).  ~dist_key(d) is ~0 -- the key the exact kernel reserves for skipped rows and the sorters
// for padding -- only for the NaN whose bits are all set; that NaN takes the next key down and ties with 0xFFF...FE.
__host__ __device__ inline uint64_t order_key(double d, bool desc) {
  const uint64_t k = dist_key(d);
  return !desc ? k : (k ? ~k : ~1ull);
}
__host__ __device__ inline uint32_t f32_key(float f) {  // ascending key of a float (total order)
  uint32_t b;
#ifdef __CUDA_ARCH__
  asm volatile("mov.b32 %0, %1;" : "=r"(b) : "f"(f));
#else
  memcpy(&b, &f, 4);
#endif
  return (b >> 31) ? ~b : (b | 0x80000000u);
}

// ---- streaming threshold refinement (screen_tc.cu, candidates.cu) -------------------------------------------------
// Per query a 256-bin histogram of the scores appended so far, log-linear above the query's floor `lo`:
//   t = (score - lo) / w0 + 1 (>= 1),  bin = (bits(t) - bits(1.0f)) >> 19  -- 16 bins per octave of t, clamped to 255.
// bin() is monotone and edge(bin(s)) <= s up to float rounding (the refiner subtracts a guard), so
// "suffix count from the top reaches k at bin b" proves that the k-th best score seen so far is >= edge(b).
constexpr uint32_t HIST_BINS = 256;
constexpr uint32_t PROBE_TILES_MAX = 64;                   // tiles scored by the probe launch
constexpr uint32_t PROBE_STRIDE = PROBE_TILES_MAX * 8;     // chunk maxima per query (8 chunks of 32 rows per tile)
struct HistParam {
  float lo;      // floor: tau at the time the histogram was seeded
  float inv_w0;  // 1 / w0
  float w0;      // width scale (a quarter of the query's error margin, never 0)
  float margin;  // 2.1 x the screen's error bound in score units: tau = (k-th best score) - margin
};
__host__ __device__ inline uint32_t hist_bin(const HistParam& p, float score) {
  float t = (score - p.lo) * p.inv_w0 + 1.0f;
  t = t >= 1.0f ? t : 1.0f;  // also maps NaN to bin 0
  uint32_t b;
#ifdef __CUDA_ARCH__
  b = (__float_as_uint(t) - 0x3F800000u) >> 19;
#else
  uint32_t u;
  memcpy(&u, &t, 4);
  b = (u - 0x3F800000u) >> 19;
#endif
  return b < HIST_BINS - 1 ? b : HIST_BINS - 1;
}
__host__ __device__ inline double hist_edge(const HistParam& p, uint32_t b) {  // lower edge of bin b
  const uint32_t u = 0x3F800000u + (b << 19);
  float t;
#ifdef __CUDA_ARCH__
  t = __uint_as_float(u);
#else
  memcpy(&t, &u, 4);
#endif
  return (double)p.lo + (double)p.w0 * ((double)t - 1.0);
}

struct PassDesc {
  uint32_t stride;  // tiles t = i * stride
  uint32_t excl;    // 0: every i; else = the schedule ratio R: skip i % R == 0 (already done by an earlier pass)
  uint32_t count;   // number of tiles in this pass
  uint32_t perm;    // 0: visit in order; else an odd multiplier coprime with `count`: the j-th tile visited is
                    // (j * perm) % count, so that every stretch of the streaming pass samples the whole corpus
};
__host__ __device__ inline uint32_t pass_tile(const PassDesc& p, uint32_t w) {
  if (p.perm) w = (uint32_t)(((uint64_t)w * p.perm) % p.count);
  uint32_t i = p.excl ? (w / (p.excl - 1)) * p.excl + (w % (p.excl - 1)) + 1 : w;
  return i * p.stride;
}

// ---- per-query row filters (sdb_knn_*_filtered) --------------------------------------------------------------------
// bits: n_filters bitmaps of `words` uint32 words each (bit r = bit r % 32 of word r / 32); qf: the filter index of each
// query of the launch (offset like every other per-query array of a query-chunked launch).  bits == nullptr: no filter.
struct FiltArg {
  const uint32_t* bits = nullptr;
  const uint32_t* qf = nullptr;
  uint32_t words = 0;
  // int8 screens: also clear rejected rows from the consumers' hit masks (set when some query of the batch has a
  // selective filter, which keeps its threshold low; with dense filters the drain warp's test alone is cheaper)
  uint32_t mask_hits = 0;
};
// filtered batches: a query whose filter passes at most this many rows skips the screen (the direct regime): its
// passing rows are compacted into its candidate list and ranked by the exact re-rank (DESIGN.md section 5)
constexpr uint32_t DIRECT_MAX_ROWS = 4096;
// ... and a filter passing fewer than 1/MASK_HITS_DIV of the rows switches FiltArg::mask_hits on
constexpr uint64_t MASK_HITS_DIV = 20;
// does query q rank corpus row `row`?  Rows past the bitmap (the screen copies' padding) never pass.
__device__ __forceinline__ bool filt_pass(const FiltArg& f, uint32_t q, uint32_t row) {
  const uint32_t w = row >> 5;
  return w < f.words && ((__ldg(f.bits + (size_t)__ldg(f.qf + q) * f.words + w) >> (row & 31u)) & 1u) != 0;
}
// the row filters of one filtered call as the caller hands them over: n_filters bitmaps (host or device memory, where
// the call's queries are), query_filter on the host (NULL: every query uses filter 0).  n_rows_total: the global rows
// the bitmaps of a sharded call cover (ceil(n_rows_total / 32) words each, bit r = global row r); 0 for an unsharded
// call, whose bitmaps cover the corpus' own rows.  bits == nullptr: an unfiltered call.
struct RowFilters {
  const uint32_t* bits = nullptr;
  uint32_t n_filters = 0;
  const uint32_t* query_filter = nullptr;
  uint64_t n_rows_total = 0;
};

// What a batch ranks (sdb_corpus_order_*): the value of vector function fn per row (an sdb_metric id or an
// sdb_vector_fn), ascending or descending.  KNN batches rank the corpus metric ascending (fn = -1).
struct Ranking {
  int fn = -1;
  bool desc = false;
};

// What the Dot and Centred screens score per row:
//   Cosine     acc / |x|          (own: COSINE corpora and the centred operands of PEARSON ones; cross: EUCLIDEAN ones)
//   Euclid     2 acc - |x|^2      (own: EUCLIDEAN corpora; cross: COSINE ones)
//   Dot        acc                dot_ranking batches on either Dot metric
//   EuclidFar  2 acc + |x|^2      euclidean descending, acc against -q: |x|^2 - 2 x.q = d^2 - |q|^2
// acc = x~.q~, the dot of the screen copies.  (Lp / Count / Exact corpora: Euclid, which none of their stages reads.)
enum class Score { Cosine, Euclid, Dot, EuclidFar };
// A batch's view of a Dot or Centred corpus, decided once per batch (view_of) and handed to every stage that depends on
// it (prep_queries, cand_begin, the screens, cand_refine, cand_add_specials, the re-rank, cand_final).
struct View {
  Score sc = Score::Euclid;
  bool neg = false;    // the screen copies are those of -q (the re-rank keeps q)
  bool cross = false;  // per-row array and special list: the cross state (d_xnorm, d_xspecial), else d_snorm, d_special
  int steps = SDB_EUCLIDEAN;  // the re-rank's accumulation: SDB_COSINE (x.q), SDB_EUCLIDEAN ((x - q)^2), SDB_FN_DOT
  bool sim = false;    // ... and its finish: the cosine similarity instead of the cosine distance
  bool desc = false;   // the ranking's direction (Ranking::desc): the re-rank keys descending, cand_final proves that
};
// One rung of a batch's precision ladder (plan_batch, api.cu): a screen and the candidate-list capacity per query.
struct Rung {
  sdb_screen scr;
  uint32_t cap;
};
// What a remembered ladder rung belongs to (Corpus::remembered): the first-choice screen of the batch that settled on
// it, its k and the view_key of its view (dot batches' candidate sets are not KNN's)
struct RungKey {
  sdb_screen first = SDB_SCREEN_AUTO;
  uint32_t k = 0;
  int view = 0;
  bool operator==(const RungKey& o) const { return first == o.first && k == o.k && view == o.view; }
};
// How a brute-force batch runs, decided once at submit (plan_batch, api.cu) from the corpus, the ranking, k and the
// corpus' screen, schedule and proof mode as they stand then.  Every stage and the wait read the plan instead of those
// settings, so a batch in flight is finished the way it was submitted.
struct Plan {
  enum class Route { Empty, Exact, Counted, Screened };  // of the whole batch
  Route route = Route::Empty;
  Ranking rank;
  View v;
  Rung ladder[5] = {};          // Screened: the precision ladder, cheapest first
  uint32_t n_ladder = 0;
  uint32_t n_batch_rungs = 0;   // rungs a whole batch may climb
  RungKey key;                  // key.first: the whole batch's first-choice screen (NONE_EXACT: none)
  bool single_exact = false;    // a run of one query takes the exact kernel (AUTO on MANHATTAN, CHEBYSHEV, HAMMING)
  bool direct_ok = false;       // filtered queries may take the direct regime
  bool stream_refine = true;    // tensor-core schedule: one streaming launch (else the multi-pass schedule)
  bool exact = true;            // proof and exact fallbacks (false: approximate mode); stage B on tensor-core screens
  bool cancel_at_wait = false;  // dot and cross rankings report a cancel raised while the batch is in flight
  // a run of nq queries: the whole batch, a mixed batch's screened head or a repair sub-batch.  The single-query rule
  // applies to the run's own query count.
  bool counted(uint32_t nq) const { return route == Route::Counted && !(single_exact && nq == 1); }
  uint32_t rungs(uint32_t nq) const { return single_exact && nq == 1 ? 0u : n_ladder; }
};

struct Comm;  // comm.cu: NCCL communicator attached to a context (nullptr = single shard)

struct Ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;      // odd ticket slots: batch i+1 runs here, so its screen overlaps batch i's tail
  cudaStream_t copy_stream = nullptr;  // host<->device copies of the asynchronous entry points
  uint64_t launches = 0;
  std::mutex mu;
  void* encode_tiled = nullptr;  // cuTensorMapEncodeTiled (driver entry point), resolved lazily
  PinnedBuf<uint8_t> h_stage;    // pinned staging buffer for large device->host results (grow-only)
  Comm* comm = nullptr;
  // cancellation (sdb_ctx_cancel): one int in pinned memory that the host side polls between kernel phases, mirrored
  // into a word in DEVICE memory (copied on its own stream by sdb_ctx_cancel) that long-running kernels (the HNSW walk)
  // poll per query -- polling the pinned word itself from thousands of warps is a PCIe read each (ncu r2: 8 % of the
  // walk's stall samples)
  PinnedBuf<volatile int> h_cancel;
  DevBuf<int> d_cancel;
  cudaStream_t cancel_stream = nullptr;
  int prio_high = 0;  // greatest launch priority of the device (cudaDeviceGetStreamPriorityRange)
  int tc_pair_ctas = 0;  // CTAs of the int8 streaming screen launched as resident 2-CTA clusters (0: no pair launch)
  cudaEvent_t trace_epoch = nullptr;  // SDB_TRACE
  double trace_host0 = 0.0;           // host clock (s) at the epoch
};
inline bool ctx_cancelled(const Ctx* ctx) { return ctx->h_cancel && *ctx->h_cancel != 0; }

// per-device kernel attributes (dynamic shared-memory limits).  cudaFuncSetAttribute is per DEVICE, so these run in
// sdb_ctx_create after cudaSetDevice -- never behind a process-wide flag (a second context on another GPU of the same
// process would otherwise launch with the 48 KB default and fail).
sdb_status screen_tc_init_device(Ctx* ctx);
sdb_status candidates_init_device();
sdb_status exact_init_device();
void comm_destroy(Ctx* ctx);  // comm.cu
void comm_corpus_released(struct Corpus* c);  // comm.cu: drops the corpus's sharded-search state (slot buffers, arena)
int comm_size(const Ctx* ctx);
int comm_rank(const Ctx* ctx);
sdb_status comm_allreduce_sum(Ctx* ctx, void* d_buf, size_t count, int elem_bytes, cudaStream_t st);

struct Cand {  // one screened candidate
  float score; // larger = closer
  uint32_t row;
};

// one asynchronous batch (sdb_knn_submit* ... sdb_knn_wait): everything wait() needs to finish it on the host side
struct Ticket {
  bool busy = false;
  uint32_t id = 0;
  const double* d_queries = nullptr;  // caller's device queries (must stay valid until wait)
  uint32_t nq = 0, k = 0;
  uint64_t row_base = 0;
  uint64_t *d_out_rows = nullptr, *h_out_rows = nullptr;  // device result (caller's or the slot's) / optional host copy
  double *d_out_dist = nullptr, *h_out_dist = nullptr;
  uint32_t *d_out_count = nullptr, *h_out_count = nullptr;
  const volatile int* cancel = nullptr;
  cudaStream_t stream = nullptr;  // every kernel / copy of this batch (slot parity picks the context's stream)
  int set = 0;                    // scratch set of this batch
  Plan plan;
  int screen = 0;       // sdb_screen this batch ran
  uint32_t rung = 0, n_repaired = 0;  // rung: of plan.ladder, where the whole batch stands
  uint32_t n_passes = 0;
  uint64_t launches0 = 0;
  cudaEvent_t ev_begin = nullptr, ev_screen0 = nullptr, ev_screen1 = nullptr, ev_end = nullptr;
  PinnedBuf<uint32_t> h_flags;   // per query, bit0 overflow, bit1 proof failed
  uint32_t* h_qflags = nullptr;  // pinned: per query, bit0 needs the exact path, bit1 NaN input
  uint32_t* h_stat = nullptr;    // pinned: [0] queries flagged, [1] candidates re-ranked, [2] max per query, [3] survivors gathered
  uint32_t h_cap = 0;
  // host-buffer entry points: per-slot device staging
  DevBuf<double> d_in_q;
  ResultBufs res;
  cudaEvent_t ev_h2d = nullptr, ev_out = nullptr;
  cudaEvent_t ev_main = nullptr;  // recorded after this batch's last screen launch (the next batch's screen waits for it)
  bool wait_h2d = false;  // the batch's stream still has to wait for ev_h2d (inputs travelling on the copy stream)
  // filtered batches: filt.bits = the caller's device bitmaps or d_in_filt (host bitmaps staged per slot), filt.qf =
  // d_qf (per query filter index, also kept on the host in h_qf); unfiltered batches: filt.bits == nullptr
  FiltArg filt;
  std::vector<uint32_t> h_qf;
  DevBuf<uint32_t> d_qf, d_in_filt;
  // stage_filters: a sharded call's span of its host bitmaps (before the slice), and the set bits of device bitmaps
  DevBuf<uint32_t> d_in_span;
  DevBuf<unsigned long long> d_fcnt;
  PinnedBuf<unsigned long long> h_fcnt;
  // a permuted batch: the screened sub-batch's counters (d_stat), which the direct sub-batch's cand_begin resets
  DevBuf<uint32_t> d_stat_scr;
  // direct regime: the last n_direct queries of the batch skip the screen.  A batch that mixes both kinds runs
  // permuted (screened queries first): d_queries / d_out_* / h_qf are then the permuted copies (d_pq, pres) and the
  // results are scattered through d_perm (permuted position -> caller's query) to d_fin_*, the caller's outputs
  uint32_t n_direct = 0;
  bool permuted = false;
  DevBuf<double> d_pq;
  DevBuf<uint32_t> d_perm;
  ResultBufs pres;
  uint64_t* d_fin_rows = nullptr;
  double* d_fin_dist = nullptr;
  uint32_t* d_fin_count = nullptr;
  // SDB_TRACE=1: named timestamps of this batch on its stream, printed at wait time relative to the context's epoch
  std::vector<std::pair<const char*, cudaEvent_t>> trace;
};
constexpr int N_TICKETS = 4;
bool trace_enabled();
void trace_mark(Ctx* ctx, Ticket& t, const char* name, cudaStream_t st);  // api.cu
void trace_dump(Ctx* ctx, Ticket& t);
void trace_host(Ctx* ctx, uint32_t ticket, const char* name);  // host-side timestamp on the same time base

// Per-batch search scratch.  Each corpus holds two sets (Corpus::sets): a ticket's slot parity names its set (and its
// stream), so consecutive batches alternate between them and the screen of batch i+1 can run while the tail of batch i
// (candidate selection, f32 re-score, exact re-rank, final ordering, all-gather + merge) is still in flight.  Every
// stage of a batch takes its set explicitly; what the corpus holds beside the sets is shared by every batch.
struct Scratch {
  uint32_t sc_nq = 0, sc_cap = 0;
  DevBuf<double> d_q64;
  DevBuf<float> d_q32;
  DevBuf<__nv_bfloat16> d_qbf16;
  DevBuf<double> d_qmag;
  DevBuf<double2> d_qmom;     // PEARSON: {m2, S2} per query (mean and sum of squared deviations, the exact kernel's)
  DevBuf<uint32_t> d_qflags;  // bit0: query needs the exact path; bit1: query has NaN input
  DevBuf<float> d_qbferr;     // |q - bf16(q)| / |q| per query
  DevBuf<int8_t> d_q8;        // int8 queries nq_pad x dim_pad8
  DevBuf<float> d_q8scale;    // max|q|/127 per query
  DevBuf<float> d_q8err;      // |q - dequant(q)| / |q| per query
  DevBuf<uint32_t> d_qkey;    // count path, u32 keys for f32 rows, u64 for f64 rows: HAMMING: the queries' equality
                              // keys; JACCARD: each query's distinct keys, sorted (count_prep_queries)
  DevBuf<uint32_t> d_qjac;    // JACCARD count path: per query {u_q, n_look}, then scratch flags [nq][dim]
  DevBuf<uint32_t> d_mscale;  // MINKOWSKI screen: [0] the batch's largest |q^_i| (f32 bits), [1] its scale exponent e
  DevBuf<Cand> d_sub;         // thread-private candidate sub-lists of the tensor-core screens
  DevBuf<uint32_t> d_sub_cnt; // [nq][sub_slots]
  uint32_t sub_slots = 0, sub_cap = 0, last_slots = 0;
  DevBuf<float> d_bscale;     // per query: factor that turns tau into similarity*|q| units (1 or q8scale * i8_scale)
  DevBuf<float> d_beps;       // per query: rigorous screen error bound (cosine units / relative dot error)
  DevBuf<float> d_margin;     // per query: 2.1 x that bound in score units (0 in approximate mode)
  DevBuf<float> d_margin2;    // stage B (f32 re-score of the candidates): margin, error bound, threshold
  DevBuf<float> d_beps2;
  DevBuf<float> d_tau2;
  DevBuf<float> d_qlow;       // per query: lower / upper bound of any score (histogram geometry)
  DevBuf<float> d_qcap;
  DevBuf<HistParam> d_hparam; // per query histogram geometry of the streaming screen
  DevBuf<uint32_t> d_hist;    // [nq][HIST_BINS]
  DevBuf<float> d_probe;      // [nq][PROBE_STRIDE] chunk maxima of the probe launch
  DevBuf<float> d_tau;
  DevBuf<Cand> d_cand;
  DevBuf<uint32_t> d_cand_cnt;
  DevBuf<uint32_t> d_flags;   // per query: bit0 overflow, bit1 verification failed
  DevBuf<uint32_t> d_stat;    // [0] queries flagged by cand_final, [1] candidates re-ranked, [2] max per query, [3] gathered
  DevBuf<uint64_t> d_rr_key;  // re-rank results: nq x rr_stride
  DevBuf<double> d_rr_dist;
  DevBuf<uint32_t> d_rr_row;
  uint32_t rr_stride = 0;
};

// Test-only snapshot of one batch's stage-A candidate lists (sdb_debug_screen_batch).  The enqueue functions fill it
// when the batch they run carries one, which is never the case in production.
struct ScreenTap {
  std::vector<uint32_t> gathered;  // per query: most entries any stage-A selection gathered, before capping
  std::vector<Cand> list_a;        // [nq][cap]: kept list after the last stage-A selection
  std::vector<uint32_t> cnt_a;
  std::vector<Cand> list_r;        // [nq][cap]: the same list after cand_refine re-scored it in f32 (empty if it did not run)
};

struct Corpus {
  Ctx* ctx = nullptr;
  uint32_t dim = 0, dim_pad = 0;  // dim_pad: bf16 screen copy row length (multiple of 64)
  sdb_dtype dtype = SDB_F32;
  sdb_metric metric = SDB_COSINE;
  sdb_screen screen = SDB_SCREEN_AUTO;
  bool exact = true;   // false: skip the proof / exact fallback (approximate mode)
  bool stream_refine = true;  // tensor-core screens: one streaming launch with in-kernel threshold refinement
  double minkowski_p = 3.0;   // order of SDB_MINKOWSKI
  struct {
    RungKey key;
    uint32_t rung = 0;
  } remembered;  // the ladder rung the last screened batch settled on, and what it belongs to (api.cu)
  uint64_t cap = 0, n = 0;
  uint64_t row_base = 0;            // global id of row 0 (row-sharded corpora)
  bool finalized = false;
  DevBuf<char> d_rows;              // master copy, cap x dim (f32 or f64)
  DevBuf<double> d_mag;          // exact f64 magnitude per row (reference arithmetic)
  DevBuf<float> d_snorm;         // cosine: 1/|x| ; euclid: |x|^2 ; pearson: 1/|x - m1| ; NaN = never a screen candidate
  DevBuf<double2> d_mom;         // PEARSON corpora with screen copies: {m1, S1} per row (finalize_pearson_kernel)
  DevBuf<uint32_t> d_jfirst;     // JACCARD corpora (when it fits): first-occurrence bitmask [cap][ceil(dim / 32)]
  DevBuf<uint32_t> d_jux;        // ... and the number of distinct values per row
  DevBuf<__nv_bfloat16> d_bf16;  // screen copy cap_pad x dim_pad (rows padded to TILE_ROWS)
  float bf16_rel_err = 0.00390625f; // max over rows of |x - bf16(x)| / |x| (measured at finalize, rounded up)
  DevBuf<int8_t> d_i8;           // int8 screen copy cap_pad x dim_pad8 of the normalised rows (one global scale), cosine only
  uint32_t dim_pad8 = 0;            // multiple of 128
  float max_rel_qerr = 0.f;         // max over rows of |x/|x| - s * x8|
  float i8_scale = 1.f;             // global scale s of the int8 copy
  DevBuf<uint8_t> d_skip;        // optional skip mask
  DevBuf<uint8_t> d_removed;     // tombstones (sdb_corpus_remove); OR-ed with the skip mask at finalize
  uint64_t n_removed = 0;
  DevBuf<uint32_t> d_special;    // rows ranked exactly on every query
  uint32_t n_special = 0;
  uint32_t n_outliers = 0;          // of those: rows made special because one component dominates (int8 scale)
  bool special_overflow = false;
  // cross state of a COSINE / EUCLIDEAN corpus with a bf16 copy (finalize_cross_kernel), read by the views that rank the
  // other metric (View::cross): the other metric's screening norm -- |x|^2 on COSINE corpora, 1/|x| on EUCLIDEAN ones,
  // NaN wherever d_snorm is NaN -- and the union of the own special rows with those the other metric's rule adds
  DevBuf<float> d_xnorm;
  DevBuf<uint32_t> d_xspecial;
  uint32_t n_xspecial = 0;
  bool xspecial_overflow = false;  // more than SPECIAL_CAP: the cross views take the exact kernel (KNN does not)
  float max_norm = 0.f;
  // exact path scratch
  DevBuf<uint64_t> d_ex_key;  // N keys
  DevBuf<double> d_ex_val;    // N distances (the key maps -0.0 to 0.0; the result returns the value itself)
  DevBuf<uint32_t> d_sel;     // radix-select state
  DevBuf<double> d_fb_q;      // fallback query scratch (one query: f64 copy, |q|, flags)
  DevBuf<double> d_rp_q;      // repair sub-batch: the failed queries of a batch, gathered, and their results
  DevBuf<uint32_t> d_rp_qf;   // ... and their filter indices (filtered batches)
  ResultBufs rp;
  DevBuf<double> d_fb_qmag;
  DevBuf<uint32_t> d_fb_qflags;
  Scratch sets[2];  // per-batch scratch (see Scratch); Ticket::set names a batch's
  cudaEvent_t last_main = nullptr;  // ev_main of the batch whose screen was enqueued last
  // asynchronous batches
  Ticket tickets[N_TICKETS];
  uint32_t next_ticket = 1;
  sdb_knn_stats stats{};
  std::mutex mu;
};

// The order of a MINKOWSKI corpus that the f32 screen serves (screen_lp.cu): an integer 1 .. 8, whose |t|^p is a short
// chain of f32 multiplications.  0 for every other metric and order (non-integers, p < 1, p > 8, +-inf): those stay on
// the exact kernel, which calls pow() per element.
inline int minkowski_screen_order(const Corpus* c) {
  if (c->metric != SDB_MINKOWSKI) return 0;
  const double p = c->minkowski_p;
  return (p >= 1.0 && p <= 8.0 && p == (double)(int)p) ? (int)p : 0;
}
// The scoring family of a corpus: the per-query bound, candidate re-rank and proof that serve its brute-force searches,
// on which every stage of a batch switches.  Evaluated per batch, never stored: sdb_corpus_set_minkowski_order may move
// a finalized MINKOWSKI corpus between Lp and Exact.  Dot: COSINE, EUCLIDEAN.  Centred: PEARSON with its moments
// (d_mom).  Lp: MANHATTAN, CHEBYSHEV, MINKOWSKI of a screened order.  Count: HAMMING, JACCARD with its first-occurrence
// state (d_jfirst); count_ranked batches take the count path (exact counts of every row per row range, count.cu,
// then cand_final with tau = -inf), the others the exact kernel.  Exact: the exact kernel alone.
enum class Family { Dot, Centred, Lp, Count, Exact };
inline Family family(const Corpus* c) {
  switch (c->metric) {
    case SDB_COSINE: case SDB_EUCLIDEAN: return Family::Dot;
    case SDB_PEARSON: return c->d_mom ? Family::Centred : Family::Exact;
    case SDB_MANHATTAN: case SDB_CHEBYSHEV: return Family::Lp;
    case SDB_MINKOWSKI: return minkowski_screen_order(c) > 0 ? Family::Lp : Family::Exact;
    case SDB_HAMMING: return Family::Count;
    default: return c->d_jfirst ? Family::Count : Family::Exact;  // SDB_JACCARD
  }
}
constexpr uint32_t COUNT_CAP_MAX = 16384;  // candidate entries per query of the count path: n_ranges k at most
inline bool count_ranked(const Corpus* c, uint32_t k, sdb_screen screen) {
  return family(c) == Family::Count && k >= 1 && k <= 256 && screen != SDB_SCREEN_NONE_EXACT;
}
// The ranking of KNN itself, the corpus metric ascending: KnnTopK's DistanceEntry order and SortTopK's are both
// Number::cmp and then scan position, so it takes the KNN path unchanged.
inline bool knn_ranking(const Corpus* c, const Ranking& r) { return !r.desc && (r.fn < 0 || r.fn == (int)c->metric); }
// vector::similarity::cosine descending on a COSINE corpus: the distance 1 - s is computed from the same s and does not
// increase as s grows, so the Dot screens' candidate sets hold its top k; the re-rank keys s descending and cand_final
// proves the result with the similarity's upper bound (DESIGN.md section 5, ORDER BY).
inline bool cosine_desc(const Corpus* c, const Ranking& r) {
  return r.desc && r.fn == SDB_FN_SIMILARITY_COSINE && c->metric == SDB_COSINE;
}
// The corpus metric descending where that needs no new screen:
//  - HAMMING / JACCARD on the count path: it computes every row's value exactly, so the direction is a key transform
//    of its per-range top-k and of the merge after it (count.cu), with nothing to prove;
//  - PEARSON with its moments (Centred): the screens score cos(dx, +dq) instead of cos(dx, -dq), largest for the
//    largest pearson, and cand_final mirrors the proof (DESIGN.md section 5, ORDER BY).
inline bool metric_desc(const Corpus* c, const Ranking& r) {
  const Family f = family(c);
  return r.desc && r.fn == (int)c->metric && (f == Family::Count || f == Family::Centred);
}
// vector::dot in either direction on a Dot corpus (COSINE or EUCLIDEAN with its bf16 copy): maximum (DESC) or minimum
// (ASC) inner product.  The screens score x.q (DESC) or x.(-q) (ASC) with no norm term, the re-rank computes the
// reference's dot and cand_final proves the order with the dot's bound (DESIGN.md sections 2 and 5, ORDER BY).
inline bool dot_ranking(const Corpus* c, const Ranking& r) { return r.fn == SDB_FN_DOT && family(c) == Family::Dot; }
// The other cosine and euclidean rankings of a Dot corpus with its cross state (d_xnorm): vector::distance::cosine or
// vector::similarity::cosine in the order KNN / cosine_desc do not take (farthest first, least similar first), on either
// metric, and vector::distance::euclidean in either order on COSINE corpora and descending (farthest first) on
// EUCLIDEAN ones.  The screens score the cosine or the euclidean form of the ranked function towards q or -q, with the
// per-row array of that form (view_of), and cand_final proves the order with that form's bound (DESIGN.md sections 2
// and 5, ORDER BY).
inline bool cross_ranking(const Corpus* c, const Ranking& r) {
  const bool cos_fn = r.fn == SDB_COSINE || r.fn == SDB_FN_SIMILARITY_COSINE;
  if (family(c) != Family::Dot || !c->d_xnorm || (!cos_fn && r.fn != SDB_EUCLIDEAN)) return false;
  return !knn_ranking(c, r) && !cosine_desc(c, r);
}
// the rankings the screens (and the count path) serve; every other one is ranked by the exact kernel alone.  Those
// that are descending are cosine_desc, metric_desc, dot_ranking and cross_ranking, and every stage takes
// Ranking::desc as it is.
inline bool screened_ranking(const Corpus* c, const Ranking& r) {
  return knn_ranking(c, r) || cosine_desc(c, r) || metric_desc(c, r) || dot_ranking(c, r) || cross_ranking(c, r);
}
inline View view_of(const Corpus* c, const Ranking& r) {
  View v;
  v.desc = r.desc;
  if (dot_ranking(c, r)) {
    v.sc = Score::Dot, v.neg = !r.desc, v.steps = SDB_FN_DOT;
  } else if (cross_ranking(c, r) && r.fn != SDB_EUCLIDEAN) {
    // cosine distance ascending and similarity descending look towards q; the other two orders towards -q
    v.sc = Score::Cosine, v.neg = (r.fn == SDB_COSINE) == r.desc, v.cross = c->metric != SDB_COSINE;
    v.steps = SDB_COSINE, v.sim = r.fn == SDB_FN_SIMILARITY_COSINE;
  } else if (cross_ranking(c, r)) {
    v.sc = r.desc ? Score::EuclidFar : Score::Euclid, v.neg = r.desc, v.cross = c->metric != SDB_EUCLIDEAN;
  } else if (c->metric == SDB_COSINE || family(c) == Family::Centred) {
    v.sc = Score::Cosine, v.steps = SDB_COSINE, v.sim = cosine_desc(c, r);
  }
  return v;
}
// the remembered ladder rung belongs to what the screens select: score, query sign and per-row array
inline int view_key(const View& v) { return (int)v.sc | (v.neg ? 8 : 0) | (v.cross ? 16 : 0); }
inline const float* view_snorm(const Corpus* c, const View& v) { return v.cross ? c->d_xnorm.get() : c->d_snorm.get(); }
inline const uint32_t* view_special(const Corpus* c, const View& v) {
  return v.cross ? c->d_xspecial.get() : c->d_special.get();
}
inline uint32_t view_n_special(const Corpus* c, const View& v) { return v.cross ? c->n_xspecial : c->n_special; }

// ---- the brute-force driver (api.cu), as its entry points and the sharded search (comm.cu) use it ------------------
// one batch as a caller hands it over: queries and row filters on the host (host_in) or the device; outputs on the host
// (host_out: the batch writes the slot's res buffers and copy_out copies them) or the device
struct KnnCall {
  const double* queries = nullptr;
  bool host_in = false;
  RowFilters rf;  // rf.bits == nullptr: unfiltered; rf.n_rows_total != 0: a shard's part of global bitmaps
  uint64_t row_base = 0;
  uint64_t* out_rows = nullptr;
  double* out_dist = nullptr;
  uint32_t* out_count = nullptr;
  bool host_out = false;
  const volatile int* cancel = nullptr;
  Ranking rank;  // sdb_corpus_order_*: queries == nullptr for SDB_FN_MAGNITUDE, which takes no query
};
// a free ticket slot, or nullptr with the "too many batches in flight" error (the caller returns SDB_EOVERFLOW)
Ticket* claim_ticket(Corpus* c);
// stages the call's host inputs on the copy stream and enqueues the batch on the claimed ticket t; the caller holds c->mu
sdb_status submit_call(Corpus* c, Ticket* t, uint32_t nq, uint32_t k, const KnnCall& call);
sdb_status check_filters(uint32_t nq, const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter);
// the checks every sdb_corpus_order_* call shares (fn, order, NULL queries or outputs, k <= 4096, the filters); *rank is
// the batch's ranking
sdb_status order_args(Corpus* c, const double* queries, uint32_t nq, int fn, int order, uint32_t k,
                      const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter, const uint64_t* out_rows,
                      const double* out_value, const uint32_t* out_count, Ranking* rank);
// by ticket id, for a sharded batch: completion (ladder re-runs, exact fallbacks, statistics), release, the 16-byte
// block header enqueued into d_hdr, the batch's stream and a trace mark on it
sdb_status knn_finish_for_shard(Corpus* c, uint32_t ticket, bool* repaired);
sdb_status knn_release_ticket(Corpus* c, uint32_t ticket);
sdb_status knn_shard_header(Corpus* c, uint32_t ticket, void* d_hdr);
cudaStream_t knn_ticket_stream(Corpus* c, uint32_t ticket);
void knn_trace_mark(Corpus* c, uint32_t ticket, const char* name);
sdb_status topk_merge_launch(Ctx* ctx, uint32_t n_lists, uint32_t nq, uint32_t k, const uint64_t* d_rows,
                             const double* d_dist, const uint32_t* d_counts, uint64_t stride_rows, uint64_t stride_dist,
                             uint64_t stride_counts, uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                             bool desc, cudaStream_t st);

// tiling shared by the f32 Lp screen (screen_lp.cu) and the count path (count.cu)
constexpr int LP_THREADS = 256;
constexpr int LP_RB = 128;          // rows per CTA step (a pass tile is two steps)
constexpr int LP_KC = 32;           // columns per shared-memory chunk
constexpr int LP_STRIDE = LP_KC + 4;
constexpr int LP_TQ = 4;            // queries per thread

// ---- launch wrappers (defined in the .cu files) ---------------------------------------------------
// corpus.cu
sdb_status corpus_finalize_device(Corpus* c);
sdb_status corpus_remove_device(Corpus* c, const uint64_t* h_ids, uint64_t n);
sdb_status corpus_reapply_tombstones(Corpus* c, cudaStream_t st);
// The stages of a batch take its scratch set s and, where rows are screened or ranked, its row filter filt.
// screen_simt.cu: the SIMT_F32 screen of Dot corpora (f32 rows), scoring the view v
sdb_status screen_simt_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                            cudaStream_t st, const View& v);
// screen_lp.cu: the SIMT_F32 screen of Lp corpora, f32 L1 / L-infinity / Lp (score = -s~), f32 and f64 rows
sdb_status screen_lp_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                          cudaStream_t st);
// count.cu: the count path of Count corpora: rows split into count_ranges() ranges, each query's candidate entries
// (cnt, rr_*) = the union of its ranges' k best (distance, row) pairs with their exact distances; needs prep_queries
// (which runs count_prep_queries for Count corpora) and cand_begin
uint32_t count_ranges(const Corpus* c, uint32_t nq, uint32_t k);
sdb_status count_prep_queries(const Corpus* c, Scratch& s, uint32_t nq, cudaStream_t st);
// desc: the k largest (value, -row) per range instead of the k smallest (metric_desc batches)
sdb_status count_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k, cudaStream_t st,
                      bool desc = false);
// screen_tc.cu
// mode 0: pass 0 (every score of the pass's tiles written to fixed slots), 1: threshold pass, 2: streaming pass with
// in-kernel threshold refinement (histogram + refiner warp), 3: probe (chunk maxima of a few tiles, no candidates)
// v: the batch's view (the int8 screen serves Score::Cosine on the own screening norm only)
sdb_status screen_tc_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k, const PassDesc& p,
                          bool int8, int mode, cudaStream_t st, const View& v);
bool screen_tc_available();
// candidates.cu
// grows s to nq queries x cap candidates (a set that grows loses its contents)
sdb_status scratch_for(const Corpus* c, Scratch& s, uint32_t nq, uint32_t cap);
// v: the batch's view.  Centred: View::desc takes the screen copies of +dq / |dq| (a metric_desc batch) instead of
// -dq / |dq|; Dot corpora: View::neg takes the screen copies of -q (the re-rank keeps q)
sdb_status prep_queries(const Corpus* c, Scratch& s, const double* d_queries, uint32_t nq, cudaStream_t st,
                        const View& v);
// one query prepared into the fallback scratch (d_fb_*), independent of the batch scratch
sdb_status prep_fallback_query(Corpus* c, const double* d_query, cudaStream_t st);
// resets tau / counts / flags and derives, per query, the screen's error bound, the selection margin and the score range
// (exact: the batch's proof mode, Plan::exact; approximate mode selects with no margin)
sdb_status cand_begin(const Corpus* c, Scratch& s, uint32_t nq, int screen, cudaStream_t st, const View& v, bool exact);
sdb_status cand_set_count(const Corpus* c, Scratch& s, uint32_t nq, uint32_t value, cudaStream_t st);
// per query: gather the main list + the private sub-lists, find the k-th best score s_k, keep every candidate with
// score >= tau = s_k - margin (all of them while fewer than k exist), publish tau.  (The streaming pass's histogram is
// seeded by cand_seed_from_probe.)
sdb_status cand_select(const Corpus* c, Scratch& s, uint32_t nq, uint32_t k, bool drop_invalid, uint32_t n_slots,
                       cudaStream_t st, int stage = 0);
// stage B: re-score every kept candidate in f32 (master rows x f32 query) so that cand_select(stage 1) can shrink the
// set before the FP64-bound exact re-rank
sdb_status cand_refine(const Corpus* c, Scratch& s, uint32_t nq, cudaStream_t st, const View& v);
// after a probe launch over n_tiles tiles: tau = (k-th largest chunk maximum) - margin, histogram geometry, empty lists
sdb_status cand_seed_from_probe(const Corpus* c, Scratch& s, uint32_t nq, uint32_t k, uint32_t n_tiles,
                                cudaStream_t st);
// filtered batches: after a pass-0 launch, give the entries of rows a query's filter rejects a NaN score, which
// cand_select drops like any invalid row
sdb_status cand_filter_list(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st);
// filtered batches: append each query's passing special rows to its list (the re-rank and cand_final then run without
// the shared special-row tail); a list that has no room is flagged as overflowed
sdb_status cand_add_specials(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st,
                             const View& v);
// direct regime (filtered): each query's list = the rows its filter passes that are neither skipped nor removed
sdb_status cand_direct(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st);
// View::desc (the descending screened rankings): the re-rank keys its values descending, and cand_final proves that
// order.  v (Dot corpora): the re-rank computes the view's function (View::steps, View::sim) over its special list, and
// cand_final proves the order with the bound of the view's score
sdb_status cand_rerank(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st,
                       bool small_sets, const View& v);
sdb_status cand_final(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k, uint64_t row_base,
                      uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count, cudaStream_t st,
                      const View& v);
// exact.cu: query vector / |q| / flags are passed explicitly (a batch scratch row or the fallback scratch).
// filter: nullptr, or the query's bitmap (filter_words words): rows whose bit is clear are not ranked.
// rank: the value ranked (any vector function) and its direction; the default is the corpus metric ascending (KNN).
sdb_status exact_query(Corpus* c, const double* d_q64, const double* d_qmag, const uint32_t* d_qflags, uint32_t k,
                       uint64_t row_base, uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                       cudaStream_t st, const uint32_t* filter = nullptr, uint32_t filter_words = 0,
                       const Ranking& rank = Ranking());
sdb_status exact_project(const Corpus* c, int fn, const double* d_q64, const double* d_qmag, const uint32_t* d_qflags,
                         double* d_vals, cudaStream_t st);
// gen.cu
sdb_status gen_fill_f32(Ctx* ctx, float* d_out, uint64_t seed, uint64_t first, uint64_t n, cudaStream_t st);

// hnsw.cu: range / monotonicity check of a device CSR handed over the ABI (SDB_EINVAL with a message on violation)
sdb_status csr_check(Ctx* ctx, const uint64_t* d_rp, const uint32_t* d_ci, uint64_t n_rows, uint64_t n_edges,
                     uint64_t id_limit, unsigned long long counts[2], const char* what, cudaStream_t st);
sdb_status csr_validate(Ctx* ctx, const uint64_t* d_rp, const uint32_t* d_ci, uint64_t n_rows, uint64_t n_edges,
                        uint64_t id_limit, const char* what, cudaStream_t st);
// graph.cu: out[0..n) = exclusive scan of in[0..n); *d_total = sum (in/out may alias)
sdb_status exclusive_scan(Ctx* ctx, const uint64_t* d_in, uint64_t* d_out, uint64_t n, uint64_t* d_total, cudaStream_t st);
// stage.cu: He / Hn value decoders (host blobs in, device arrays out)
sdb_status stage_decode_vectors(Ctx* ctx, const uint8_t* blob, const uint64_t* off, const uint64_t* ids, uint64_t n,
                                uint32_t dim, sdb_dtype out_dtype, uint64_t n_rows, void* d_out, uint8_t* d_present,
                                uint64_t* n_bad, cudaStream_t st, int native = -1);  // native: see stage_vectors_kernel
sdb_status stage_decode_nodes(Ctx* ctx, const uint8_t* blob, const uint64_t* off, const uint64_t* node_ids, uint64_t n,
                              uint64_t n_elems, DevBuf<uint64_t>* d_row_ptr_out, DevBuf<uint32_t>* d_col_idx_out,
                              uint64_t* n_edges, uint64_t* n_bad, cudaStream_t st);

inline void count_launch(Ctx* ctx, uint64_t n = 1) { ctx->launches += n; }

}  // namespace sdb

struct sdb_ctx : sdb::Ctx {};
struct sdb_corpus : sdb::Corpus {};
