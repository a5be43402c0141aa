// screen_lp.cu -- f32 screen of MANHATTAN / CHEBYSHEV / MINKOWSKI (integer order 1 .. 8) corpora, shaped like an SGEMM
// on the FP32 pipe.
//
// score(q, x) = -s~,  s~ = sum_i |x^_i - q^_i|  (MANHATTAN, f32, any summation order)
//                     s~ = max_i |x^_i - q^_i|  (CHEBYSHEV)
//                     s~ = fl32((sum_i |s x^_i - s q^_i|^p)^(1/p) / s)  (MINKOWSKI of order p, s = 2^-e per batch; the
//                          power sum in f32, the root in f64 for the pairs that pass the power-space prefilter only;
//                          2 - 5 FP32 instructions per element, minkowski_fma)
// q^ = the query rounded to f32 (prep_queries), x^ = the row: f32 rows as stored, f64 rows rounded to f32 once per
// staged element.  Every (query, row, element) costs two FP32 instructions: FADD, then FADD or FMNMX with an |.|
// operand modifier.  A larger score is better, as in the other screens; rows with score >= tau[q] are appended to the
// query's candidate list exactly as screen_simt_kernel does.  cand_begin_lp_kernel / cand_begin_minkowski_kernel
// (candidates.cu) hold the error bound of s~ against the reference's f64 distance that makes the proof in cand_final rigorous.
//
// A CTA owns QB (8, 32 or 64) queries x 128 rows, 256 threads, a TQ(4) x TR register block per thread.  The K dimension is staged
// in chunks of 32 columns through shared memory (row-major, stride 36 floats: conflict-free LDS.128 for the register
// blocks, conflict-free STS for the staging), the next chunk travelling in registers while the current one is scored.
// The global loads are plain coalesced 128-byte row segments: at QB = 64 a chunk costs each thread 16 + 8 loads
// against 2048 FP32 instructions, so the kernel is bound by FP32 issue, not by the loads, and any row length works.
// Accumulators persist across chunks; the threshold test runs after the last one.
// Work item = (256-row pass tile, query block), grid-stride over pass.count x ceil(nq / QB): any nq works, and the
// query blocks of one tile run next to each other, so a tile is read from HBM about once per pass.
#include <algorithm>
#include <type_traits>

#include "exactmath.cuh"
#include "internal.cuh"

namespace sdb {

constexpr int LP_THREADS = 256;
constexpr int LP_RB = 128;          // rows per CTA step (a pass tile is two steps)
constexpr int LP_KC = 32;           // columns per shared-memory chunk
constexpr int LP_STRIDE = LP_KC + 4;
constexpr int LP_TQ = 4;            // queries per thread

// MINKOWSKI of integer order P: |t|^p of one element, a fixed chain of P - 1 or fewer f32 multiplications (every
// factor |t| <= 1 under the launch's scale) ending in one FFMA into the accumulator.  Relative to |t|^p the chain's
// roundings compound to at most (1 + u)^(p - 1) (p = 8: t2 = t t, t4 = t2 t2, t4 t4 carries t2's rounding four times and
// t4's twice), and a factor that underflows costs at most p 2^-150 absolute (cand_begin_minkowski_kernel's bound).
template <int P>
__device__ __forceinline__ float minkowski_fma(float t, float acc) {
  if (P == 1) return acc + fabsf(t);
  if (P == 2) return fmaf(t, t, acc);
  const float a = fabsf(t), t2 = t * t;
  if (P == 3) return fmaf(t2, a, acc);
  if (P == 4) return fmaf(t2, t2, acc);
  if (P == 5) return fmaf(t2 * t2, a, acc);
  if (P == 6) {
    const float t3 = t2 * a;
    return fmaf(t3, t3, acc);
  }
  if (P == 7) return fmaf(t2 * t2, t2 * a, acc);
  const float t4 = t2 * t2;
  return fmaf(t4, t4, acc);
}

// MINKOWSKI score of a power sum S~ = sum_i |t_i|^p that passed the power-space prefilter: the norm in f64, scaled back
// by 2^e (exact) and rounded to nearest f32 once.  Out of line: it runs for the few pairs near the threshold only.
template <int P>
__device__ __noinline__ float minkowski_score(float s, int e) {
  const double r = P == 1 ? (double)s : pow((double)s, 1.0 / P);
  return -__double2float_rn(ldexp(r, e));
}

// The prefilter's power-space threshold for tau: S~ > tp  =>  minkowski_score(S~) < tau, so that no row the norm-space
// test keeps is dropped.  (-tau (1 + 2^-20) + 2^-148) s, to the p-th power in f64 (p roundings of 2^-53 at most, and
// f64 pow() within 2^-44 of the root, DESIGN.md section 2), rounded up.  tau > 0 or NaN: nothing can pass.
template <int P>
__device__ __forceinline__ float minkowski_threshold(float tau, float s) {
  const double a = -(double)tau;
  if (!(a >= 0.0)) return -1.f;
  const double b = (a * (1.0 + 0x1p-20) + 0x1p-148) * (double)s;
  double r = b;
#pragma unroll
  for (int i = 1; i < P; i++) r *= b;
  return __double2float_ru(r * (1.0 + 0x1p-40));
}

// P = 0: MANHATTAN / CHEBYSHEV (METRIC).  P = 1 .. 8: MINKOWSKI of that order, on rows and queries scaled by
// s = 2^-e (mscale[1] = e, cand_begin_minkowski_kernel) while staging, so that every |t| <= 1: no power sum overflows.
// The score is the f32 norm -fl32(S~^(1/p) 2^e); the threshold test runs in power space first (minkowski_threshold).
template <int METRIC, typename T, bool FILT, int QB, int P>
__device__ __forceinline__ void screen_lp_body(const T* __restrict__ rows, const float* __restrict__ snorm,
                                               uint32_t dim, uint64_t n_rows, const float* __restrict__ q32,
                                               uint32_t nq, PassDesc pass, const float* __restrict__ tau,
                                               Cand* __restrict__ cand, uint32_t* __restrict__ cand_cnt, uint32_t cap,
                                               FiltArg filt, const uint32_t* __restrict__ mscale) {
  constexpr int NTQ = QB / LP_TQ;              // threads along the queries
  constexpr int NTR = LP_THREADS / NTQ;        // threads along the rows
  constexpr int TR = LP_RB / NTR;              // rows per thread: r = tr + NTR * i
  constexpr int XL = LP_RB * LP_KC / LP_THREADS;  // staged row elements per thread and chunk (16)
  constexpr int QL = QB * LP_KC / LP_THREADS;     // staged query elements per thread and chunk
  static_assert(NTQ * LP_TQ == QB && NTR * TR == LP_RB && QL >= 1, "tile shape");
  __shared__ __align__(16) float s_x[LP_RB * LP_STRIDE];
  __shared__ __align__(16) float s_q[QB * LP_STRIDE];
  const uint32_t tid = threadIdx.x, tr = tid % NTR, tq = tid / NTR;
  const uint32_t n_qb = (nq + QB - 1) / QB;
  const uint32_t n_chunks = (dim + LP_KC - 1) / LP_KC;
  const uint64_t items = (uint64_t)pass.count * n_qb;
  int m_e = 0;
  float m_s = 1.f;
  if constexpr (P > 0) {
    m_e = (int)__ldg(mscale + 1);
    m_s = ldexpf(1.f, -m_e);  // 2^-129 .. 2^126: exact (a subnormal f32 below 2^-126)
  }
  for (uint64_t w = blockIdx.x; w < items; w += gridDim.x) {
    const uint32_t qb0 = (uint32_t)(w % n_qb) * QB;
    const uint64_t tile_row0 = (uint64_t)pass_tile(pass, (uint32_t)(w / n_qb)) * TILE_ROWS;
    for (uint32_t half = 0; half < TILE_ROWS / LP_RB; half++) {
      const uint64_t row0 = tile_row0 + (uint64_t)half * LP_RB;
      if (row0 >= n_rows) break;
      float acc[TR][LP_TQ];
#pragma unroll
      for (int i = 0; i < TR; i++)
#pragma unroll
        for (int j = 0; j < LP_TQ; j++) acc[i][j] = 0.f;
      // element e = tid + 256 l of a chunk: row (or query) e / 32, column e % 32 -> one 32-column row segment per warp
      T xr[XL];
      float qr[QL];
      auto load = [&](uint32_t c0) {
#pragma unroll
        for (int l = 0; l < XL; l++) {
          const uint32_t e = tid + LP_THREADS * l, c = c0 + (e & 31u);
          const uint64_t r = row0 + (e >> 5);
          xr[l] = (r < n_rows && c < dim) ? __ldg(rows + r * dim + c) : T(0);
        }
#pragma unroll
        for (int l = 0; l < QL; l++) {
          const uint32_t e = tid + LP_THREADS * l, c = c0 + (e & 31u), q = qb0 + (e >> 5);
          qr[l] = (q < nq && c < dim) ? __ldg(q32 + (size_t)q * dim + c) : 0.f;
        }
      };
      load(0);
      for (uint32_t ch = 0; ch < n_chunks; ch++) {
        __syncthreads();  // the previous chunk has been scored
#pragma unroll
        for (int l = 0; l < XL; l++) {
          const uint32_t e = tid + LP_THREADS * l;
          if constexpr (P > 0) s_x[(e >> 5) * LP_STRIDE + (e & 31u)] = (float)xr[l] * m_s;
          else s_x[(e >> 5) * LP_STRIDE + (e & 31u)] = (float)xr[l];  // f64 rows: rounded to nearest f32 here, once
        }
#pragma unroll
        for (int l = 0; l < QL; l++) {
          const uint32_t e = tid + LP_THREADS * l;
          if constexpr (P > 0) s_q[(e >> 5) * LP_STRIDE + (e & 31u)] = qr[l] * m_s;
          else s_q[(e >> 5) * LP_STRIDE + (e & 31u)] = qr[l];
        }
        __syncthreads();
        if (ch + 1 < n_chunks) load((ch + 1) * LP_KC);
#pragma unroll 2
        for (int kk = 0; kk < LP_KC; kk += 4) {
          float4 qv[LP_TQ];
#pragma unroll
          for (int j = 0; j < LP_TQ; j++) qv[j] = *reinterpret_cast<const float4*>(s_q + (tq * LP_TQ + j) * LP_STRIDE + kk);
#pragma unroll
          for (int i = 0; i < TR; i++) {
            const float4 xv = *reinterpret_cast<const float4*>(s_x + (tr + NTR * i) * LP_STRIDE + kk);
#pragma unroll
            for (int j = 0; j < LP_TQ; j++) {
              if constexpr (P > 0) {
                acc[i][j] = minkowski_fma<P>(xv.x - qv[j].x, acc[i][j]);
                acc[i][j] = minkowski_fma<P>(xv.y - qv[j].y, acc[i][j]);
                acc[i][j] = minkowski_fma<P>(xv.z - qv[j].z, acc[i][j]);
                acc[i][j] = minkowski_fma<P>(xv.w - qv[j].w, acc[i][j]);
              } else if (METRIC == SDB_MANHATTAN) {
                acc[i][j] += fabsf(xv.x - qv[j].x);
                acc[i][j] += fabsf(xv.y - qv[j].y);
                acc[i][j] += fabsf(xv.z - qv[j].z);
                acc[i][j] += fabsf(xv.w - qv[j].w);
              } else {
                acc[i][j] = fmaxf(acc[i][j], fabsf(xv.x - qv[j].x));
                acc[i][j] = fmaxf(acc[i][j], fabsf(xv.y - qv[j].y));
                acc[i][j] = fmaxf(acc[i][j], fabsf(xv.z - qv[j].z));
                acc[i][j] = fmaxf(acc[i][j], fabsf(xv.w - qv[j].w));
              }
            }
          }
        }
      }
      // threshold test: score = -(s~ + snorm); snorm is 0 for screened rows and NaN for skipped / special / removed /
      // padding rows, whose NaN score never passes
      float my_tau[LP_TQ];
#pragma unroll
      for (int j = 0; j < LP_TQ; j++) {
        const uint32_t q = qb0 + tq * LP_TQ + j;
        my_tau[j] = q < nq ? __ldg(tau + q) : __int_as_float(0x7fc00000);
      }
      float my_tp[LP_TQ];  // MINKOWSKI: the power-space prefilter of my_tau
      if constexpr (P > 0) {
#pragma unroll
        for (int j = 0; j < LP_TQ; j++) my_tp[j] = minkowski_threshold<P>(my_tau[j], m_s);
      }
#pragma unroll
      for (int i = 0; i < TR; i++) {
        const uint64_t row = row0 + tr + NTR * i;
        if (row >= n_rows) continue;
        const float sn = __ldg(snorm + row);
#pragma unroll
        for (int j = 0; j < LP_TQ; j++) {
          const uint32_t q = qb0 + tq * LP_TQ + j;
          if constexpr (P > 0) {
            const float s = acc[i][j] + sn;  // NaN for rows that are never candidates
            if (s <= my_tp[j]) {
              const float sc = minkowski_score<P>(s, m_e);
              if (sc >= my_tau[j] && (!FILT || filt_pass(filt, q, (uint32_t)row))) {
                const uint32_t pos = atomicAdd(cand_cnt + q, 1u);
                if (pos < cap) {
                  Cand cd;
                  cd.score = sc;
                  cd.row = (uint32_t)row;
                  cand[(size_t)q * cap + pos] = cd;
                }
              }
            }
          } else {
            const float sc = -(acc[i][j] + sn);
            if (sc >= my_tau[j] && (!FILT || filt_pass(filt, q, (uint32_t)row))) {
              const uint32_t pos = atomicAdd(cand_cnt + q, 1u);
              if (pos < cap) {
                Cand cd;
                cd.score = sc;
                cd.row = (uint32_t)row;
                cand[(size_t)q * cap + pos] = cd;
              }
            }
          }
        }
      }
    }
  }
}

template <int METRIC, typename T, bool FILT, int QB>
__global__ void __launch_bounds__(LP_THREADS, QB >= 32 || sizeof(T) == 8 ? 1 : 2) screen_lp_kernel(
    const T* __restrict__ rows, const float* __restrict__ snorm, uint32_t dim, uint64_t n_rows,
    const float* __restrict__ q32, uint32_t nq, PassDesc pass, const float* __restrict__ tau, Cand* __restrict__ cand,
    uint32_t* __restrict__ cand_cnt, uint32_t cap, FiltArg filt) {
  screen_lp_body<METRIC, T, FILT, QB, 0>(rows, snorm, dim, n_rows, q32, nq, pass, tau, cand, cand_cnt, cap, filt,
                                         nullptr);
}
template <int P, typename T, bool FILT, int QB>
__global__ void __launch_bounds__(LP_THREADS, QB >= 32 || sizeof(T) == 8 ? 1 : 2) screen_minkowski_kernel(
    const T* __restrict__ rows, const float* __restrict__ snorm, uint32_t dim, uint64_t n_rows,
    const float* __restrict__ q32, uint32_t nq, PassDesc pass, const float* __restrict__ tau, Cand* __restrict__ cand,
    uint32_t* __restrict__ cand_cnt, uint32_t cap, FiltArg filt, const uint32_t* __restrict__ mscale) {
  screen_lp_body<SDB_MINKOWSKI, T, FILT, QB, P>(rows, snorm, dim, n_rows, q32, nq, pass, tau, cand, cand_cnt, cap,
                                                filt, mscale);
}

template <int METRIC, int P, typename T, bool FILT, int QB>
static sdb_status launch_lp(Corpus* c, uint32_t nq, const PassDesc& p, cudaStream_t st) {
  // P = 0: MANHATTAN / CHEBYSHEV; P = 1 .. 8: MINKOWSKI of that order
  auto kern = [] {
    if constexpr (P == 0) return screen_lp_kernel<METRIC, T, FILT, QB>;
    else return screen_minkowski_kernel<P, T, FILT, QB>;
  }();
  // resident CTAs per SM: a property of the instantiation (static shared memory, registers) on sm_90a, asked once
  static const int per_sm = [kern]() {
    int v = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, kern, LP_THREADS, 0) != cudaSuccess) {
      cudaGetLastError();
      v = 1;
    }
    return v < 1 ? 1 : v;
  }();
  const uint64_t items = (uint64_t)p.count * ((nq + QB - 1) / QB);
  uint64_t grid = (uint64_t)c->ctx->sm_count * per_sm;
  if (grid > items) grid = items;
  if constexpr (P == 0)
    kern<<<(unsigned)grid, LP_THREADS, 0, st>>>((const T*)c->d_rows.get(), c->d_snorm, c->dim, c->n, c->d_q32, nq, p,
                                                c->d_tau, c->d_cand, c->d_cand_cnt, c->sc_cap, c->filt);
  else
    kern<<<(unsigned)grid, LP_THREADS, 0, st>>>((const T*)c->d_rows.get(), c->d_snorm, c->dim, c->n, c->d_q32, nq, p,
                                                c->d_tau, c->d_cand, c->d_cand_cnt, c->sc_cap, c->filt, c->d_mscale);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// the query block follows the batch: small batches are HBM-bound, and a block larger than the batch spends FP32 work
// on padding queries (an 8-query block at most 7 / 8 of it, a 32-query block for 17-32 queries at most 15 / 32)
template <int METRIC, int P, typename T, bool FILT>
static sdb_status launch_lp_qb(Corpus* c, uint32_t nq, const PassDesc& p, cudaStream_t st) {
  if (nq <= 16) return launch_lp<METRIC, P, T, FILT, 8>(c, nq, p, st);
  if (nq <= 32) return launch_lp<METRIC, P, T, FILT, 32>(c, nq, p, st);
  return launch_lp<METRIC, P, T, FILT, 64>(c, nq, p, st);
}
template <int METRIC, int P, typename T>
static sdb_status launch_lp_filt(Corpus* c, uint32_t nq, const PassDesc& p, cudaStream_t st) {
  return c->filt.bits ? launch_lp_qb<METRIC, P, T, true>(c, nq, p, st) : launch_lp_qb<METRIC, P, T, false>(c, nq, p, st);
}
template <int METRIC, int P = 0>
static sdb_status launch_lp_type(Corpus* c, uint32_t nq, const PassDesc& p, cudaStream_t st) {
  return c->dtype == SDB_F32 ? launch_lp_filt<METRIC, P, float>(c, nq, p, st)
                             : launch_lp_filt<METRIC, P, double>(c, nq, p, st);
}

sdb_status screen_lp_pass(Corpus* c, uint32_t nq, const PassDesc& p, cudaStream_t st) {
  if (p.count == 0 || nq == 0) return SDB_OK;
  switch (minkowski_screen_order(c)) {
    case 1: return launch_lp_type<SDB_MINKOWSKI, 1>(c, nq, p, st);
    case 2: return launch_lp_type<SDB_MINKOWSKI, 2>(c, nq, p, st);
    case 3: return launch_lp_type<SDB_MINKOWSKI, 3>(c, nq, p, st);
    case 4: return launch_lp_type<SDB_MINKOWSKI, 4>(c, nq, p, st);
    case 5: return launch_lp_type<SDB_MINKOWSKI, 5>(c, nq, p, st);
    case 6: return launch_lp_type<SDB_MINKOWSKI, 6>(c, nq, p, st);
    case 7: return launch_lp_type<SDB_MINKOWSKI, 7>(c, nq, p, st);
    case 8: return launch_lp_type<SDB_MINKOWSKI, 8>(c, nq, p, st);
    default: break;
  }
  return c->metric == SDB_MANHATTAN ? launch_lp_type<SDB_MANHATTAN>(c, nq, p, st)
                                    : launch_lp_type<SDB_CHEBYSHEV>(c, nq, p, st);
}

// ---- HAMMING: exact mismatch counts, ranked per row range (DESIGN.md section 2, "HAMMING count path") ---------------
// The tiling above with equality keys instead of floats (eq_key_f32 / eq_key_f64, exactmath.cuh): a (query, row,
// element) costs one integer compare and one add, and the count is the reference's distance exactly.  Selection: the
// rows are cut into n_ranges contiguous ranges of LP_RB-row steps; a work item is (range, query block), and per query
// it keeps the k smallest (count, row) pairs of its range in shared memory.  The union of the ranges' lists holds the
// global top k by (count, row) however many counts tie, so the query's list is that union (n_ranges k <= the list
// capacity), its entries already carry their exact distances (rr_*), and cand_final orders it with tau = -inf.
// A warp owns whole queries (NTR <= 32 threads along the rows: all 128 rows of a step for its TQ queries per group),
// so a list is only ever touched by one warp and needs no block-wide synchronisation.
template <typename K>
__device__ __forceinline__ void count_ld4(const K* p, K (&v)[4]) {
  if constexpr (sizeof(K) == 4) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    v[0] = u.x, v[1] = u.y, v[2] = u.z, v[3] = u.w;
  } else {
    const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(p), b = *reinterpret_cast<const ulonglong2*>(p + 2);
    v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
  }
}
template <typename T>
using CountKey = EqKey<T>;

// List entries: HAMMING packs (count << 32 | row) into one integer; JACCARD's distance is a ratio, so its entries are
// (dist_key(d), row) pairs.  Both order as (distance, row), which is unique per list.
struct JEntry {
  unsigned long long key;
  uint32_t row;
};
__device__ __forceinline__ bool operator<(const JEntry& a, const JEntry& b) {
  return a.key < b.key || (a.key == b.key && a.row < b.row);
}
__device__ __forceinline__ bool operator==(const JEntry& a, const JEntry& b) { return a.key == b.key && a.row == b.row; }
__device__ __forceinline__ uint64_t entry_shfl(uint64_t v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ uint64_t entry_shfl_xor(uint64_t v, int o) { return __shfl_xor_sync(0xffffffffu, v, o); }
__device__ __forceinline__ JEntry entry_shfl(const JEntry& v, int src) {
  return JEntry{__shfl_sync(0xffffffffu, v.key, src), __shfl_sync(0xffffffffu, v.row, src)};
}
__device__ __forceinline__ JEntry entry_shfl_xor(const JEntry& v, int o) {
  return JEntry{__shfl_xor_sync(0xffffffffu, v.key, o), __shfl_xor_sync(0xffffffffu, v.row, o)};
}

// one entry into the list of local query ql; every lane of the warp calls it with the same entry
template <typename E>
__device__ __forceinline__ void count_list_insert(E* __restrict__ L, E* s_max, uint32_t* s_pos, uint32_t* s_fill,
                                                  uint32_t ql, uint32_t k, E e, uint32_t lane) {
  const uint32_t fill = s_fill[ql];
  const bool full = fill >= k;
  const bool take = !full || e < s_max[ql];
  const uint32_t at = full ? s_pos[ql] : fill;
  __syncwarp();  // every lane has read the list's state before lane 0 changes it
  if (!take) return;
  if (lane == 0) {
    L[at] = e;
    if (!full) s_fill[ql] = fill + 1;
  }
  __syncwarp();
  if (!full && fill + 1 < k) return;  // the largest entry matters once the list is full
  E best{};
  uint32_t pos = 0;
  bool has = false;
  for (uint32_t p = lane; p < k; p += 32) {
    const E v = L[p];
    if (!has || best < v) best = v, pos = p, has = true;
  }
  E m = has ? best : E{};
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const E y = entry_shfl_xor(m, o);
    m = m < y ? y : m;
  }
  const uint32_t holder = __ffs(__ballot_sync(0xffffffffu, has && best == m)) - 1;
  pos = __shfl_sync(0xffffffffu, pos, holder);
  if (lane == 0) s_max[ql] = m, s_pos[ql] = pos;
  __syncwarp();
}

template <typename T, bool FILT, int QB, int TQ>
__global__ void __launch_bounds__(LP_THREADS, 1) count_hamming_kernel(
    const T* __restrict__ rows, uint32_t dim, uint64_t n_rows, const uint8_t* __restrict__ skip,
    const CountKey<T>* __restrict__ qkey, uint32_t nq, uint32_t k, uint32_t n_ranges, uint32_t* __restrict__ cnt,
    uint64_t* __restrict__ rr_key, double* __restrict__ rr_dist, uint32_t* __restrict__ rr_row, uint32_t rr_stride,
    FiltArg filt) {
  using K = CountKey<T>;
  constexpr int NTQ = QB / TQ, NTR = LP_THREADS / NTQ, TR = LP_RB / NTR;
  constexpr int XL = LP_RB * LP_KC / LP_THREADS, QL = QB * LP_KC / LP_THREADS;
  static_assert(NTQ * TQ == QB && NTR * TR == LP_RB && QL >= 1 && NTR <= 32 && 32 % NTR == 0, "tile shape");
  __shared__ __align__(16) K s_x[LP_RB * LP_STRIDE];
  __shared__ __align__(16) K s_q[QB * LP_STRIDE];
  __shared__ uint64_t s_max[QB];  // per local query: the list's largest entry (valid once it is full) ...
  __shared__ uint32_t s_pos[QB];  // ... its position
  __shared__ uint32_t s_fill[QB];
  extern __shared__ uint64_t s_list[];  // [QB][k]
  const uint32_t tid = threadIdx.x, tr = tid % NTR, tq = tid / NTR, lane = tid & 31u;
  const uint32_t n_qb = (nq + QB - 1) / QB;
  const uint32_t n_chunks = (dim + LP_KC - 1) / LP_KC;
  const uint64_t n_steps = (n_rows + LP_RB - 1) / LP_RB;
  const uint64_t items = (uint64_t)n_ranges * n_qb;
  for (uint64_t w = blockIdx.x; w < items; w += gridDim.x) {
    const uint32_t qb0 = (uint32_t)(w % n_qb) * QB, range = (uint32_t)(w / n_qb);
    if (tr == 0)
#pragma unroll
      for (int j = 0; j < TQ; j++) s_fill[tq * TQ + j] = 0, s_max[tq * TQ + j] = ~0ull;
    __syncwarp();
    const uint64_t s_end = (range + 1) * n_steps / n_ranges;
    for (uint64_t step = range * n_steps / n_ranges; step < s_end; step++) {
      const uint64_t row0 = step * LP_RB;
      uint32_t acc[TR][TQ];
#pragma unroll
      for (int i = 0; i < TR; i++)
#pragma unroll
        for (int j = 0; j < TQ; j++) acc[i][j] = 0;
      T xr[XL];
      K qr[QL];
      auto load = [&](uint32_t c0) {
#pragma unroll
        for (int l = 0; l < XL; l++) {
          const uint32_t e = tid + LP_THREADS * l, c = c0 + (e & 31u);
          const uint64_t r = row0 + (e >> 5);
          xr[l] = (r < n_rows && c < dim) ? __ldg(rows + r * dim + c) : T(0);
        }
#pragma unroll
        for (int l = 0; l < QL; l++) {
          const uint32_t e = tid + LP_THREADS * l, c = c0 + (e & 31u), q = qb0 + (e >> 5);
          qr[l] = (q < nq && c < dim) ? __ldg(qkey + (size_t)q * dim + c) : K(0);
        }
      };
      load(0);
      for (uint32_t ch = 0; ch < n_chunks; ch++) {
        __syncthreads();  // the previous chunk has been counted
#pragma unroll
        for (int l = 0; l < XL; l++) {
          const uint32_t e = tid + LP_THREADS * l;
          if constexpr (sizeof(T) == 8) s_x[(e >> 5) * LP_STRIDE + (e & 31u)] = eq_key_f64(xr[l]);
          else s_x[(e >> 5) * LP_STRIDE + (e & 31u)] = eq_key_f32(xr[l]);
        }
#pragma unroll
        for (int l = 0; l < QL; l++) {
          const uint32_t e = tid + LP_THREADS * l;
          s_q[(e >> 5) * LP_STRIDE + (e & 31u)] = qr[l];
        }
        __syncthreads();
        if (ch + 1 < n_chunks) load((ch + 1) * LP_KC);
#pragma unroll 2
        for (int kk = 0; kk < LP_KC; kk += 4) {
          K qv[TQ][4];
#pragma unroll
          for (int j = 0; j < TQ; j++) count_ld4(s_q + (tq * TQ + j) * LP_STRIDE + kk, qv[j]);
#pragma unroll
          for (int i = 0; i < TR; i++) {
            K xv[4];
            count_ld4(s_x + (tr + NTR * i) * LP_STRIDE + kk, xv);
#pragma unroll
            for (int j = 0; j < TQ; j++)
              acc[i][j] += (uint32_t)(xv[0] != qv[j][0]) + (uint32_t)(xv[1] != qv[j][1]) +
                           (uint32_t)(xv[2] != qv[j][2]) + (uint32_t)(xv[3] != qv[j][3]);
          }
        }
      }
      // rows this step may rank: inside the corpus, not skipped / removed (the tombstones are in the skip mask)
      bool row_ok[TR];
#pragma unroll
      for (int i = 0; i < TR; i++) {
        const uint64_t row = row0 + tr + NTR * i;
        row_ok[i] = row < n_rows && !(skip && __ldg(skip + row));
      }
      // insertion: the warp's query groups one after another, each candidate tested against the list's current maximum
#pragma unroll
      for (int g = 0; g < 32 / NTR; g++) {
        const uint32_t tq_g = (tid - lane) / NTR + g;
        const bool mine = lane / NTR == (uint32_t)g;
#pragma unroll
        for (int j = 0; j < TQ; j++) {
          const uint32_t ql = tq_g * TQ + j, q = qb0 + ql;
          if (q >= nq) continue;
          uint64_t* L = s_list + (size_t)ql * k;
#pragma unroll
          for (int i = 0; i < TR; i++) {
            const uint32_t row = (uint32_t)(row0 + tr + NTR * i);
            const uint64_t e = ((uint64_t)acc[i][j] << 32) | row;
            const bool want = mine && row_ok[i] && e < s_max[ql] && (!FILT || filt_pass(filt, q, row));
            uint32_t m = __ballot_sync(0xffffffffu, want);
            while (m) {
              const int src = __ffs(m) - 1;
              m &= m - 1;
              count_list_insert(L, s_max, s_pos, s_fill, ql, k, entry_shfl(e, src), lane);
            }
          }
        }
      }
    }
    // flush: append each list to the query's candidate entries, with the exact distance the count is
#pragma unroll
    for (int g = 0; g < 32 / NTR; g++) {
      const uint32_t tq_g = (tid - lane) / NTR + g;
#pragma unroll
      for (int j = 0; j < TQ; j++) {
        const uint32_t ql = tq_g * TQ + j, q = qb0 + ql;
        if (q >= nq) continue;
        const uint32_t fill = s_fill[ql];
        uint32_t base = 0;
        if (lane == 0 && fill) base = atomicAdd(cnt + q, fill);
        base = __shfl_sync(0xffffffffu, base, 0);
        const uint64_t* L = s_list + (size_t)ql * k;
        for (uint32_t p = lane; p < fill; p += 32) {
          const uint64_t v = L[p];
          const double d = (double)(uint32_t)(v >> 32);
          const size_t o = (size_t)q * rr_stride + base + p;
          rr_key[o] = dist_key(d);
          rr_dist[o] = d;
          rr_row[o] = (uint32_t)v;
        }
      }
    }
    __syncwarp();  // the lists are reset for the next item only after the flush has read them
  }
}

// ---- JACCARD: exact counts from the first-occurrence state, ranked per row range like HAMMING ---------------------------
// Set semantics do not fit the column tiling above (an element meets the query's whole value set, not one column), so
// the work is row-parallel: a CTA takes JQ_QB queries, one per warp, over one row range; each lane takes a row of a
// 32-row step and computes its exact distance with jaccard_counts (O(u_x log u_q)), and the warp keeps its query's k
// smallest (dist_key(d), row) entries with count_list_insert, as the HAMMING kernel does.
constexpr int JQ_QB = 8;

// per query (one CTA each): u_q = distinct values (num_eq_f64: f64 keys), and the sorted keys of those distinct values
// that a row element can equal (f32 rows: the values that some f32 widens to, eq_qkey_f32 != EQ_KEY_NONE).  O(D^2)
// per query, the per-batch pre-pass.  flags: [nq][D] scratch, bit 0 = "a first occurrence that can match".
template <typename K>
__global__ void count_jaccard_qprep_kernel(const double* __restrict__ q64, uint32_t nq, uint32_t dim,
                                           K* __restrict__ qkey, uint32_t* __restrict__ qjac,
                                           uint32_t* __restrict__ flags) {
  const uint32_t q = blockIdx.x;
  if (q >= nq) return;
  __shared__ uint32_t s_uq, s_nl;
  if (threadIdx.x == 0) s_uq = 0, s_nl = 0;
  __syncthreads();
  const double* qv = q64 + (size_t)q * dim;
  uint32_t* fl = flags + (size_t)q * dim;
  auto look = [&](double v) -> K {
    if constexpr (sizeof(K) == 8) return eq_key_f64(v);
    else return eq_qkey_f32(v);
  };
  for (uint32_t j = threadIdx.x; j < dim; j += blockDim.x) {
    const unsigned long long kj = eq_key_f64(qv[j]);
    bool first = true;
    for (uint32_t i = 0; i < j && first; i++) first = eq_key_f64(qv[i]) != kj;
    bool can = false;
    if (first) {
      atomicAdd(&s_uq, 1u);
      can = sizeof(K) == 8 || look(qv[j]) != (K)EQ_KEY_NONE;
      if (can) atomicAdd(&s_nl, 1u);
    }
    fl[j] = can ? 1u : 0u;
  }
  __syncthreads();
  for (uint32_t j = threadIdx.x; j < dim; j += blockDim.x) {
    if (!fl[j]) continue;
    const K kj = look(qv[j]);
    uint32_t pos = 0;  // distinct values have distinct keys: the rank is the sorted position
    for (uint32_t i = 0; i < dim; i++) pos += (fl[i] && look(qv[i]) < kj) ? 1u : 0u;
    qkey[(size_t)q * dim + pos] = kj;
  }
  if (threadIdx.x == 0) qjac[2 * q] = s_uq, qjac[2 * q + 1] = s_nl;
}

template <typename T, bool FILT>
__global__ void __launch_bounds__(JQ_QB * 32) count_jaccard_kernel(
    const T* __restrict__ rows, uint32_t dim, uint64_t n_rows, const uint8_t* __restrict__ skip,
    const uint32_t* __restrict__ jfirst, const uint32_t* __restrict__ jux, const EqKey<T>* __restrict__ qkey,
    const uint32_t* __restrict__ qjac, uint32_t nq, uint32_t k, uint32_t n_ranges, uint32_t* __restrict__ cnt,
    uint64_t* __restrict__ rr_key, double* __restrict__ rr_dist, uint32_t* __restrict__ rr_row, uint32_t rr_stride,
    FiltArg filt) {
  __shared__ JEntry s_max[JQ_QB];
  __shared__ uint32_t s_pos[JQ_QB], s_fill[JQ_QB];
  extern __shared__ __align__(16) unsigned char s_raw[];
  JEntry* s_list = reinterpret_cast<JEntry*>(s_raw);  // [JQ_QB][k]
  const uint32_t lane = threadIdx.x & 31u, ql = threadIdx.x >> 5;
  const uint32_t n_qb = (nq + JQ_QB - 1) / JQ_QB, words = (dim + 31) / 32;
  const uint64_t items = (uint64_t)n_ranges * n_qb;
  JEntry* L = s_list + (size_t)ql * k;
  for (uint64_t w = blockIdx.x; w < items; w += gridDim.x) {
    const uint32_t q = (uint32_t)(w % n_qb) * JQ_QB + ql, range = (uint32_t)(w / n_qb);
    if (q >= nq) continue;  // warp-uniform; the kernel has no block-wide barrier
    if (lane == 0) s_fill[ql] = 0, s_max[ql] = JEntry{~0ull, ~0u};
    __syncwarp();
    const uint32_t uq = __ldg(qjac + 2 * q), n_look = __ldg(qjac + 2 * q + 1);
    const EqKey<T>* qk = qkey + (size_t)q * dim;
    const uint64_t r_end = (range + 1) * n_rows / n_ranges;
    for (uint64_t r0 = range * n_rows / n_ranges; r0 < r_end; r0 += 32) {
      const uint64_t row = r0 + lane;
      const bool ok = row < r_end && !(skip && __ldg(skip + row)) && (!FILT || filt_pass(filt, q, (uint32_t)row));
      JEntry e{~0ull, (uint32_t)row};
      if (ok) e.key = dist_key(jaccard_counts(rows + row * dim, dim, jfirst + row * words, __ldg(jux + row), qk, n_look, uq));
      uint32_t m = __ballot_sync(0xffffffffu, ok && e < s_max[ql]);
      while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        count_list_insert(L, s_max, s_pos, s_fill, ql, k, entry_shfl(e, src), lane);
      }
    }
    // flush, as the HAMMING kernel; a JACCARD distance is never negative or NaN, so the key inverts to it
    const uint32_t fill = s_fill[ql];
    uint32_t base = 0;
    if (lane == 0 && fill) base = atomicAdd(cnt + q, fill);
    base = __shfl_sync(0xffffffffu, base, 0);
    for (uint32_t p = lane; p < fill; p += 32) {
      const JEntry v = L[p];
      const size_t o = (size_t)q * rr_stride + base + p;
      rr_key[o] = v.key;
      rr_dist[o] = __longlong_as_double((long long)(v.key ^ 0x8000000000000000ull));
      rr_row[o] = v.row;
    }
    __syncwarp();
  }
}

// the query keys of the batch, in the key type of the corpus's rows
template <typename K>
__global__ void count_qkeys_kernel(const double* __restrict__ q64, uint32_t nq, uint32_t dim, K* __restrict__ qkey) {
  const uint32_t q = blockIdx.x;
  if (q >= nq) return;
  for (uint32_t c = threadIdx.x; c < dim; c += blockDim.x) {
    const double v = q64[(size_t)q * dim + c];
    if constexpr (sizeof(K) == 8) qkey[(size_t)q * dim + c] = eq_key_f64(v);
    else qkey[(size_t)q * dim + c] = eq_qkey_f32(v);
  }
}

// (query block, queries per thread) by batch size, as launch_lp_qb: a block larger than the batch counts padding
// queries.  f64 keys stop at 32-query blocks, whose staging stays within the 48 KB of static shared memory.
template <typename T, bool FILT, int QB, int TQ>
static sdb_status launch_count(Corpus* c, uint32_t nq, uint32_t k, uint32_t n_ranges, cudaStream_t st) {
  auto kern = count_hamming_kernel<T, FILT, QB, TQ>;
  const size_t smem = sizeof(uint64_t) * QB * k;
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(uint64_t) * QB * 256)));
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, LP_THREADS, smem) != cudaSuccess || per_sm < 1) {
    cudaGetLastError();
    per_sm = 1;
  }
  const uint64_t items = (uint64_t)n_ranges * ((nq + QB - 1) / QB);
  uint64_t grid = (uint64_t)c->ctx->sm_count * per_sm;
  if (grid > items) grid = items;
  kern<<<(unsigned)grid, LP_THREADS, smem, st>>>((const T*)c->d_rows.get(), c->dim, c->n, c->d_skip,
                                                 (const CountKey<T>*)c->d_qkey.get(), nq, k, n_ranges, c->d_cand_cnt,
                                                 c->d_rr_key, c->d_rr_dist, c->d_rr_row, c->rr_stride, c->filt);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}
template <typename T, bool FILT>
static sdb_status launch_count_qb(Corpus* c, uint32_t nq, uint32_t k, uint32_t n_ranges, cudaStream_t st) {
  if (nq <= 8) return launch_count<T, FILT, 8, 1>(c, nq, k, n_ranges, st);
  if constexpr (sizeof(T) == 8) return launch_count<T, FILT, 32, 4>(c, nq, k, n_ranges, st);
  else return nq <= 32 ? launch_count<T, FILT, 32, 4>(c, nq, k, n_ranges, st)
                       : launch_count<T, FILT, 64, 4>(c, nq, k, n_ranges, st);
}
template <typename T>
static sdb_status launch_count_type(Corpus* c, uint32_t nq, uint32_t k, uint32_t n_ranges, cudaStream_t st) {
  return c->filt.bits ? launch_count_qb<T, true>(c, nq, k, n_ranges, st)
                      : launch_count_qb<T, false>(c, nq, k, n_ranges, st);
}

uint32_t count_ranges(const Corpus* c, uint32_t nq, uint32_t k) {
  // as many ranges as 4096-entry lists hold; more, up to 16384 entries, while the work items (range, query block)
  // number fewer than four per SM, so that the last round of the grid-stride loop idles few SMs; never more ranges
  // than 128-row steps
  if (k == 0) return 1;
  const uint32_t qb = nq <= 8 || c->metric == SDB_JACCARD ? 8u : (nq <= 32 || c->dtype == SDB_F64 ? 32u : 64u);
  const uint64_t n_qb = (nq + qb - 1) / qb;
  uint64_t s = 4096 / k;
  if (s * n_qb < 4ull * c->ctx->sm_count) s = std::min<uint64_t>(COUNT_CAP_MAX / k, (4ull * c->ctx->sm_count + n_qb - 1) / n_qb);
  const uint64_t n_steps = (c->n + LP_RB - 1) / LP_RB;
  if (s > n_steps) s = n_steps;
  return s < 1 ? 1u : (uint32_t)s;
}

sdb_status count_prep_queries(Corpus* c, uint32_t nq, cudaStream_t st) {
  if (nq == 0) return SDB_OK;
  if (c->metric == SDB_JACCARD) {
    if (c->dtype == SDB_F32)
      count_jaccard_qprep_kernel<uint32_t><<<nq, 256, 0, st>>>(c->d_q64, nq, c->dim, c->d_qkey.get(), c->d_qjac,
                                                               c->d_qjac + 2 * (size_t)c->sc_nq);
    else
      count_jaccard_qprep_kernel<unsigned long long><<<nq, 256, 0, st>>>(
          c->d_q64, nq, c->dim, (unsigned long long*)c->d_qkey.get(), c->d_qjac, c->d_qjac + 2 * (size_t)c->sc_nq);
  } else if (c->dtype == SDB_F32) {
    count_qkeys_kernel<uint32_t><<<nq, 128, 0, st>>>(c->d_q64, nq, c->dim, c->d_qkey.get());
  } else {
    count_qkeys_kernel<unsigned long long><<<nq, 128, 0, st>>>(c->d_q64, nq, c->dim,
                                                               (unsigned long long*)c->d_qkey.get());
  }
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

template <typename T, bool FILT>
static sdb_status launch_count_jaccard(Corpus* c, uint32_t nq, uint32_t k, uint32_t n_ranges, cudaStream_t st) {
  auto kern = count_jaccard_kernel<T, FILT>;
  const size_t smem = sizeof(JEntry) * JQ_QB * k;  // at most 32 KB
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, JQ_QB * 32, smem) != cudaSuccess || per_sm < 1) {
    cudaGetLastError();
    per_sm = 1;
  }
  const uint64_t items = (uint64_t)n_ranges * ((nq + JQ_QB - 1) / JQ_QB);
  uint64_t grid = (uint64_t)c->ctx->sm_count * per_sm;
  if (grid > items) grid = items;
  kern<<<(unsigned)grid, JQ_QB * 32, smem, st>>>((const T*)c->d_rows.get(), c->dim, c->n, c->d_skip, c->d_jfirst,
                                                 c->d_jux, (const EqKey<T>*)c->d_qkey.get(), c->d_qjac, nq, k,
                                                 n_ranges, c->d_cand_cnt, c->d_rr_key, c->d_rr_dist, c->d_rr_row,
                                                 c->rr_stride, c->filt);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

sdb_status count_pass(Corpus* c, uint32_t nq, uint32_t k, cudaStream_t st) {
  if (nq == 0 || k == 0 || c->n == 0) return SDB_OK;
  const uint32_t n_ranges = count_ranges(c, nq, k);
  if (c->metric == SDB_JACCARD) {
    if (c->dtype == SDB_F32)
      return c->filt.bits ? launch_count_jaccard<float, true>(c, nq, k, n_ranges, st)
                          : launch_count_jaccard<float, false>(c, nq, k, n_ranges, st);
    return c->filt.bits ? launch_count_jaccard<double, true>(c, nq, k, n_ranges, st)
                        : launch_count_jaccard<double, false>(c, nq, k, n_ranges, st);
  }
  return c->dtype == SDB_F32 ? launch_count_type<float>(c, nq, k, n_ranges, st)
                             : launch_count_type<double>(c, nq, k, n_ranges, st);
}

}  // namespace sdb
