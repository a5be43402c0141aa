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
#include "exactmath.cuh"
#include "internal.cuh"

namespace sdb {

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
static sdb_status launch_lp(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                            cudaStream_t st) {
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
    kern<<<(unsigned)grid, LP_THREADS, 0, st>>>((const T*)c->d_rows.get(), c->d_snorm, c->dim, c->n, s.d_q32, nq, p,
                                                s.d_tau, s.d_cand, s.d_cand_cnt, s.sc_cap, filt);
  else
    kern<<<(unsigned)grid, LP_THREADS, 0, st>>>((const T*)c->d_rows.get(), c->d_snorm, c->dim, c->n, s.d_q32, nq, p,
                                                s.d_tau, s.d_cand, s.d_cand_cnt, s.sc_cap, filt, s.d_mscale);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// the query block follows the batch: small batches are HBM-bound, and a block larger than the batch spends FP32 work
// on padding queries (an 8-query block at most 7 / 8 of it, a 32-query block for 17-32 queries at most 15 / 32)
template <int METRIC, int P, typename T, bool FILT>
static sdb_status launch_lp_qb(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                               cudaStream_t st) {
  if (nq <= 16) return launch_lp<METRIC, P, T, FILT, 8>(c, s, filt, nq, p, st);
  if (nq <= 32) return launch_lp<METRIC, P, T, FILT, 32>(c, s, filt, nq, p, st);
  return launch_lp<METRIC, P, T, FILT, 64>(c, s, filt, nq, p, st);
}
template <int METRIC, int P = 0>
static sdb_status launch_lp_type(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                                 cudaStream_t st) {
  if (c->dtype == SDB_F32)
    return filt.bits ? launch_lp_qb<METRIC, P, float, true>(c, s, filt, nq, p, st)
                     : launch_lp_qb<METRIC, P, float, false>(c, s, filt, nq, p, st);
  return filt.bits ? launch_lp_qb<METRIC, P, double, true>(c, s, filt, nq, p, st)
                   : launch_lp_qb<METRIC, P, double, false>(c, s, filt, nq, p, st);
}

sdb_status screen_lp_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                          cudaStream_t st) {
  if (p.count == 0 || nq == 0) return SDB_OK;
  switch (minkowski_screen_order(c)) {
    case 1: return launch_lp_type<SDB_MINKOWSKI, 1>(c, s, filt, nq, p, st);
    case 2: return launch_lp_type<SDB_MINKOWSKI, 2>(c, s, filt, nq, p, st);
    case 3: return launch_lp_type<SDB_MINKOWSKI, 3>(c, s, filt, nq, p, st);
    case 4: return launch_lp_type<SDB_MINKOWSKI, 4>(c, s, filt, nq, p, st);
    case 5: return launch_lp_type<SDB_MINKOWSKI, 5>(c, s, filt, nq, p, st);
    case 6: return launch_lp_type<SDB_MINKOWSKI, 6>(c, s, filt, nq, p, st);
    case 7: return launch_lp_type<SDB_MINKOWSKI, 7>(c, s, filt, nq, p, st);
    case 8: return launch_lp_type<SDB_MINKOWSKI, 8>(c, s, filt, nq, p, st);
    default: break;
  }
  return c->metric == SDB_MANHATTAN ? launch_lp_type<SDB_MANHATTAN>(c, s, filt, nq, p, st)
                                    : launch_lp_type<SDB_CHEBYSHEV>(c, s, filt, nq, p, st);
}

}  // namespace sdb
