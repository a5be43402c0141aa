// candidates.cu -- everything between the screening kernels and the answer:
//   prep_queries : f64 queries -> f32 / bf16 screen copies, exact |q|, special-query flags
//   cand_select  : per query keep the screened candidates whose score reaches tau = (k-th best score) - error margin
//   cand_rerank  : exact f64 distances (the reference's arithmetic, op for op) of the survivors
//   cand_final   : order by (distance, scan position), emit top-k, PROVE that no unscreened row could
//                  belong to it (error-bound check) or flag the query for the exact kernel.
#include <type_traits>

#include "exactmath.cuh"
#include "internal.cuh"
#include "rowwalk.cuh"

namespace sdb {

// ------------------------------------------------------------------------------------------------
// NEG: the f32 / bf16 screen copies (and the measured residual qbferr) are those of -q, negated in f64 before any
// rounding (View::neg); qmag and the flags are those of q, which the negation does not change
template <bool NEG = false>
__global__ void prep_queries_kernel(const double* __restrict__ q64, uint32_t dim, uint32_t dim_pad, int metric,
                                    float* __restrict__ q32, __nv_bfloat16* __restrict__ qbf, double* __restrict__ qmag,
                                    uint32_t* __restrict__ qflags, float* __restrict__ qbferr, uint32_t nq) {
  const uint32_t q = blockIdx.x;
  __shared__ uint32_t s_flags;
  __shared__ float s_err2;
  if (threadIdx.x == 0) {
    s_flags = 0;
    s_err2 = 0.f;
  }
  __syncthreads();
  uint32_t fl = 0;
  float err2 = 0.f;
  if (q < nq) {
    for (uint32_t c = threadIdx.x; c < dim_pad; c += blockDim.x) {
      const double v = c < dim ? (NEG ? -q64[(size_t)q * dim + c] : q64[(size_t)q * dim + c]) : 0.0;
      const float f = (float)v;
      if (q32 && c < dim) q32[(size_t)q * dim + c] = f;
      const __nv_bfloat16 h = __float2bfloat16_rn(f);
      if (qbf) qbf[(size_t)q * dim_pad + c] = h;
      const float d = f - __bfloat162float(h);
      err2 = fmaf(d, d, err2);
      if (v != v) fl |= 3u;               // NaN input: exact path, positive-NaN propagation
      else if (!isfinite(f)) fl |= 1u;    // inf or beyond f32 range: the screen cannot bound its error
    }
  } else {  // padding queries of the bf16 operand tile
    for (uint32_t c = threadIdx.x; c < dim_pad; c += blockDim.x)
      if (qbf) qbf[(size_t)q * dim_pad + c] = __float2bfloat16_rn(0.f);
  }
  if (fl) atomicOr(&s_flags, fl);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) err2 += __shfl_xor_sync(0xffffffffu, err2, o);
  if ((threadIdx.x & 31) == 0 && err2 > 0.f) atomicAdd(&s_err2, err2);
  __syncthreads();
  if (threadIdx.x == 0 && q < nq) {
    double s = 0.0;  // magnitude(): sequential f64, fnc/util/math/vector.rs:301-314
    for (uint32_t c = 0; c < dim; c++) {
      const double v = q64[(size_t)q * dim + c];
      s = __dadd_rn(s, __dmul_rn(v, v));
    }
    const double m = __dsqrt_rn(s);
    qmag[q] = m;
    uint32_t f = s_flags;
    if (metric == SDB_COSINE && (!(m > 0.0) || !isfinite(m))) f |= 1u;
    if (metric != SDB_COSINE && !isfinite(m)) f |= 1u;
    // counts are exact for any value: zero, inf, NaN (a fact of the metric: JACCARD's exact kernel relies on it too)
    if (metric == SDB_HAMMING || metric == SDB_JACCARD) f &= ~1u;
    qflags[q] = f;
    // |q - bf16(q)| / |q|, rounded up; + 2^-23 for the f64 -> f32 rounding of the query itself
    if (qbferr) qbferr[q] = (m > 0.0 && isfinite(m)) ? (sqrtf(s_err2) / (float)m) * 1.0001f + 2.4e-7f : 1.f;
  }
}

// PEARSON: the query's mean m2 and S2 = sum (q_i - m2)^2 in the exact kernel's arithmetic (sequential f64), then the
// screen copies of the NEGATED centred query scaled to unit norm, -dq / |dq| with dq_i = q_i - m2 and |dq| = sqrt(S2)
// in f64: the cosine screens score cos(dx, -dq), which is largest for the smallest pearson (DESIGN.md section 2).  The
// unit norm keeps every f32 product and partial sum of the screens and of stage B below |dx| <= 2^126 (no overflow
// for rows of any magnitude) and, for the screened rows' |dx| >= 2^-100, far above the f32 underflow.  q64 keeps the
// raw query (exact kernel, re-rank); qmag = 1, the norm of the screens' query.  The exact kernel takes a query that is
// constant (S2 = 0), not finite, has an element of dq beyond f32 range, or whose |dq| is below 2^-100 or not a normal
// f32 -- the rules of the rows (finalize_pearson_kernel).
__global__ void prep_queries_pearson_kernel(const double* __restrict__ q64, uint32_t dim, uint32_t dim_pad,
                                            float* __restrict__ q32, __nv_bfloat16* __restrict__ qbf,
                                            double* __restrict__ qmag, double2* __restrict__ qmom,
                                            uint32_t* __restrict__ qflags, float* __restrict__ qbferr, uint32_t nq,
                                            bool desc) {
  const uint32_t q = blockIdx.x;
  __shared__ uint32_t s_flags;
  __shared__ float s_err2;
  __shared__ double s_m2, s_nrm;
  if (threadIdx.x == 0) {
    s_flags = 0;
    s_err2 = 0.f;
    double s2 = 0.0;
    if (q < nq) {
      const double2 mom = pearson_moments(q64 + (size_t)q * dim, dim);
      qmom[q] = mom;
      s_m2 = mom.x;
      s2 = mom.y;
    }
    s_nrm = __dsqrt_rn(s2);
  }
  __syncthreads();
  const double m2 = s_m2, nrm = s_nrm;
  uint32_t fl = 0;
  float err2 = 0.f;
  if (q < nq) {
    for (uint32_t c = threadIdx.x; c < dim_pad; c += blockDim.x) {
      const double x = c < dim ? q64[(size_t)q * dim + c] : 0.0;
      const double dq = c < dim ? __dsub_rn(x, m2) : 0.0;
      const float f = (float)__ddiv_rn(desc ? dq : -dq, nrm);  // (desc: PEARSON DESC, largest pearson first)
      if (c < dim) q32[(size_t)q * dim + c] = f;
      const __nv_bfloat16 h = __float2bfloat16_rn(f);
      qbf[(size_t)q * dim_pad + c] = h;
      const float d = f - __bfloat162float(h);
      if (d == d) err2 = fmaf(d, d, err2);
      if (x != x) fl |= 3u;                           // NaN input: exact path, positive-NaN propagation
      else if (!isfinite((float)dq) || f != f) fl |= 1u;  // inf, or dq beyond f32 range
    }
  } else {  // padding queries of the bf16 operand tile
    for (uint32_t c = threadIdx.x; c < dim_pad; c += blockDim.x) qbf[(size_t)q * dim_pad + c] = __float2bfloat16_rn(0.f);
  }
  if (fl) atomicOr(&s_flags, fl);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) err2 += __shfl_xor_sync(0xffffffffu, err2, o);
  if ((threadIdx.x & 31) == 0 && err2 > 0.f) atomicAdd(&s_err2, err2);
  __syncthreads();
  if (threadIdx.x == 0 && q < nq) {
    qmag[q] = 1.0;
    uint32_t f = s_flags;
    const float mf = (float)nrm;
    if (!(nrm > 0.0) || !isfinite(nrm) || nrm < 0x1p-100 || !(mf >= 1.17549435e-38f && mf <= 3.40282347e38f)) f |= 1u;
    qflags[q] = f;
    // |q^ - bf16(q^)| for the unit query, rounded up; + 2^-23 for its f64 -> f32 rounding (and the f64 division)
    qbferr[q] = (f & 1u) ? 1.f : sqrtf(s_err2) * 1.0001f + 2.4e-7f;
  }
}

// symmetric int8 quantisation of the queries (same scheme as the corpus rows), one block per query
__global__ void __launch_bounds__(128) prep_queries_i8_kernel(const float* __restrict__ q32, const double* __restrict__ qmag,
                                                              uint32_t dim, uint32_t dim_pad8, uint32_t nq,
                                                              int8_t* __restrict__ q8, float* __restrict__ q8scale,
                                                              float* __restrict__ q8err) {
  __shared__ float s_red[4];
  const uint32_t q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int8_t* o = q8 + (size_t)q * dim_pad8;
  if (q >= nq) {
    for (uint32_t c = threadIdx.x; c < dim_pad8; c += blockDim.x) o[c] = 0;
    return;
  }
  const float* x = q32 + (size_t)q * dim;
  float mx = 0.f;
  for (uint32_t c = threadIdx.x; c < dim; c += blockDim.x) mx = fmaxf(mx, fabsf(x[c]));
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o2));
  if (lane == 0) s_red[warp] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(s_red[0], s_red[1]), fmaxf(s_red[2], s_red[3]));
  __syncthreads();
  const bool ok = mx > 0.f && isfinite(mx);
  const float s = ok ? mx / 127.f : 1.f, inv = 1.f / s;
  float err2 = 0.f;
  for (uint32_t c = threadIdx.x; c < dim_pad8; c += blockDim.x) {
    int v = 0;
    if (ok && c < dim) {
      v = __float2int_rn(x[c] * inv);
      v = v > 127 ? 127 : (v < -127 ? -127 : v);
      const float d = x[c] - (float)v * s;
      err2 = fmaf(d, d, err2);
    }
    o[c] = (int8_t)v;
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) err2 += __shfl_xor_sync(0xffffffffu, err2, o2);
  if (lane == 0) s_red[warp] = err2;
  __syncthreads();
  if (threadIdx.x == 0) {
    const float e = s_red[0] + s_red[1] + s_red[2] + s_red[3];
    q8scale[q] = s;
    // relative to the f64 norm; +2^-23 covers the f64 -> f32 rounding of the query itself; rounded up
    q8err[q] = ok ? (sqrtf(e) / (float)qmag[q]) * 1.0001f + 2.4e-7f : 1.f;
  }
}

// ------------------------------------------------------------------------------------------------
// start of a screen: tau = -inf, empty lists, and per query
//   beps   rigorous error bound of the screen that is about to run: cosine -> |sim~ - sim| <= beps;
//          euclid -> |score~ - score| <= beps with score = 2 q.x - |x|^2 (absolute)
//   bscale factor that turns a score into similarity * |q| units (1, or s_q * s for the int8 screen)
//   margin 2.1 x beps in SCORE units (0 in approximate mode).  The k rows with the best screened scores have exact
//          scores >= s_k - beps, so the exact k-th best is >= s_k - beps, and every row whose exact score can reach
//          that has a screened score >= s_k - 2 beps: filtering at tau = s_k - margin keeps all of them.
//   qlow / qcap  bounds of any score of this query (histogram geometry)
// Error bounds (both operands are rounded, ADVICE r1): bf16  e_x + e_q + e_x e_q  with the MEASURED residual norms
// e_x = max_rows |x - bf16(x)|/|x| (finalize) and e_q = |q - bf16(q)|/|q| (prep) -- at most 2^-8 each -- plus fp32
// accumulation D * 2^-21 and 1e-5 for the f32 screening norm; int8  (1 + e_q) e_x + e_q  (integer accumulation is
// exact); f32 SIMT (D/16 + 16) * 2^-23.
// begin_query: what every cand_begin_* kernel leaves per query -- tau = -inf, an empty list, no flags, the bounds above
// (stage B's margin2 / beps2, tau2 = -inf) and the score range qlow .. qcap
__device__ __forceinline__ void begin_query(
    uint32_t q, float* __restrict__ tau, uint32_t* __restrict__ cnt, uint32_t* __restrict__ flags,
    float* __restrict__ bscale, float* __restrict__ beps, float* __restrict__ margin, float* __restrict__ margin2,
    float* __restrict__ beps2, float* __restrict__ tau2, float* __restrict__ qlow, float* __restrict__ qcap, float bs,
    float eps, float mg, float mg2, float e2, float lo, float hi) {
  tau[q] = __int_as_float(0xff800000);  // -inf
  cnt[q] = 0;
  flags[q] = 0;
  bscale[q] = bs;
  beps[q] = eps;
  margin[q] = mg;
  margin2[q] = mg2;
  beps2[q] = e2;
  tau2[q] = __int_as_float(0xff800000);
  qlow[q] = lo;
  qcap[q] = hi;
}
__global__ void cand_begin_kernel(float* __restrict__ tau, uint32_t* __restrict__ cnt, uint32_t* __restrict__ flags,
                                  uint32_t* __restrict__ stat, float* __restrict__ bscale, float* __restrict__ beps,
                                  float* __restrict__ margin, float* __restrict__ margin2, float* __restrict__ beps2,
                                  float* __restrict__ tau2, float* __restrict__ qlow, float* __restrict__ qcap,
                                  const double* __restrict__ qmag, const float* __restrict__ q8scale,
                                  const float* __restrict__ q8err, const float* __restrict__ qbferr, uint32_t nq,
                                  int screen, int metric, uint32_t dim, float max_rel_qerr, float i8_scale,
                                  float bf16_rel_err, float max_norm, int exact, int f64_rows, int far) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q == 0) {
    stat[0] = 0;
    stat[1] = 0;
    stat[2] = 0;
    stat[3] = 0;
  }
  if (q >= nq) return;
  const double qm = qmag[q];
  // f64 rows, cosine: products q_i x_i below 2^-126 may be flushed by the tensor cores (and lose their low bits in
  // stage B's f32 FMA chain), an ABSOLUTE dot error of at most D 2^-126 that no relative term covers.  Screened f64
  // rows have |x| >= 2^-100 (finalize_rows_kernel), so in similarity units it is at most D 2^-26 / |q|: nothing for
  // ordinary queries, while a query so small that it matters gets a bound too wide to prove anything (exact kernel).
  const double u_abs = (f64_rows && metric == SDB_COSINE) ? dim * 0x1p-26 / qm : 0.0;
  double eps_rel, bs = 1.0;
  if (screen == SDB_SCREEN_TC_INT8) {
    const double eq = q8err[q];
    eps_rel = (1.0 + eq) * (double)max_rel_qerr + eq + 2e-6;
    bs = (double)q8scale[q] * (double)i8_scale * 1.000001;
  } else if (screen == SDB_SCREEN_TC_BF16) {
    const double eq = qbferr[q], ex = bf16_rel_err;
    eps_rel = ex + eq + ex * eq + dim * 4.76837158e-7 + 1e-5 + u_abs;
  } else {
    eps_rel = (dim / 16.0 + 16.0) * 1.1920929e-7;
  }
  double eps, mg, lo, hi;
  if (metric == SDB_COSINE) {
    eps = eps_rel;
    mg = 2.1 * eps * qm / bs;
    hi = qm / bs * (1.01 + eps);
    lo = -hi;
  } else {
    const double mn = (double)max_norm;
    eps = 2.0 * eps_rel * qm * mn + 4.8e-7 * (mn * mn + 2.0 * qm * mn) + 1e-30;
    mg = 2.1 * eps;
    hi = qm * qm * 1.01 + eps + 1e-30;
    lo = -(mn * mn + 2.0 * qm * mn) * 1.01 - eps - 1e-30;
    // EuclidFar: |x|^2 - 2 x.q = d^2 - |q|^2 lies in [-|q|^2, M^2 + 2 |q| M], and its error is Euclid's (the same two
    // terms, 2 acc and |x|^2, with the sign of one flipped)
    if (far) {
      const double t = hi;
      hi = -lo;
      lo = -t;
    }
  }
  if (!exact) mg = 0.0;
  if (!(qm > 0.0) || !isfinite(qm) || !isfinite(mg) || !isfinite(hi) || !isfinite(lo)) {  // exact path anyway (qflags)
    mg = 0.0;
    hi = 1.0;
    lo = -1.0;
  }
  // stage B (cand_refine: f32 re-score of the candidates with the f32 rows and the f32 query): any summation order of
  // D products in f32 with FMA stays within (D + 16) * 2^-24 of sum |q_i x_i| <= |q||x| (the +16 covers the f64 -> f32
  // rounding of the query, the f32 screening norm and the final scaling).  f64 rows are rounded to f32 as they are
  // gathered, which moves the dot product by at most 2^-24 sum |q_i x_i| more, plus the underflow term above
  double e2_rel = (dim + 16.0) * 5.9604645e-8;
  if (f64_rows) e2_rel += 5.9604644775390625e-8 + u_abs;
  double e2, mg2;
  if (metric == SDB_COSINE) {
    e2 = e2_rel;
    mg2 = 2.1 * e2 * qm;
  } else {
    const double mn = (double)max_norm;
    e2 = 2.0 * e2_rel * qm * mn + 2.4e-7 * mn * mn + 1e-30;
    mg2 = 2.1 * e2;
  }
  if (!exact || !(qm > 0.0) || !isfinite(qm) || !isfinite(mg2)) mg2 = 0.0;
  begin_query(q, tau, cnt, flags, bscale, beps, margin, margin2, beps2, tau2, qlow, qcap, (float)bs,
              __double2float_ru(eps), __double2float_ru(mg), __double2float_ru(mg2), __double2float_ru(e2),
              __double2float_rd(lo), __double2float_ru(hi));
}
// The same for MANHATTAN / CHEBYSHEV corpora (screen_lp.cu: score = -s~), one warp per query.  beps bounds |s~ - d|
// for every screened row, d = the reference's distance (sequential f64 over the f64 values).  With u = 2^-24,
// Q = sum_i |q^_i|, Qm = max_i |q^_i| (q^ = fl32(q)) and M = max_norm (largest sum_i |x^_i| resp. max_i |x^_i| of a
// screened row; x^ = fl32(x), so x^ = x for f32 rows):
//  - q^_i = q_i (1 + d1) + a1, |d1| <= u, |a1| <= 2^-150 (f32 underflow); the same for x^_i of f64 rows;
//  - t_i = fl32(x^_i - q^_i) = (x^_i - q^_i)(1 + d2), |d2| <= u (an f32 difference in the subnormal range is exact);
//  - MANHATTAN: f32 sums of D non-negative terms in any order err by at most (D-1) u / (1 - (D-1) u) relative (f32
//    additions of non-negative numbers never lose more to underflow); the reference's sequential f64 sum and its f64
//    differences by at most D 2^-53 relative.  Every term is bounded by W = M + Q: sum_i |x^_i - q^_i| <= M + Q, and
//    sum_i |x_i| + |q_i| <= (1 + u) W + D 2^-149.  Summed: |s~ - d| <= (D + 3) u (1 + 2 (D + 3) u) W + D 2^-52 W
//    + D 2^-147;
//  - CHEBYSHEV: a maximum adds no error; |t_i - |x_i - q_i|| <= u (|x^_i| + |q^_i|) (1 + u) + u |q_i| + u |x_i| + 2^-149
//    and the reference's f64 difference adds 2^-53 relative: |s~ - d| <= (3 u + 2^-52) (M + Qm) (1 + 2^-20) + 2^-147.
// A query or a corpus whose W is not a finite f32 gets an infinite bound (tau then proves nothing: exact fallback).
// Stage B (cand_refine) does not run for these metrics: tau2 stays -inf.
__global__ void __launch_bounds__(128) cand_begin_lp_kernel(float* __restrict__ tau, uint32_t* __restrict__ cnt,
                                                            uint32_t* __restrict__ flags, uint32_t* __restrict__ stat,
                                                            float* __restrict__ bscale, float* __restrict__ beps,
                                                            float* __restrict__ margin, float* __restrict__ margin2,
                                                            float* __restrict__ beps2, float* __restrict__ tau2,
                                                            float* __restrict__ qlow, float* __restrict__ qcap,
                                                            const float* __restrict__ q32, uint32_t nq, int metric,
                                                            uint32_t dim, float max_norm, int exact) {
  const uint32_t lane = threadIdx.x & 31u, q = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (blockIdx.x == 0 && threadIdx.x < 4) stat[threadIdx.x] = 0;
  if (q >= nq) return;
  double l1 = 0.0;
  float amax = 0.f;
  for (uint32_t c = lane; c < dim; c += 32) {
    const float v = fabsf(q32[(size_t)q * dim + c]);
    l1 += (double)v;
    amax = fmaxf(amax, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l1 += __shfl_xor_sync(0xffffffffu, l1, o);
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  }
  if (lane != 0) return;
  const double D = (double)dim, u = 0x1p-24;
  double eps, w;
  if (metric == SDB_MANHATTAN) {
    w = (double)max_norm + l1 * (1.0 + 0x1p-30);
    eps = ((D + 3.0) * u * (1.0 + 2.0 * (D + 3.0) * u) + D * 0x1p-52) * w + D * 0x1p-147;
  } else {
    w = (double)max_norm + (double)amax;
    eps = (3.0 * u + 0x1p-52) * w * (1.0 + 0x1p-20) + 0x1p-147;
  }
  double mg = 2.1 * eps, hi = eps + 1e-30, lo = -(w * 1.01 + eps) - 1e-30;
  if (!(w <= 3.4028234663852886e38) || !isfinite(eps)) {  // s~ may overflow f32: no bound
    eps = INFINITY;
    mg = 0.0;
    hi = 1.0;
    lo = -1.0;
  }
  if (!exact) mg = 0.0;
  begin_query(q, tau, cnt, flags, bscale, beps, margin, margin2, beps2, tau2, qlow, qcap, 1.f, __double2float_ru(eps),
              __double2float_ru(mg), 0.f, 0.f, __double2float_rd(lo), __double2float_ru(hi));
}

// MINKOWSKI of integer order p (1 .. 8, minkowski_screen_order): the launch's scale first.  The screen multiplies
// every staged element by s = 2^-e, with 2^e > M + Qb: M = max_norm (the largest |x^_i| of a screened row), Qb = the
// largest |q^_i| of the batch's queries that the screen can bound (qflags bit 0 clear).  Then every |s x^_i - s q^_i|
// <= 1, so no product of minkowski_fma and no power sum of at most 65535 terms overflows.  One warp per query folds
// its largest |q^_i| into mscale[0] (non-negative f32 bits order as integers); cand_begin_minkowski_kernel reads it.
__global__ void __launch_bounds__(128) minkowski_batch_max_kernel(const float* __restrict__ q32,
                                                                  const uint32_t* __restrict__ qflags, uint32_t nq,
                                                                  uint32_t dim, uint32_t* __restrict__ mscale) {
  const uint32_t lane = threadIdx.x & 31u, q = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (q >= nq || (qflags[q] & 1u)) return;
  float amax = 0.f;
  for (uint32_t c = lane; c < dim; c += 32) amax = fmaxf(amax, fabsf(q32[(size_t)q * dim + c]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (lane == 0) atomicMax(mscale, __float_as_uint(amax));
}

// The bound of the MINKOWSKI screen (screen_lp.cu, score = -n~, n~ = fl32(S~^(1/p) 2^e)), one warp per query.  beps
// bounds |n~ - d| for every screened row, d = the exact kernel's distance (pow(sum_i pow(|x_i - q_i|, p), 1/p) in f64,
// sequentially).  With u = 2^-24, R = D^(1/p), M = max_norm, |q^|_p = the query's f32 copy's p-norm and
// W = (R M + |q^|_p + R 2^-148)(1 + 2u) >= |x|_p + |q|_p (the f64 values), by the triangle inequality of the p-norm:
//  - rounding x and q to f32: u W, plus R 2^-149 for the elements that land in or below f32's subnormal range (each
//    moves by up to 2^-150 there, whatever the launch's scale: this term is not multiplied by 2^e);
//  - the f32 subtraction (u W) and the final rounding of n~ (u W, 2^-149 subnormal);
//  - the multiplication chain and the sequential FFMA sum: a relative error g = (D + p - 1) u / (1 - (D + p - 1) u) of
//    the power sum, g / (p (1 - g)) of its root;
//  - underflow under the scale: staging products that land below 2^-126 (2^-150 each, R 2^-149 in norm, times 2^e),
//    and chain / sum roundings below 2^-126 (at most D (p^2 + 1) 2^-149 in the power sum: its p-th root, times 2^e);
//  - the root in f64: CUDA's pow() is within 2 ulp (CUDA C++ Programming Guide, double-precision mathematical functions)
//    and 1/p is rounded (|ln S~| / p 2^-53 relative, S~ >= 2^-149): 2^-44 relative;
//  - the exact kernel: its f64 differences, pow() calls (2 ulp each), sequential sum and final pow() with a rounded 1/p
//    err by at most (D + 2p + 810) 2^-53 relative, and its f64 underflow by (D 2^-1073)^(1/p) absolute.
// beps = (3u + g / (p (1 - g)) + 2^-44 + (D + 2p + 810) 2^-53) W (1 + 2^-20) + R 2^-149 + R 2^-149 2^e
//        + (D (p^2 + 1) 2^-149)^(1/p) 2^e + (D 2^-1073)^(1/p) + 2^-149.
// A query or corpus whose W is not a finite f32, or whose W^p could overflow the exact kernel's f64 sum, gets an
// infinite bound (tau then proves nothing: exact fallback).  Stage B does not run: tau2 stays -inf.
__global__ void __launch_bounds__(128) cand_begin_minkowski_kernel(
    float* __restrict__ tau, uint32_t* __restrict__ cnt, uint32_t* __restrict__ flags, uint32_t* __restrict__ stat,
    float* __restrict__ bscale, float* __restrict__ beps, float* __restrict__ margin, float* __restrict__ margin2,
    float* __restrict__ beps2, float* __restrict__ tau2, float* __restrict__ qlow, float* __restrict__ qcap,
    const float* __restrict__ q32, uint32_t nq, uint32_t dim, int p, float max_norm, uint32_t* __restrict__ mscale,
    int exact) {
  const uint32_t lane = threadIdx.x & 31u, q = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (blockIdx.x == 0 && threadIdx.x < 4) stat[threadIdx.x] = 0;
  // the launch's scale exponent: M + Qb < 2^e (frexp), at least -126 so that s = 2^-e is a finite f32
  const double v = (double)max_norm + (double)__uint_as_float(mscale[0]);
  int e = -126;
  if (v > 0.0) {
    frexp(v, &e);
    if (e < -126) e = -126;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) mscale[1] = (uint32_t)e;
  if (q >= nq) return;
  float amax = 0.f;
  for (uint32_t c = lane; c < dim; c += 32) amax = fmaxf(amax, fabsf(q32[(size_t)q * dim + c]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  // |q^|_p = amax (sum_i (|q^_i| / amax)^p)^(1/p): no overflow for any finite query
  double sp = 0.0;
  if (amax > 0.f && isfinite(amax)) {
    const double inv = 1.0 / (double)amax;
    for (uint32_t c = lane; c < dim; c += 32) {
      const double r = (double)fabsf(q32[(size_t)q * dim + c]) * inv;
      double t = r;
      for (int i = 1; i < p; i++) t *= r;
      sp += t;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sp += __shfl_xor_sync(0xffffffffu, sp, o);
  if (lane != 0) return;
  const double D = (double)dim, u = 0x1p-24, P = (double)p, up = 1.0 + 0x1p-40;
  const double R = pow(D, 1.0 / P) * up, se = ldexp(1.0, e);
  const double qn = amax > 0.f ? (double)amax * pow(sp, 1.0 / P) * up : (double)amax;
  const double w = (R * (double)max_norm + qn + R * 0x1p-148) * (1.0 + 2.0 * u);
  const double gn = (D + P - 1.0) * u, g = gn / (1.0 - gn);
  const double rel = 3.0 * u + g / (P * (1.0 - g)) + 0x1p-44 + (D + 2.0 * P + 810.0) * 0x1p-53;
  double eps = rel * w * (1.0 + 0x1p-20) + R * 0x1p-149 + R * 0x1p-149 * se + pow(D * (P * P + 1.0) * 0x1p-149, 1.0 / P) * up * se +
               pow(D * 0x1p-1073, 1.0 / P) * up + 0x1p-149;
  double mg = 2.1 * eps, hi = eps + 1e-30, lo = -(w * 1.01 + eps) - 1e-30;
  if (!(w <= 3.4028234663852886e38) || !(pow(w, P) <= 1e307) || !isfinite(eps)) {  // no bound
    eps = INFINITY;
    mg = 0.0;
    hi = 1.0;
    lo = -1.0;
  }
  if (!exact) mg = 0.0;
  begin_query(q, tau, cnt, flags, bscale, beps, margin, margin2, beps2, tau2, qlow, qcap, 1.f, __double2float_ru(eps),
              __double2float_ru(mg), 0.f, 0.f, __double2float_rd(lo), __double2float_ru(hi));
}

// Score::Dot (dot_ranking batches): the screens score s~ = x~.q~, with q~ the screen copy of q (DESC) or of -q (ASC),
// and beps bounds |s~ - x.(+-q)| for every screened row.  M = max_norm >= |x| of every screened row (f32, rounded up).
//  - Operand rounding: x~.q~ - x.q = (x~ - x).q~ + x.(q~ - q), so |.| <= (e_x (1 + e_q) + e_q) |x||q| with the measured
//    residuals e_x (bf16_rel_err) and e_q (qbferr: of the copy actually used, -q for ASC) of cand_begin_kernel.
//  - f32 accumulation: at most D 2^-21 of sum |x~_i q~_i| <= |x~||q~| <= 1.01 |x||q| (bf16); the SIMT f32 screen's
//    whole relative term is (D/16 + 16) 2^-23 as above.  So e_rel = e_x + e_q + e_x e_q + 1.01 D 2^-21 (bf16).
//  - Absolute terms, which no relative one covers: an element of the f32 query or of a stage-B row in f32's subnormal
//    range rounds by up to 2^-150 (at most D 2^-150 (|q| + M) over the dot), and the tensor cores or the f32 chains may
//    flush operands, products and partial sums below 2^-126 (at most D 2^-126 (1 + |q| + M) in all); also the
//    reference's own f64 underflow (D 2^-1074; cand_final's eps_ref is relative).  All are inside
//    e_abs = D 2^-120 (1 + |q| + M), for f32 and f64 rows alike.
// beps = e_rel |q| M + e_abs, margin = 2.1 beps in score (= dot) units, bscale = 1, every score lies in
// +-(|q| M 1.01 + beps) (histogram range).  Stage B (cand_refine: f32 rows, or f64 rows rounded to f32 (+2^-24),
// against the f32 copy): beps2 = e2_rel |q| M + e_abs with cand_begin_kernel's e2_rel.  A zero or non-finite |q| takes
// the exact kernel (prep_queries' flags); a bound or score range that is not a finite f32 becomes an infinite bound
// (tau then proves nothing: exact fallback).
__global__ void cand_begin_dot_kernel(float* __restrict__ tau, uint32_t* __restrict__ cnt, uint32_t* __restrict__ flags,
                                      uint32_t* __restrict__ stat, float* __restrict__ bscale, float* __restrict__ beps,
                                      float* __restrict__ margin, float* __restrict__ margin2,
                                      float* __restrict__ beps2, float* __restrict__ tau2, float* __restrict__ qlow,
                                      float* __restrict__ qcap, const double* __restrict__ qmag,
                                      const float* __restrict__ qbferr, uint32_t nq, int screen, uint32_t dim,
                                      float bf16_rel_err, float max_norm, int exact, int f64_rows) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0 && threadIdx.x < 4) stat[threadIdx.x] = 0;
  if (q >= nq) return;
  const double qm = qmag[q], mn = (double)max_norm, D = (double)dim;
  double e_rel;
  if (screen == SDB_SCREEN_TC_BF16) {
    const double eq = qbferr[q], ex = bf16_rel_err;
    e_rel = ex + eq + ex * eq + 1.01 * D * 0x1p-21;
  } else {
    e_rel = (D / 16.0 + 16.0) * 0x1p-23;
  }
  const double e_abs = D * 0x1p-120 * (1.0 + qm + mn);
  double eps = e_rel * qm * mn + e_abs;
  double e2 = ((D + 16.0) * 0x1p-24 + (f64_rows ? 0x1p-24 : 0.0)) * qm * mn + e_abs;
  double mg = 2.1 * eps, mg2 = 2.1 * e2, hi = qm * mn * 1.01 + eps + 1e-30;
  if (!(qm > 0.0) || !(hi <= 3.4028234663852886e38) || !(mg <= 3.4028234663852886e38)) {  // no bound
    eps = e2 = INFINITY;
    mg = mg2 = 0.0;
    hi = 1.0;
  }
  if (!exact) mg = mg2 = 0.0;
  begin_query(q, tau, cnt, flags, bscale, beps, margin, margin2, beps2, tau2, qlow, qcap, 1.f, __double2float_ru(eps),
              __double2float_ru(mg), __double2float_ru(mg2), __double2float_ru(e2), __double2float_rd(-hi),
              __double2float_ru(hi));
}

sdb_status cand_begin(const Corpus* c, Scratch& s, uint32_t nq, int screen, cudaStream_t st, const View& v,
                      bool exact) {
  if (v.sc == Score::Dot) {
    cand_begin_dot_kernel<<<(nq + 255) / 256, 256, 0, st>>>(s.d_tau, s.d_cand_cnt, s.d_flags, s.d_stat, s.d_bscale,
                                                            s.d_beps, s.d_margin, s.d_margin2, s.d_beps2, s.d_tau2,
                                                            s.d_qlow, s.d_qcap, s.d_qmag, s.d_qbferr, nq, screen,
                                                            c->dim, c->bf16_rel_err, c->max_norm, exact ? 1 : 0,
                                                            c->dtype == SDB_F64 ? 1 : 0);
    count_launch(c->ctx);
    SDB_CUDA(cudaGetLastError());
    return SDB_OK;
  }
  switch (family(c)) {
    case Family::Lp:
      if (const int p = minkowski_screen_order(c)) {
        SDB_CUDA(cudaMemsetAsync(s.d_mscale, 0, sizeof(uint32_t), st));
        minkowski_batch_max_kernel<<<(nq + 3) / 4, 128, 0, st>>>(s.d_q32, s.d_qflags, nq, c->dim, s.d_mscale);
        cand_begin_minkowski_kernel<<<(nq + 3) / 4, 128, 0, st>>>(s.d_tau, s.d_cand_cnt, s.d_flags, s.d_stat,
                                                                  s.d_bscale, s.d_beps, s.d_margin, s.d_margin2,
                                                                  s.d_beps2, s.d_tau2, s.d_qlow, s.d_qcap, s.d_q32,
                                                                  nq, c->dim, p, c->max_norm, s.d_mscale,
                                                                  exact ? 1 : 0);
        count_launch(c->ctx);
      } else {
        cand_begin_lp_kernel<<<(nq + 3) / 4, 128, 0, st>>>(s.d_tau, s.d_cand_cnt, s.d_flags, s.d_stat,
                                                           s.d_bscale, s.d_beps, s.d_margin, s.d_margin2,
                                                           s.d_beps2, s.d_tau2, s.d_qlow, s.d_qcap, s.d_q32, nq,
                                                           (int)c->metric, c->dim, c->max_norm, exact ? 1 : 0);
      }
      break;
    case Family::Centred:
      // the cosine bounds of the centred operands with the F64 terms (the rows are centred in f64, whatever their
      // type); the gap between their cosine and the reference's pearson is cand_final's eps_ref
      cand_begin_kernel<<<(nq + 255) / 256, 256, 0, st>>>(s.d_tau, s.d_cand_cnt, s.d_flags, s.d_stat, s.d_bscale,
                                                          s.d_beps, s.d_margin, s.d_margin2, s.d_beps2, s.d_tau2,
                                                          s.d_qlow, s.d_qcap, s.d_qmag, s.d_q8scale, s.d_q8err,
                                                          s.d_qbferr, nq, screen, (int)SDB_COSINE, c->dim,
                                                          c->max_rel_qerr, c->i8_scale, c->bf16_rel_err, c->max_norm,
                                                          exact ? 1 : 0, 1, 0);
      break;
    case Family::Dot: {
      // the bound's form is the view's score, not the corpus metric: Cosine (relative, with the F64 rows' underflow
      // term), or Euclid / EuclidFar (absolute, with max_norm -- an upper bound of |x| over the own screened rows,
      // which include the cross view's)
      const int form = v.sc == Score::Cosine ? (int)SDB_COSINE : (int)SDB_EUCLIDEAN;
      cand_begin_kernel<<<(nq + 255) / 256, 256, 0, st>>>(s.d_tau, s.d_cand_cnt, s.d_flags, s.d_stat, s.d_bscale,
                                                          s.d_beps, s.d_margin, s.d_margin2, s.d_beps2, s.d_tau2,
                                                          s.d_qlow, s.d_qcap, s.d_qmag, s.d_q8scale, s.d_q8err,
                                                          s.d_qbferr, nq, screen, form, c->dim, c->max_rel_qerr,
                                                          c->i8_scale, c->bf16_rel_err, c->max_norm, exact ? 1 : 0,
                                                          c->dtype == SDB_F64 ? 1 : 0, v.sc == Score::EuclidFar);
      break;
    }
    case Family::Count:  // (Count, Exact: the reset of tau, counts, flags and stat; their bounds go unused)
    case Family::Exact:
      cand_begin_kernel<<<(nq + 255) / 256, 256, 0, st>>>(s.d_tau, s.d_cand_cnt, s.d_flags, s.d_stat, s.d_bscale,
                                                          s.d_beps, s.d_margin, s.d_margin2, s.d_beps2, s.d_tau2,
                                                          s.d_qlow, s.d_qcap, s.d_qmag, s.d_q8scale, s.d_q8err,
                                                          s.d_qbferr, nq, screen, (int)c->metric, c->dim,
                                                          c->max_rel_qerr, c->i8_scale, c->bf16_rel_err, c->max_norm,
                                                          exact ? 1 : 0, c->dtype == SDB_F64 ? 1 : 0, 0);
      break;
  }
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

sdb_status scratch_for(const Corpus* c, Scratch& s, uint32_t nq, uint32_t cap) {
  const uint32_t nq_pad = (nq + 127) / 128 * 128;
  if (s.sc_nq >= nq_pad && s.sc_cap >= cap) return SDB_OK;
  const uint32_t nqa = nq_pad > s.sc_nq ? nq_pad : s.sc_nq;
  const uint32_t capa = cap > s.sc_cap ? cap : s.sc_cap;
  s = Scratch();  // everything below is reallocated: prepared queries, candidate lists ... are gone
  auto alloc = [&]() -> sdb_status {
    s.rr_stride = capa + SPECIAL_CAP;
    SDB_CUDA(s.d_q64.reserve((size_t)nqa * c->dim));
    SDB_CUDA(s.d_q32.reserve((size_t)nqa * c->dim));
    SDB_CUDA(s.d_qbf16.reserve((size_t)nqa * c->dim_pad));
    SDB_CUDA(s.d_qmag.reserve(nqa));
    SDB_CUDA(s.d_qflags.reserve(nqa));
    SDB_CUDA(s.d_qbferr.reserve(nqa));
    SDB_CUDA(s.d_tau.reserve(nqa));
    SDB_CUDA(s.d_cand.reserve((size_t)nqa * capa));
    SDB_CUDA(s.d_cand_cnt.reserve(nqa));
    SDB_CUDA(s.d_flags.reserve(nqa));
    SDB_CUDA(s.d_stat.reserve(4));
    SDB_CUDA(s.d_rr_key.reserve((size_t)nqa * s.rr_stride));
    SDB_CUDA(s.d_rr_dist.reserve((size_t)nqa * s.rr_stride));
    SDB_CUDA(s.d_rr_row.reserve((size_t)nqa * s.rr_stride));
    SDB_CUDA(s.d_q8.reserve((size_t)nqa * (c->dim_pad8 ? c->dim_pad8 : 128)));
    SDB_CUDA(s.d_q8scale.reserve(nqa));
    SDB_CUDA(s.d_q8err.reserve(nqa));
    SDB_CUDA(s.d_mscale.reserve(2));
    switch (family(c)) {
      case Family::Centred: SDB_CUDA(s.d_qmom.reserve(nqa)); break;
      case Family::Count:
        SDB_CUDA(s.d_qkey.reserve((size_t)nqa * c->dim * (c->dtype == SDB_F64 ? 2 : 1)));
        if (c->metric == SDB_JACCARD) SDB_CUDA(s.d_qjac.reserve((size_t)nqa * (2 + c->dim)));
        break;
      default: break;
    }
    SDB_CUDA(s.d_bscale.reserve(nqa));
    SDB_CUDA(s.d_beps.reserve(nqa));
    SDB_CUDA(s.d_margin.reserve(nqa));
    SDB_CUDA(s.d_margin2.reserve(nqa));
    SDB_CUDA(s.d_beps2.reserve(nqa));
    SDB_CUDA(s.d_tau2.reserve(nqa));
    SDB_CUDA(s.d_qlow.reserve(nqa));
    SDB_CUDA(s.d_qcap.reserve(nqa));
    SDB_CUDA(s.d_hparam.reserve(nqa));
    SDB_CUDA(s.d_hist.reserve((size_t)nqa * HIST_BINS));
    SDB_CUDA(s.d_probe.reserve((size_t)nqa * PROBE_STRIDE));
    s.sub_slots = 2 * (uint32_t)c->ctx->sm_count;
    s.sub_cap = 16;
    SDB_CUDA(s.d_sub.reserve((size_t)nqa * s.sub_slots * s.sub_cap));
    SDB_CUDA(s.d_sub_cnt.reserve((size_t)nqa * s.sub_slots));
    return SDB_OK;
  };
  const sdb_status rc = alloc();
  if (rc != SDB_OK) {
    s = Scratch();  // empty: the next batch allocates it again
    return rc;
  }
  s.sc_nq = nqa;
  s.sc_cap = capa;
  return SDB_OK;
}

sdb_status prep_queries(const Corpus* c, Scratch& s, const double* d_queries, uint32_t nq, cudaStream_t st,
                        const View& v) {
  // d_queries may alias s.d_q64
  if (d_queries != s.d_q64)
    SDB_CUDA(cudaMemcpyAsync(s.d_q64, d_queries, sizeof(double) * (size_t)nq * c->dim, cudaMemcpyDeviceToDevice, st));
  const uint32_t nq_pad = (nq + 127) / 128 * 128;
  const Family f = family(c);
  if (f == Family::Centred)
    prep_queries_pearson_kernel<<<nq_pad, 128, 0, st>>>(s.d_q64, c->dim, c->dim_pad, s.d_q32, s.d_qbf16, s.d_qmag,
                                                        s.d_qmom, s.d_qflags, s.d_qbferr, nq, v.desc);
  else if (v.neg || v.sc == Score::Dot || v.cross) {
    // the query rule of the view's score: Cosine and Dot (COSINE's) send a zero or non-finite |q| to the exact kernel
    // -- a cosine view of a EUCLIDEAN corpus with |q| = 0 is NaN for every row --, Euclid / EuclidFar a non-finite one
    auto prep = v.neg ? prep_queries_kernel<true> : prep_queries_kernel<false>;
    const int rule = v.sc == Score::Euclid || v.sc == Score::EuclidFar ? (int)SDB_EUCLIDEAN : (int)SDB_COSINE;
    prep<<<nq_pad, 128, 0, st>>>(s.d_q64, c->dim, c->dim_pad, rule, s.d_q32, s.d_qbf16, s.d_qmag, s.d_qflags,
                                 s.d_qbferr, nq);
  } else
    prep_queries_kernel<<<nq_pad, 128, 0, st>>>(s.d_q64, c->dim, c->dim_pad, (int)c->metric, s.d_q32, s.d_qbf16,
                                                s.d_qmag, s.d_qflags, s.d_qbferr, nq);
  count_launch(c->ctx);
  if (f == Family::Count) SDB_TRY(count_prep_queries(c, s, nq, st));
  if (c->d_i8) {
    prep_queries_i8_kernel<<<nq_pad, 128, 0, st>>>(s.d_q32, s.d_qmag, c->dim, c->dim_pad8, nq, s.d_q8, s.d_q8scale,
                                                   s.d_q8err);
    count_launch(c->ctx);
  }
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

sdb_status prep_fallback_query(Corpus* c, const double* d_query, cudaStream_t st) {
  SDB_CUDA(c->d_fb_q.reserve(c->dim));
  SDB_CUDA(c->d_fb_qmag.reserve(1));
  SDB_CUDA(c->d_fb_qflags.reserve(1));
  if (d_query != c->d_fb_q)
    SDB_CUDA(cudaMemcpyAsync(c->d_fb_q, d_query, sizeof(double) * c->dim, cudaMemcpyDeviceToDevice, st));
  // the f32 / bf16 copies are not needed by the exact kernel: q32 goes to a throw-away row of the f64 buffer's size
  prep_queries_kernel<<<1, 128, 0, st>>>(c->d_fb_q, c->dim, c->dim, (int)c->metric, nullptr, nullptr, c->d_fb_qmag,
                                         c->d_fb_qflags, nullptr, 1);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// ------------------------------------------------------------------------------------------------
__global__ void cand_set_count_kernel(uint32_t* cnt, uint32_t nq, uint32_t value) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) cnt[i] = value;
}
sdb_status cand_set_count(const Corpus* c, Scratch& s, uint32_t nq, uint32_t value, cudaStream_t st) {
  cand_set_count_kernel<<<(nq + 255) / 256, 256, 0, st>>>(s.d_cand_cnt, nq, value);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// filtered batches: a pass-0 launch wrote every row of its tiles to fixed slots; the rows a query's filter rejects get
// a NaN score, and cand_select drops them with the invalid rows
__global__ void __launch_bounds__(256) cand_filter_list_kernel(Cand* __restrict__ cand, const uint32_t* __restrict__ cnt,
                                                                uint32_t cap, FiltArg filt) {
  const uint32_t q = blockIdx.x;
  const uint32_t n = cnt[q] < cap ? cnt[q] : cap;
  Cand* cq = cand + (size_t)q * cap;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
    if (!filt_pass(filt, q, cq[i].row)) cq[i].score = __int_as_float(0x7fc00000);
}
sdb_status cand_filter_list(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st) {
  cand_filter_list_kernel<<<nq, 256, 0, st>>>(s.d_cand, s.d_cand_cnt, s.sc_cap, filt);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// filtered batches: the special rows (ranked exactly on every query of an unfiltered batch) join the list of each query
// whose filter passes them, so that the re-rank and the final ordering see exactly the query's own row set
__global__ void __launch_bounds__(256) cand_add_specials_kernel(Cand* __restrict__ cand, uint32_t* __restrict__ cnt,
                                                                 uint32_t* __restrict__ flags, uint32_t cap,
                                                                 const uint32_t* __restrict__ special, uint32_t n_special,
                                                                 FiltArg filt) {
  const uint32_t q = blockIdx.x;
  for (uint32_t i = threadIdx.x; i < n_special; i += blockDim.x) {
    const uint32_t row = special[i];
    if (!filt_pass(filt, q, row)) continue;
    const uint32_t pos = atomicAdd(cnt + q, 1u);
    if (pos < cap) {
      Cand cd;
      cd.score = __int_as_float(0x7f800000);
      cd.row = row;
      cand[(size_t)q * cap + pos] = cd;
    } else {
      atomicOr(flags + q, 1u);  // no room: the query is re-run
    }
  }
}
sdb_status cand_add_specials(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st,
                             const View& v) {
  const uint32_t n_sp = view_n_special(c, v);
  if (!n_sp) return SDB_OK;
  cand_add_specials_kernel<<<nq, 256, 0, st>>>(s.d_cand, s.d_cand_cnt, s.d_flags, s.sc_cap, view_special(c, v), n_sp,
                                               filt);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// direct regime: the query's bitmap words, set bit by set bit; rows past the corpus and skipped / removed rows (the
// tombstones are in the skip mask) are left out.  List order does not matter: cand_final orders by (distance, row).
__global__ void __launch_bounds__(256) cand_direct_kernel(Cand* __restrict__ cand, uint32_t* __restrict__ cnt,
                                                           uint32_t* __restrict__ flags, uint32_t cap, FiltArg filt,
                                                           const uint8_t* __restrict__ skip, uint64_t n) {
  const uint32_t q = blockIdx.x;
  const uint64_t need = (n + 31) / 32;
  const uint32_t nw = need < filt.words ? (uint32_t)need : filt.words;
  const uint32_t* b = filt.bits + (size_t)__ldg(filt.qf + q) * filt.words;
  for (uint32_t w = threadIdx.x; w < nw; w += blockDim.x) {
    uint32_t x = __ldg(b + w);
    while (x) {
      const uint32_t r = w * 32u + (uint32_t)(__ffs(x) - 1);
      x &= x - 1u;
      if (r >= n || (skip && skip[r])) continue;
      const uint32_t pos = atomicAdd(cnt + q, 1u);
      if (pos < cap) {
        Cand cd;
        cd.score = __int_as_float(0x7f800000);
        cd.row = r;
        cand[(size_t)q * cap + pos] = cd;
      } else {
        atomicOr(flags + q, 1u);  // more rows than the list holds: the query is re-run (cannot happen below cap)
      }
    }
  }
}
sdb_status cand_direct(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st) {
  cand_direct_kernel<<<nq, 256, 0, st>>>(s.d_cand, s.d_cand_cnt, s.d_flags, s.sc_cap, filt, c->d_skip, c->n);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

constexpr uint32_t SEL_SMEM_KEYS = 1408;  // 11 KB: cand_select fits beside a resident screen CTA (15 KB are free)

__device__ __forceinline__ Cand key_to_cand(uint64_t key) {
  uint32_t fk = (uint32_t)(key >> 32);
  fk = (fk >> 31) ? (fk & 0x7fffffffu) : ~fk;
  Cand cd;
  cd.score = __uint_as_float(fk);
  cd.row = 0xFFFFFFFFu - (uint32_t)key;
  return cd;
}

// Seed of the streaming pass from a probe launch: the probe wrote, per query, the maximum score of every 32-row chunk
// of a few tiles.  The chunks are disjoint row sets, so the k-th largest chunk maximum s is reached by at least k
// different rows: the k-th best score of the corpus is >= s, and tau = s - margin is a valid first threshold.  Also
// sets up the query's histogram (geometry, zero counts) and empties its lists.  One block of 128 threads per query.
__global__ void __launch_bounds__(128) cand_seed_probe_kernel(const float* __restrict__ probe, uint32_t n_vals, uint32_t k,
                                                              const float* __restrict__ margin,
                                                              const float* __restrict__ qlow, const float* __restrict__ qcap,
                                                              float* __restrict__ tau, uint32_t* __restrict__ cnt,
                                                              HistParam* __restrict__ hparam, uint32_t* __restrict__ hist) {
  __shared__ uint32_t s_key[PROBE_STRIDE];
  const uint32_t q = blockIdx.x;
  uint32_t p2 = 1;
  while (p2 < n_vals) p2 <<= 1;
  for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
    float v = __int_as_float(0xff800000);
    if (i < n_vals) v = probe[(size_t)q * PROBE_STRIDE + i];
    s_key[i] = (v == v) ? f32_key(v) : f32_key(__int_as_float(0xff800000));
  }
  __syncthreads();
  for (uint32_t kk = 2; kk <= p2; kk <<= 1)  // descending bitonic sort of <= 512 keys
    for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const uint32_t a = s_key[i], b = s_key[ixj];
          const bool up = ((i & kk) == 0);
          if (up ? a < b : a > b) {
            s_key[i] = b;
            s_key[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  for (uint32_t i = threadIdx.x; i < HIST_BINS; i += blockDim.x) hist[(size_t)q * HIST_BINS + i] = 0;
  if (threadIdx.x == 0) {
    float t = __int_as_float(0xff800000);
    const float mg = margin[q];
    if (k != 0 && k <= n_vals) {
      uint32_t fk = s_key[k - 1];
      fk = (fk >> 31) ? (fk & 0x7fffffffu) : ~fk;
      const float s_k = __uint_as_float(fk);
      if (s_k > __int_as_float(0xff800000)) t = mg > 0.f ? __fsub_rd(s_k, mg) : s_k;
    }
    HistParam hp;
    hp.lo = t > __int_as_float(0xff800000) ? t : qlow[q];
    float w0 = fmaxf(mg * 0.25f, (qcap[q] - qlow[q]) * 6.1035156e-5f);
    if (!(w0 > 1e-30f) || !isfinite(w0)) w0 = 1e-30f;
    hp.w0 = w0;
    hp.inv_w0 = 1.f / w0;
    hp.margin = mg;
    hparam[q] = hp;
    tau[q] = t;
    cnt[q] = 0;
  }
}
sdb_status cand_seed_from_probe(const Corpus* c, Scratch& s, uint32_t nq, uint32_t k, uint32_t n_tiles,
                                cudaStream_t st) {
  cand_seed_probe_kernel<<<nq, 128, 0, st>>>(s.d_probe, n_tiles * 8, k, s.d_margin, s.d_qlow, s.d_qcap, s.d_tau,
                                             s.d_cand_cnt, s.d_hparam, s.d_hist);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// Per query: gather the main list and the thread-private sub-lists of the tensor-core screens, find the k-th best
// screened score s_k, and keep every candidate with score >= tau = s_k - margin (see cand_begin_kernel).  While fewer
// than k candidates exist everything is kept and tau stays where it is.  tau only ever rises: all rows with a score
// >= an earlier tau were appended under thresholds <= that tau, so the kept set always contains every row seen so far
// whose score reaches the current tau.
__global__ void __launch_bounds__(256) cand_select_kernel(Cand* __restrict__ cand, uint32_t* __restrict__ cnt,
                                                           float* __restrict__ tau, uint32_t* __restrict__ flags,
                                                           uint32_t cap, uint32_t k, const float* __restrict__ margin,
                                                           const float* __restrict__ snorm, const Cand* __restrict__ sub,
                                                           const uint32_t* __restrict__ sub_cnt, uint32_t n_slots,
                                                           uint32_t subcap, uint32_t* __restrict__ stat,
                                                           uint64_t* __restrict__ g_keys, uint32_t g_stride) {
  // keys live in a small shared-memory window (the kernel must fit next to a resident screen CTA: 12 KB); a query that
  // gathered more -- a tight cluster -- sorts in its row of the (still unused) re-rank key buffer instead
  __shared__ uint64_t s_keys_win[SEL_SMEM_KEYS];
  __shared__ uint32_t s_upper;
  __shared__ uint32_t s_n, s_over;
  __shared__ uint32_t s_hist[256];
  __shared__ uint64_t s_prefix;
  __shared__ uint32_t s_remaining, s_out;
  const uint32_t q = blockIdx.x;
  uint32_t n_main = cnt[q];
  if (threadIdx.x == 0) {
    s_over = n_main > cap ? 1u : 0u;
    s_n = 0;
    s_prefix = 0;
    s_remaining = k;
    s_out = 0;
    s_upper = n_main > cap ? cap : n_main;
  }
  if (n_main > cap) n_main = cap;
  __syncthreads();
  {  // upper bound of what the gather can produce decides where the keys go (uniform per block)
    uint32_t part = 0;
    for (uint32_t s = threadIdx.x; s < n_slots; s += blockDim.x) {
      const uint32_t c = sub_cnt[(size_t)q * n_slots + s];
      part += c > subcap ? subcap : c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((threadIdx.x & 31u) == 0 && part) atomicAdd(&s_upper, part);
  }
  __syncthreads();
  uint64_t* s_keys = s_upper > SEL_SMEM_KEYS ? g_keys + (size_t)q * g_stride : s_keys_win;
  auto push = [&](Cand cd) {
    float sc = cd.score;
    if (snorm) {  // integer screens score invalid rows 0: the row's NaN screening norm marks them
      const float sn = snorm[cd.row];
      if (!(sn == sn)) sc = sn;
    }
    if (sc == sc) {  // NaN scores (skipped / special / padding rows) are dropped
      const uint32_t i = atomicAdd(&s_n, 1u);
      if (i < cap) s_keys[i] = ((uint64_t)f32_key(sc) << 32) | (uint64_t)(0xFFFFFFFFu - cd.row);
      else s_over = 1u;
    }
  };
  Cand* cq = cand + (size_t)q * cap;
  for (uint32_t i = threadIdx.x; i < n_main; i += blockDim.x) push(cq[i]);
  for (uint32_t s = threadIdx.x; s < n_slots; s += blockDim.x) {
    uint32_t c = sub_cnt[(size_t)q * n_slots + s];
    if (c > subcap) c = subcap;  // the rest went to the main list
    const Cand* sp = sub + ((size_t)q * n_slots + s) * subcap;
    for (uint32_t e = 0; e < c; e++) push(sp[e]);
  }
  __syncthreads();
  const uint32_t n = s_n < cap ? s_n : cap;
  if (threadIdx.x == 0 && s_over) flags[q] |= 1u;  // candidates were dropped: this query must be re-run exactly
  if (threadIdx.x == 0 && stat) atomicAdd(stat + 3, s_n);  // survivors gathered (diagnostics)
  const float tau_old = tau[q];
  float tau_new = tau_old;
  uint64_t kth = 0;
  const float mg = margin[q];
  if (k != 0 && n >= k) {
    // ---- exact selection of the k-th largest 64-bit key (keys are unique: the row is part of the key) by an MSB-first
    //      radix select, 8 bits per round.  Warp-aggregated histogram updates: the scores of one query share their
    //      leading bytes, so plain shared-memory atomics would serialise on one bin.
    const uint32_t lane = threadIdx.x & 31u;
    // with a margin only the k-th SCORE matters (the keep rule is score >= s_k - margin): 4 rounds over the score half
    // of the key; approximate mode keeps exactly k entries and needs the full (score, row) key: 8 rounds
    const uint32_t n_rounds = mg > 0.f ? 4u : 8u;
    for (uint32_t round = 0; round < n_rounds; round++) {
      const uint32_t shift = 56 - 8 * round;
      s_hist[threadIdx.x] = 0;
      __syncthreads();
      const uint64_t prefix = s_prefix;
      for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {  // uniform trip count: every lane reaches the match below
        const uint32_t i = i0 + threadIdx.x;
        uint32_t digit = 0xFFFFFFFFu;
        if (i < n) {
          const uint64_t key = s_keys[i];
          if (round == 0 || (key >> (shift + 8)) == prefix) digit = (uint32_t)(key >> shift) & 255u;
        }
        const uint32_t peers = __match_any_sync(0xffffffffu, digit);
        if (digit != 0xFFFFFFFFu && lane == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&s_hist[digit], (uint32_t)__popc(peers));
      }
      __syncthreads();
      if (threadIdx.x < 32) {  // one warp: find the digit d with  #(digits > d) < remaining <= #(digits >= d)
        uint32_t c[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
          c[j] = s_hist[255 - (lane * 8 + j)];  // lane 0 holds the 8 largest digits
          sum += c[j];
        }
        uint32_t incl = sum;  // inclusive prefix over lanes (descending digits)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= (uint32_t)o) incl += t;
        }
        const uint32_t rem = s_remaining;
        __syncwarp();  // every lane has read s_remaining before the selected lane overwrites it
        const uint32_t before = incl - sum;  // keys with a digit above this lane's range
        if (before < rem && rem <= incl) {
          uint32_t acc = before;
#pragma unroll
          for (int j = 0; j < 8; j++) {
            if (acc < rem && rem <= acc + c[j]) {
              s_prefix = (prefix << 8) | (uint64_t)(255 - (lane * 8 + j));
              s_remaining = rem - acc;
            }
            acc += c[j];
          }
        }
      }
      __syncthreads();
    }
    kth = n_rounds == 8 ? s_prefix : (s_prefix << 32);  // the k-th largest key itself (score half only with a margin)
    const float s_k = key_to_cand(kth).score;
    const float thr = mg > 0.f ? __fsub_rd(s_k, mg) : s_k;
    tau_new = thr > tau_old ? thr : tau_old;  // (tau_old = -inf the first time)
  }
  // ---- keep: everything while no threshold exists; else score >= tau (approximate mode, margin 0: key >= k-th key) ----
  const bool by_key = (k != 0 && n >= k) && !(mg > 0.f) && tau_new == key_to_cand(kth).score;
  // the kept entries overwrite the head of the main list: positions < n_main were all read during the gather above
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t key = s_keys[i];
    const Cand cd = key_to_cand(key);
    const bool keep = by_key ? key >= kth : cd.score >= tau_new;  // tau_new = -inf keeps everything
    if (keep) cq[atomicAdd(&s_out, 1u)] = cd;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    tau[q] = tau_new;
    cnt[q] = s_out;
  }
}

sdb_status cand_select(const Corpus* c, Scratch& s, uint32_t nq, uint32_t k, bool drop_invalid, uint32_t n_slots,
                       cudaStream_t st, int stage) {
  if (stage == 1) {  // stage B: the lists hold f32 scores now; own threshold / margin, nothing else to gather
    cand_select_kernel<<<nq, 256, 0, st>>>(s.d_cand, s.d_cand_cnt, s.d_tau2, s.d_flags, s.sc_cap, k, s.d_margin2,
                                           nullptr, s.d_sub, s.d_sub_cnt, 0u, s.sub_cap, nullptr, s.d_rr_key,
                                           s.rr_stride);
    count_launch(c->ctx);
    SDB_CUDA(cudaGetLastError());
    return SDB_OK;
  }
  cand_select_kernel<<<nq, 256, 0, st>>>(  // 256 threads: several blocks per SM, the whole batch is one wave
      s.d_cand, s.d_cand_cnt, s.d_tau, s.d_flags, s.sc_cap, k, s.d_margin, drop_invalid ? c->d_snorm.get() : nullptr,
      s.d_sub, s.d_sub_cnt, n_slots, s.sub_cap, s.d_stat, s.d_rr_key, s.rr_stride);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// ------------------------------------------------------------------------------------------------
// stage B: f32 re-score of the candidates.  FP64 is the scarce resource of this part (the sequential-f64 re-rank is
// bound by the FP64 pipe, not by memory), so the candidates of the coarse screen -- everything within the int8 / bf16
// error margin of the k-th best, ~100 rows per query on spread-out data, thousands inside a tight cluster -- are first
// re-scored with the f32 master rows and the f32 query on the FP32 pipe: one warp per row, row-contiguous LDG.128,
// shuffle reduction.  The error of that score is bounded rigorously (cand_begin_kernel: beps2), so the same rule
// "keep everything within 2.1 x the bound of the k-th best" (cand_select, stage 1) shrinks the set to k plus a few
// near-ties, and only those reach the f64 kernel.
// f64 rows: gathered as f64 (16-byte loads when the row length is even) and rounded to f32 element by element before
// the same FMA chain; no f32 copy of the corpus is kept (cand_begin_kernel adds the rounding to beps2).
// CENTRED (PEARSON, f32 and f64 rows): every element is centred in f64 with the row's own mean and then rounded to f32,
// fl32(x_i - m1), against the f32 copy of -dq: the rounding is relative per element, as for f64 cosine rows, so the
// same stage-B bound holds for dx.  (Subtracting fl32(m1) in f32 would err by 2^-24 |m1| per element, absolutely:
// unbounded relative to |dx| for rows whose offset dwarfs their spread.)
// S: the score (View::sc), from the f32 dot a: a / |x|, 2 a - |x|^2, a itself or 2 a + |x|^2
template <typename T, Score S, bool CENTRED = false>
__global__ void __launch_bounds__(128) cand_refine_f32_kernel(const T* __restrict__ rows, uint32_t dim,
                                                               const float* __restrict__ snorm,
                                                               const float* __restrict__ q32, Cand* __restrict__ cand,
                                                               const uint32_t* __restrict__ cnt, uint32_t cap,
                                                               const double2* __restrict__ mom) {
  const uint32_t q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t n_c = cnt[q] < cap ? cnt[q] : cap;
  const float* qv = q32 + (size_t)q * dim;
  Cand* cq = cand + (size_t)q * cap;
  const uint32_t warps_total = gridDim.y * 4;
  const bool vec4 = (dim & 3u) == 0;
  for (uint32_t e0 = (blockIdx.y * 4 + warp) * 2; e0 < n_c; e0 += warps_total * 2) {  // two rows per warp in flight
    const uint32_t r0 = cq[e0].row;
    const bool has1 = e0 + 1 < n_c;
    const uint32_t r1 = has1 ? cq[e0 + 1].row : r0;
    const T* x0 = rows + (size_t)r0 * dim;
    const T* x1 = rows + (size_t)r1 * dim;
    float a0 = 0.f, a1 = 0.f;
    if constexpr (CENTRED) {
      const double m0 = __ldg(&mom[r0].x), m1 = __ldg(&mom[r1].x);
      for (uint32_t c = lane; c < dim; c += 32) {
        const float w = __ldg(qv + c);
        a0 = fmaf(__double2float_rn(__dsub_rn((double)__ldg(x0 + c), m0)), w, a0);
        a1 = fmaf(__double2float_rn(__dsub_rn((double)__ldg(x1 + c), m1)), w, a1);
      }
    } else if constexpr (std::is_same<T, double>::value) {
      if ((dim & 1u) == 0) {
#pragma unroll 2
        for (uint32_t c = lane * 2; c < dim; c += 64) {
          const double2 u = __ldg(reinterpret_cast<const double2*>(x0 + c));
          const double2 v = __ldg(reinterpret_cast<const double2*>(x1 + c));
          const float2 w = __ldg(reinterpret_cast<const float2*>(qv + c));
          a0 = fmaf(__double2float_rn(u.x), w.x, a0); a0 = fmaf(__double2float_rn(u.y), w.y, a0);
          a1 = fmaf(__double2float_rn(v.x), w.x, a1); a1 = fmaf(__double2float_rn(v.y), w.y, a1);
        }
      } else {
        for (uint32_t c = lane; c < dim; c += 32) {
          const float w = __ldg(qv + c);
          a0 = fmaf(__double2float_rn(__ldg(x0 + c)), w, a0);
          a1 = fmaf(__double2float_rn(__ldg(x1 + c)), w, a1);
        }
      }
    } else if (vec4) {
      for (uint32_t c = lane * 4; c < dim; c += 128) {
        const float4 u = __ldg(reinterpret_cast<const float4*>(x0 + c));
        const float4 v = __ldg(reinterpret_cast<const float4*>(x1 + c));
        const float4 w = __ldg(reinterpret_cast<const float4*>(qv + c));
        a0 = fmaf(u.x, w.x, a0); a0 = fmaf(u.y, w.y, a0); a0 = fmaf(u.z, w.z, a0); a0 = fmaf(u.w, w.w, a0);
        a1 = fmaf(v.x, w.x, a1); a1 = fmaf(v.y, w.y, a1); a1 = fmaf(v.z, w.z, a1); a1 = fmaf(v.w, w.w, a1);
      }
    } else {
      for (uint32_t c = lane; c < dim; c += 32) {
        const float w = __ldg(qv + c);
        a0 = fmaf(__ldg(x0 + c), w, a0);
        a1 = fmaf(__ldg(x1 + c), w, a1);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if (lane == 0) {
      if constexpr (S == Score::Dot) {
        cq[e0].score = a0;
        if (has1) cq[e0 + 1].score = a1;
      } else if constexpr (S == Score::EuclidFar) {
        cq[e0].score = fmaf(2.f, a0, __ldg(snorm + r0));
        if (has1) cq[e0 + 1].score = fmaf(2.f, a1, __ldg(snorm + r1));
      } else {
        const float s0 = __ldg(snorm + r0);
        cq[e0].score = S == Score::Cosine ? a0 * s0 : fmaf(2.f, a0, -s0);
        if (has1) {
          const float s1 = __ldg(snorm + r1);
          cq[e0 + 1].score = S == Score::Cosine ? a1 * s1 : fmaf(2.f, a1, -s1);
        }
      }
    }
  }
}
template <Score S>
static void refine_dot(const Corpus* c, Scratch& s, uint32_t nq, cudaStream_t st, const float* snorm) {
  const dim3 grid(nq, 8);
  if (c->dtype == SDB_F32)
    cand_refine_f32_kernel<float, S><<<grid, 128, 0, st>>>((const float*)c->d_rows.get(), c->dim, snorm, s.d_q32,
                                                           s.d_cand, s.d_cand_cnt, s.sc_cap, nullptr);
  else
    cand_refine_f32_kernel<double, S><<<grid, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, snorm, s.d_q32,
                                                            s.d_cand, s.d_cand_cnt, s.sc_cap, nullptr);
}
sdb_status cand_refine(const Corpus* c, Scratch& s, uint32_t nq, cudaStream_t st, const View& v) {
  const dim3 grid(nq, 8);  // 128-thread blocks (register budget beside a resident screen CTA)
  const float* f32_rows = (const float*)c->d_rows.get();
  const double* f64_rows = (const double*)c->d_rows.get();
  switch (family(c)) {
    case Family::Centred:
      if (c->dtype == SDB_F32)
        cand_refine_f32_kernel<float, Score::Cosine, true><<<grid, 128, 0, st>>>(
            f32_rows, c->dim, c->d_snorm, s.d_q32, s.d_cand, s.d_cand_cnt, s.sc_cap, c->d_mom);
      else
        cand_refine_f32_kernel<double, Score::Cosine, true><<<grid, 128, 0, st>>>(
            f64_rows, c->dim, c->d_snorm, s.d_q32, s.d_cand, s.d_cand_cnt, s.sc_cap, c->d_mom);
      break;
    case Family::Dot:
    {
      const float* sn = view_snorm(c, v);
      if (v.sc == Score::Cosine) refine_dot<Score::Cosine>(c, s, nq, st, sn);
      else if (v.sc == Score::Euclid) refine_dot<Score::Euclid>(c, s, nq, st, sn);
      else if (v.sc == Score::EuclidFar) refine_dot<Score::EuclidFar>(c, s, nq, st, sn);
      else refine_dot<Score::Dot>(c, s, nq, st, sn);
    }
      break;
    default: break;  // stage B follows the tensor-core screens (Dot, Centred) only
  }
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// ------------------------------------------------------------------------------------------------
// exact re-rank: per query, every list entry (candidates first, then the special rows) gets the reference's distance
// (RefAcc, exactmath.cuh) and is stored at its entry index for cand_final.  Candidate counts vary per query by orders
// of magnitude (a handful ... a whole cluster).  COSINE / EUCLIDEAN have three load schemes (packed, v4, staged below);
// the other metrics give each entry to one thread (cand_rerank_entry_kernel).
constexpr uint32_t QCHUNK = 1024;  // query columns staged in shared memory per step

constexpr uint32_t RR_GROUPS_Y = 4;  // blocks per query; block y takes the groups y, y + 4, ... of its query

struct RerankOut {  // nq x stride results: the value's key, the value, the row
  uint64_t* key;
  double* dist;
  uint32_t* row;
  uint32_t stride;
  bool desc;  // the descending rankings: keyed descending
  bool sim;   // COSINE steps: the value is the cosine similarity, not the distance (View::sim)
};
__device__ __forceinline__ void rr_store(const RerankOut& out, uint32_t q, uint32_t e, uint32_t row, double d) {
  const size_t o = (size_t)q * out.stride + e;
  out.key[o] = order_key(d, out.desc);
  out.dist[o] = d;
  out.row[o] = row;
}
static RerankOut rr_out(const Scratch& s, bool desc = false, bool sim = false) {
  return RerankOut{s.d_rr_key, s.d_rr_dist, s.d_rr_row, s.rr_stride, desc, sim};
}

// the COSINE / EUCLIDEAN finish of one entry (sim: the cosine similarity instead of the distance; DOT: vector::dot,
// whose entries accumulated the cosine steps).  cosine: the entries accumulated the cosine steps, whatever the corpus
// metric (a cosine view of a EUCLIDEAN corpus finishes with its |x|, d_mag, as a COSINE corpus does)
template <bool DOT = false>
__device__ __forceinline__ double dot_finish(bool cosine, bool sim, const RefSum& s, const double* mag, uint32_t row,
                                             double qm, bool q_nan) {
  if (DOT) return RefAcc<SDB_FN_DOT>{}.finish(s, q_nan);
  if (!cosine) return RefAcc<SDB_EUCLIDEAN>{}.finish(s, q_nan);
  return sim ? RefAcc<SDB_FN_SIMILARITY_COSINE>{}.finish(s, mag[row], qm, q_nan)
             : RefAcc<SDB_COSINE>{}.finish(s, mag[row], qm, q_nan);
}

// Staged: blocks (x = query, y = 0..3) stride over groups of 128 entries; each warp takes 32 entries and walks their
// rows 32 columns at a time: 32 coalesced 128-byte row segments are requested back to back (all in flight before the
// first is consumed -- the kernel is bound by the latency of these gathers, not by the f64 arithmetic), transposed
// through shared memory, and every lane then accumulates ITS row strictly left to right.
// metric: the view's steps (SDB_COSINE or SDB_EUCLIDEAN), not the corpus metric.  DOT (Score::Dot): metric is
// SDB_COSINE (the dot's steps) and the entries finish as vector::dot; so in the others.
constexpr uint32_t RR_WARPS = 4, RR_COLS = 32;
template <typename T, bool DOT = false>
__global__ void __launch_bounds__(RR_WARPS * 32) cand_rerank_kernel(
    const T* __restrict__ rows, uint32_t dim, int metric, const double* __restrict__ mag,
    const double* __restrict__ q64, const double* __restrict__ qmag, const uint32_t* __restrict__ qflags,
    const Cand* __restrict__ cand, const uint32_t* __restrict__ cnt, uint32_t cap, const uint32_t* __restrict__ special,
    uint32_t n_special, RerankOut out) {
  __shared__ T tile[RR_WARPS][32][RR_COLS + 1];
  __shared__ double s_q[QCHUNK];
  const uint32_t q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t n_c = cnt[q] < cap ? cnt[q] : cap;
  const uint32_t n_e = n_c + n_special;
  const bool q_nan = (qflags[q] & 2u) != 0;
  const double qm = qmag[q];
  for (uint32_t e_first = blockIdx.y * (RR_WARPS * 32); e_first < n_e; e_first += gridDim.y * (RR_WARPS * 32)) {  // uniform per block
    const uint32_t e = e_first + warp * 32 + lane;
    uint32_t my_row = NO_ROW;
    if (e < n_c) my_row = cand[(size_t)q * cap + e].row;
    else if (e < n_e) my_row = special[e - n_c];
    const bool warp_active = e_first + warp * 32 < n_e;
    RefSum acc;
    for (uint32_t cb = 0; cb < dim; cb += QCHUNK) {
      const uint32_t cw = dim - cb < QCHUNK ? dim - cb : QCHUNK;
      __syncthreads();
      for (uint32_t i = threadIdx.x; i < cw; i += blockDim.x) s_q[i] = q64[(size_t)q * dim + cb + i];
      __syncthreads();
      if (!warp_active) continue;
      const T* base = rows + cb;
      for (uint32_t c0 = 0; c0 < cw; c0 += RR_COLS) {
        T vals[32];
#pragma unroll
        for (int r = 0; r < 32; r++) {  // 32 independent 128-byte gathers in flight
          const uint32_t row = __shfl_sync(0xffffffffu, my_row, r);
          const uint32_t c = c0 + lane;
          vals[r] = (row != NO_ROW && c < cw) ? __ldg(base + (size_t)row * dim + c) : T(0);
        }
#pragma unroll
        for (int r = 0; r < 32; r++) tile[warp][r][lane] = vals[r];
        __syncwarp();
        if (my_row != NO_ROW) {
          const uint32_t lim = cw - c0 < RR_COLS ? cw - c0 : RR_COLS;
          if (metric == SDB_COSINE) {
            for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_COSINE>{}.step(acc, (double)tile[warp][lane][j], s_q[c0 + j]);
          } else {
            for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_EUCLIDEAN>{}.step(acc, (double)tile[warp][lane][j], s_q[c0 + j]);
          }
        }
        __syncwarp();
      }
    }
    if (my_row != NO_ROW) rr_store(out, q, e, my_row, dot_finish<DOT>(metric == SDB_COSINE, out.sim, acc, mag, my_row, qm, q_nan));
  }
}

// f32 rows whose length is a multiple of 4 (16-byte aligned rows): the gathers are issued ROW-contiguously -- one
// LDG.128 per lane covers 512 consecutive bytes of ONE row, so DRAM sees 512-byte bursts per candidate row instead of
// 128-byte pieces of 32 different rows (random 128-byte gathers reach ~2 TB/s on HBM3e, page-friendly ones several
// times that).  The 32 x 128 tile is then walked per lane with conflict-free LDS.128 (row stride 132 floats).
constexpr uint32_t RRV_COLS = 128, RRV_STRIDE = RRV_COLS + 4;
template <bool DOT = false>
__global__ void __launch_bounds__(RR_WARPS * 32) cand_rerank_v4_kernel(
    const float* __restrict__ rows, uint32_t dim, int metric, const double* __restrict__ mag,
    const double* __restrict__ q64, const double* __restrict__ qmag, const uint32_t* __restrict__ qflags,
    const Cand* __restrict__ cand, const uint32_t* __restrict__ cnt, uint32_t cap, const uint32_t* __restrict__ special,
    uint32_t n_special, RerankOut out) {
  extern __shared__ __align__(16) uint8_t rr_smem[];
  double* s_q = reinterpret_cast<double*>(rr_smem);                                   // [QCHUNK]
  float* tiles = reinterpret_cast<float*>(rr_smem + sizeof(double) * QCHUNK);          // [RR_WARPS][32][RRV_STRIDE]
  const uint32_t q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* tile = tiles + (size_t)warp * 32 * RRV_STRIDE;
  const uint32_t n_c = cnt[q] < cap ? cnt[q] : cap;
  const uint32_t n_e = n_c + n_special;
  const bool q_nan = (qflags[q] & 2u) != 0;
  const double qm = qmag[q];
  for (uint32_t e_first = blockIdx.y * (RR_WARPS * 32); e_first < n_e; e_first += gridDim.y * (RR_WARPS * 32)) {  // uniform per block
    const uint32_t e = e_first + warp * 32 + lane;
    uint32_t my_row = NO_ROW;
    if (e < n_c) my_row = cand[(size_t)q * cap + e].row;
    else if (e < n_e) my_row = special[e - n_c];
    const bool warp_active = e_first + warp * 32 < n_e;
    RefSum acc;
    for (uint32_t cb = 0; cb < dim; cb += QCHUNK) {
      const uint32_t cw = dim - cb < QCHUNK ? dim - cb : QCHUNK;  // multiple of 4
      __syncthreads();
      for (uint32_t i = threadIdx.x; i < cw; i += blockDim.x) s_q[i] = q64[(size_t)q * dim + cb + i];
      __syncthreads();
      if (!warp_active) continue;
      for (uint32_t c0 = 0; c0 < cw; c0 += RRV_COLS) {
        const uint32_t c = c0 + lane * 4;  // this lane's 4 columns of every row
#pragma unroll
        for (int half = 0; half < 2; half++) {
          float4 vals[16];
#pragma unroll
          for (int r = 0; r < 16; r++) {  // 16 independent 512-byte row bursts in flight
            const uint32_t row = __shfl_sync(0xffffffffu, my_row, half * 16 + r);
            vals[r] = (row != NO_ROW && c < cw) ? __ldg(reinterpret_cast<const float4*>(rows + (size_t)row * dim + cb + c))
                                                : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int r = 0; r < 16; r++)
            *reinterpret_cast<float4*>(tile + (size_t)(half * 16 + r) * RRV_STRIDE + lane * 4) = vals[r];
        }
        __syncwarp();
        if (my_row != NO_ROW) {
          const uint32_t lim = cw - c0 < RRV_COLS ? cw - c0 : RRV_COLS;  // multiple of 4
          const float* mine = tile + (size_t)lane * RRV_STRIDE;
          if (metric == SDB_COSINE) {
            const RefAcc<SDB_COSINE> ref;
            for (uint32_t j = 0; j < lim; j += 4) {
              const float4 v = *reinterpret_cast<const float4*>(mine + j);
              ref.step(acc, (double)v.x, s_q[c0 + j]);
              ref.step(acc, (double)v.y, s_q[c0 + j + 1]);
              ref.step(acc, (double)v.z, s_q[c0 + j + 2]);
              ref.step(acc, (double)v.w, s_q[c0 + j + 3]);
            }
          } else {
            const RefAcc<SDB_EUCLIDEAN> ref;
            for (uint32_t j = 0; j < lim; j += 4) {
              const float4 v = *reinterpret_cast<const float4*>(mine + j);
              ref.step(acc, (double)v.x, s_q[c0 + j]);
              ref.step(acc, (double)v.y, s_q[c0 + j + 1]);
              ref.step(acc, (double)v.z, s_q[c0 + j + 2]);
              ref.step(acc, (double)v.w, s_q[c0 + j + 3]);
            }
          }
        }
        __syncwarp();
      }
    }
    if (my_row != NO_ROW) rr_store(out, q, e, my_row, dot_finish<DOT>(metric == SDB_COSINE, out.sim, acc, mag, my_row, qm, q_nan));
  }
}
constexpr size_t RRV_SMEM = sizeof(double) * QCHUNK + sizeof(float) * RR_WARPS * 32 * RRV_STRIDE;  // 75.8 KB


// After the f32 stage a query keeps k candidates plus a few near-ties (about 10 at k = 10), and the exact re-rank is one
// strictly sequential f64 chain per candidate: FP64-issue-bound, nothing to gain from staging.  This variant uses NO
// shared memory and 16 lanes per query (two queries per warp), so that (a) twice as many chains share every FP64
// warp-instruction as with one query per warp, and (b) its blocks run beside the resident screen CTA of the next batch
// (the staged variant's 6 KB per warp let only two warps per SM in, and the re-rank took 0.58 ms instead of 0.1 ms
// whenever it overlapped a screen -- SDB_TRACE timeline, round 2).  Every lane streams its own row (16-byte loads; the
// second half of each 32-byte sector comes from L1) and reads the query from global memory (one address per half-warp).
// f64 rows stream as double2 (16-byte) loads when the row length is even.  M: the view's steps, SDB_COSINE,
// SDB_EUCLIDEAN or SDB_FN_DOT (Score::Dot on either metric).
template <typename T, int M>
__global__ void __launch_bounds__(128) cand_rerank_packed_kernel(
    const T* __restrict__ rows, uint32_t dim, const double* __restrict__ mag, const double* __restrict__ q64,
    const double* __restrict__ qmag, const uint32_t* __restrict__ qflags, const Cand* __restrict__ cand,
    const uint32_t* __restrict__ cnt, uint32_t cap, const uint32_t* __restrict__ special, uint32_t n_special, uint32_t nq,
    RerankOut out) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t q = (blockIdx.x * 4 + warp) * 2 + (lane >> 4), l16 = lane & 15u;
  if (q >= nq) return;
  const uint32_t n_c = cnt[q] < cap ? cnt[q] : cap;
  const uint32_t n_e = n_c + n_special;
  const bool q_nan = (qflags[q] & 2u) != 0;
  const double qm = qmag[q];
  const double* qv = q64 + (size_t)q * dim;
  const bool vec4 = (dim & 3u) == 0;
  const RefAcc<M> ref;
  for (uint32_t e = l16; e < n_e; e += 16) {
    const uint32_t my_row = e < n_c ? cand[(size_t)q * cap + e].row : special[e - n_c];
    const T* x = rows + (size_t)my_row * dim;
    RefSum acc;
    if constexpr (std::is_same<T, double>::value) {
      if ((dim & 1u) == 0) {
#pragma unroll 2
        for (uint32_t j = 0; j < dim; j += 2) {
          const double2 v = __ldg(reinterpret_cast<const double2*>(x + j));
          const double2 qa = __ldg(reinterpret_cast<const double2*>(qv + j));
          ref.step(acc, v.x, qa.x);
          ref.step(acc, v.y, qa.y);
        }
      } else {
        for (uint32_t j = 0; j < dim; j++) ref.step(acc, __ldg(x + j), __ldg(qv + j));
      }
    } else if (vec4) {
#pragma unroll 2
      for (uint32_t j = 0; j < dim; j += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + j));
        const double2 qa = __ldg(reinterpret_cast<const double2*>(qv + j));
        const double2 qb = __ldg(reinterpret_cast<const double2*>(qv + j + 2));
        ref.step(acc, (double)v.x, qa.x);
        ref.step(acc, (double)v.y, qa.y);
        ref.step(acc, (double)v.z, qb.x);
        ref.step(acc, (double)v.w, qb.y);
      }
    } else {
      for (uint32_t j = 0; j < dim; j++) ref.step(acc, (double)__ldg(x + j), __ldg(qv + j));
    }
    rr_store(out, q, e, my_row, dot_finish<M == SDB_FN_DOT>(M == SDB_COSINE, out.sim, acc, mag, my_row, qm, q_nan));
  }
}

// The per-metric inputs of cand_rerank_entry_kernel
struct EntryArgs {
  double mink_p;        // MINKOWSKI: the order
  const double2* mom;   // PEARSON: {m1, S1} per row (finalize_pearson_kernel)
  const double2* qmom;  // ... and {m2, S2} per query (prep_queries_pearson_kernel)
  const uint32_t* jfirst;  // JACCARD: the rows' first-occurrence bitmasks and distinct counts (finalize) ...
  const uint32_t* jux;
  const void* qkey;        // ... and the batch's sorted query keys, EqKey<T>, and {u_q, n_look} (count_prep_queries)
  const uint32_t* qjac;
};

// Every metric but COSINE / EUCLIDEAN: one thread per list entry, its row streamed left to right (the query's elements
// are the same address across the warp); blocks (x = query, y = 0 .. RR_GROUPS_Y - 1) stride over the query's entries.
//  - MANHATTAN / CHEBYSHEV / MINKOWSKI: screened and in the direct regime of filtered batches; HAMMING / JACCARD: the
//    direct regime only (the count path's lists carry exact distances).
//  - PEARSON runs exact_keys_kernel's two passes in one, from the stored means: the row's m1 and S1 and the query's m2
//    and S2 are that kernel's mean and deviation sums bit for bit.
//  - JACCARD: jaccard_counts from the corpus's first-occurrence state and the batch's query keys.
template <typename T, int M>
__global__ void __launch_bounds__(128) cand_rerank_entry_kernel(
    const T* __restrict__ rows, uint32_t dim, const double* __restrict__ q64, const uint32_t* __restrict__ qflags,
    const Cand* __restrict__ cand, const uint32_t* __restrict__ cnt, uint32_t cap, const uint32_t* __restrict__ special,
    uint32_t n_special, RerankOut out, EntryArgs a) {
  const uint32_t q = blockIdx.x;
  const uint32_t n_c = cnt[q] < cap ? cnt[q] : cap;
  const uint32_t n_e = n_c + n_special;
  const bool q_nan = (qflags[q] & 2u) != 0;
  const double* qv = q64 + (size_t)q * dim;
  double2 qm = make_double2(0.0, 0.0);
  double sd2 = 0.0;
  if constexpr (M == SDB_PEARSON) {
    qm = __ldg(a.qmom + q);
    sd2 = RefAcc<SDB_PEARSON>::sd(qm.y, dim);
  }
  for (uint32_t e = blockIdx.y * blockDim.x + threadIdx.x; e < n_e; e += gridDim.y * blockDim.x) {
    const uint32_t row = e < n_c ? cand[(size_t)q * cap + e].row : special[e - n_c];
    const T* x = rows + (size_t)row * dim;
    double d;
    if constexpr (M == SDB_JACCARD) {
      const uint32_t words = (dim + 31) / 32;
      d = jaccard_counts(x, dim, a.jfirst + (size_t)row * words, __ldg(a.jux + row),
                         static_cast<const EqKey<T>*>(a.qkey) + (size_t)q * dim, __ldg(a.qjac + 2 * q + 1),
                         __ldg(a.qjac + 2 * q));
    } else if constexpr (M == SDB_PEARSON) {
      const double2 rm = __ldg(a.mom + row);
      const RefAcc<SDB_PEARSON> ref{rm.x, qm.x};
      RefSum acc;
      for (uint32_t j = 0; j < dim; j++) ref.step(acc, (double)__ldg(x + j), __ldg(qv + j));
      d = ref.finish(acc, dim, RefAcc<SDB_PEARSON>::sd(rm.y, dim), sd2, q_nan);
    } else {
      RefAcc<M> ref;
      if constexpr (M == SDB_MINKOWSKI) ref.p = a.mink_p;
      RefSum acc{RefAcc<M>::start};
      for (uint32_t j = 0; j < dim; j++) ref.step(acc, (double)__ldg(x + j), __ldg(qv + j));
      d = ref.finish(acc, q_nan);
    }
    rr_store(out, q, e, row, d);
  }
}

template <int M>
static void rerank_entry(const Corpus* c, Scratch& s, uint32_t nq, uint32_t n_sp, bool desc, cudaStream_t st) {
  const dim3 grid(nq, RR_GROUPS_Y);
  const EntryArgs a{c->minkowski_p, c->d_mom, s.d_qmom, c->d_jfirst, c->d_jux, s.d_qkey.get(), s.d_qjac};
  if (c->dtype == SDB_F32)
    cand_rerank_entry_kernel<float, M><<<grid, 128, 0, st>>>((const float*)c->d_rows.get(), c->dim, s.d_q64, s.d_qflags,
                                                             s.d_cand, s.d_cand_cnt, s.sc_cap, c->d_special, n_sp,
                                                             rr_out(s, desc), a);
  else
    cand_rerank_entry_kernel<double, M><<<grid, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, s.d_q64,
                                                              s.d_qflags, s.d_cand, s.d_cand_cnt, s.sc_cap,
                                                              c->d_special, n_sp, rr_out(s, desc), a);
}

template <typename T>
static void rerank_packed(const Corpus* c, Scratch& s, uint32_t nq, uint32_t n_sp, const View& v, cudaStream_t st) {
  auto kern = v.steps == SDB_FN_DOT ? cand_rerank_packed_kernel<T, SDB_FN_DOT>
              : v.steps == SDB_COSINE ? cand_rerank_packed_kernel<T, SDB_COSINE>
                                      : cand_rerank_packed_kernel<T, SDB_EUCLIDEAN>;
  kern<<<(nq + 7) / 8, 128, 0, st>>>((const T*)c->d_rows.get(), c->dim, c->d_mag, s.d_q64, s.d_qmag, s.d_qflags,
                                     s.d_cand, s.d_cand_cnt, s.sc_cap, view_special(c, v), n_sp, nq,
                                     rr_out(s, v.desc, v.sim));
}

// COSINE / EUCLIDEAN: the packed kernel for the small sets stage B leaves; otherwise the vectorised one for f32 rows
// of a length divisible by 4, the staged one for the rest
template <bool DOT>
static void rerank_wide(const Corpus* c, Scratch& s, uint32_t nq, uint32_t n_sp, const View& v, cudaStream_t st) {
  const dim3 grid(nq, RR_GROUPS_Y);
  const RerankOut out = rr_out(s, v.desc, v.sim);
  const int metric = DOT ? (int)SDB_COSINE : v.steps;
  const uint32_t* sp = view_special(c, v);
  if (c->dtype == SDB_F32 && c->dim % 4 == 0)
    cand_rerank_v4_kernel<DOT><<<grid, RR_WARPS * 32, RRV_SMEM, st>>>((const float*)c->d_rows.get(), c->dim, metric,
                                                                     c->d_mag, s.d_q64, s.d_qmag, s.d_qflags, s.d_cand,
                                                                     s.d_cand_cnt, s.sc_cap, sp, n_sp, out);
  else if (c->dtype == SDB_F32)
    cand_rerank_kernel<float, DOT><<<grid, RR_WARPS * 32, 0, st>>>((const float*)c->d_rows.get(), c->dim, metric,
                                                                  c->d_mag, s.d_q64, s.d_qmag, s.d_qflags, s.d_cand,
                                                                  s.d_cand_cnt, s.sc_cap, sp, n_sp, out);
  else
    cand_rerank_kernel<double, DOT><<<grid, RR_WARPS * 32, 0, st>>>((const double*)c->d_rows.get(), c->dim, metric,
                                                                   c->d_mag, s.d_q64, s.d_qmag, s.d_qflags, s.d_cand,
                                                                   s.d_cand_cnt, s.sc_cap, sp, n_sp, out);
}
static void rerank_dot(const Corpus* c, Scratch& s, uint32_t nq, bool small_sets, uint32_t n_sp, const View& v,
                       cudaStream_t st) {
  if (small_sets && c->dtype == SDB_F32) rerank_packed<float>(c, s, nq, n_sp, v, st);
  else if (small_sets) rerank_packed<double>(c, s, nq, n_sp, v, st);
  else if (v.sc == Score::Dot) rerank_wide<true>(c, s, nq, n_sp, v, st);
  else rerank_wide<false>(c, s, nq, n_sp, v, st);
}

sdb_status cand_rerank(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, cudaStream_t st,
                       bool small_sets, const View& v) {
  const uint32_t n_sp = filt.bits ? 0u : view_n_special(c, v);  // filtered: the passing special rows are in the lists
  switch (family(c)) {
    case Family::Count:  // (the direct regime only; no special rows)
      if (c->metric == SDB_HAMMING) rerank_entry<SDB_HAMMING>(c, s, nq, n_sp, v.desc, st);
      else rerank_entry<SDB_JACCARD>(c, s, nq, n_sp, v.desc, st);
      break;
    case Family::Lp:
      if (c->metric == SDB_MANHATTAN) rerank_entry<SDB_MANHATTAN>(c, s, nq, n_sp, v.desc, st);
      else if (c->metric == SDB_MINKOWSKI) rerank_entry<SDB_MINKOWSKI>(c, s, nq, n_sp, v.desc, st);
      else rerank_entry<SDB_CHEBYSHEV>(c, s, nq, n_sp, v.desc, st);
      break;
    case Family::Centred:  // one kernel for small (after stage B) and large (direct regime, no stage B) sets
      rerank_entry<SDB_PEARSON>(c, s, nq, n_sp, v.desc, st);
      break;
    case Family::Dot:
    case Family::Exact:  // (never reaches the re-rank: the exact kernel alone ranks it)
      rerank_dot(c, s, nq, small_sets, n_sp, v, st);
      break;
  }
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// ------------------------------------------------------------------------------------------------
// final ordering + proof.  Entries sorted ascending by (Number::cmp key, row) -- exactly the
// DistanceEntry order of KnnTopK (knn_topk.rs:61-73): nearest first, earlier scan position wins ties.  A cosine_desc
// batch's keys are order_key(similarity, desc): most similar first, ties again by scan position (SortTopK's order).
// The candidate count varies per query (a handful on spread-out data, thousands inside a tight cluster), so the sort
// works on a fixed 512-entry window: up to 512 entries are sorted in one go; longer lists are folded in chunks of
// 256 into the running best 256 (k <= 256 on the screened path).
constexpr uint32_t FIN_WIN = 512, FIN_KEEP = 256;  // 8 KB of shared memory, 256 threads: co-resident with a screen CTA

__device__ __forceinline__ void bitonic_pairs(uint64_t* s_key, uint64_t* s_idx, uint32_t p2) {
  for (uint32_t kk = 2; kk <= p2; kk <<= 1) {
    for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const uint64_t ka = s_key[i], kb = s_key[ixj], ia = s_idx[i], ib = s_idx[ixj];
          const bool a_gt_b = ka > kb || (ka == kb && ia > ib);
          const bool up = ((i & kk) == 0);
          if (up ? a_gt_b : !a_gt_b) {
            s_key[i] = kb; s_key[ixj] = ka;
            s_idx[i] = ib; s_idx[ixj] = ia;
          }
        }
      }
      __syncthreads();
    }
  }
}

// What a batch's screens scored, and so which bound the proof derives from a threshold (cand_final picks it from the
// corpus family and the view):
//   Dot        Score::Dot batches; eps_ref = the reference's relative rounding of the dot times max_norm (per |q|)
//   Lp         Lp corpora
//   Centred    the cosine of the centred operands (PEARSON); eps_ref = the gap between it and the reference's pearson
//              (DESIGN.md section 2)
//   CosineNeg  Score::Cosine against the copy of -q (cosine distance DESC, similarity ASC)
//   EuclidFar  Score::EuclidFar; eps_ref = the reference's relative rounding of the euclidean distance
//   Cosine     Score::Cosine against the copy of q
//   Euclid     Score::Euclid; also the count path's lists, whose tau stays -inf
enum class Proof { Dot, Lp, Centred, CosineNeg, EuclidFar, Cosine, Euclid };

// The least key, in the batch's direction, that a row the threshold t excluded can have: its screened score is below t,
// the screen's error is at most beps and its scores are in units of bscale / |q| (stage B: tau2, beps2, bscale 1).
// 0 when the form gives no bound (a NaN or non-positive intermediate): no k-th key is below it, so nothing is proven.
template <Proof P>
__device__ __forceinline__ uint64_t proof_bound(float t, float bscale, float beps, double qm, double eps_ref,
                                                bool desc) {
  if (P == Proof::Dot) {
    // (cand_begin_dot_kernel) a non-candidate's dot with the screened query (q DESC, -q ASC) is at most t + beps, and
    // the reference's sequential f64 dot -- the value keyed -- is within eps_ref |q| of the real one.  DESC: value <= U
    // = t + beps + eps_ref |q|; ASC: value >= -U.  U is rounded up (so -U down)
    const double U = __dadd_ru(__dadd_ru((double)t, (double)beps), __dmul_ru(eps_ref, qm));
    return U == U ? order_key(desc ? U : -U, desc) : 0;
  } else if (P == Proof::Lp) {
    // score = -s~ < t for a non-candidate, so s~ > -t and d >= s~ - beps > -t - beps, rounded down.  No stage B runs
    // (tau2 = -inf)
    return dist_key((-(double)t - (double)beps) * (1.0 - 1e-12));
  } else if (P == Proof::Centred) {
    // the screen scored s = cos(dx, +-dq) |dq| / bscale (+dq DESC).  DESC: cos(dx, dq) <= t bscale / |dq| + beps  =>
    // pearson <= a + beps + eps_ref; ASC: cos(dx, dq) >= -a - beps  =>  pearson >= -a - beps - eps_ref; each bound
    // evaluated with directed rounding so that it is rounded outward
    const double a = __ddiv_ru(__dmul_ru((double)t, (double)bscale), qm);
    if (desc) return order_key(__dadd_ru(__dadd_ru(a, (double)beps), eps_ref), true);
    return dist_key(__dsub_rd(__dsub_rd(-a, (double)beps), eps_ref));
  } else if (P == Proof::CosineNeg) {
    // cos(x, -q) <= U = t bscale / |q| + beps, and the reference's value is within 1e-9 of the real one: sim >= -U,
    // dist = 1 - sim <= 1 + U.  U is rounded up; DESC keys the distance's upper bound, ASC the similarity's lower one
    const double U = __dadd_ru(__dadd_ru(__ddiv_ru(__dmul_ru((double)t, (double)bscale), qm), (double)beps), 1e-9);
    return U == U ? (desc ? order_key(__dadd_ru(1.0, U), true) : dist_key(-U)) : 0;
  } else if (P == Proof::EuclidFar) {
    // 2 x.(-q)~ + |x|^2~ < t for a non-candidate, so d^2 - |q|^2 = |x|^2 - 2 x.q <= t + beps: d^2 <= U = t + beps
    // + |q|^2 (+ the reference's f64 underflow), rounded up, and the reference's distance is at most sqrt(U)
    // (1 + eps_ref), rounded up (keyed descending)
    const double U = __dadd_ru(__dadd_ru(__dadd_ru((double)t, (double)beps), __dmul_ru(qm, qm)), 0x1p-1000);
    const double d = __dmul_ru(__dsqrt_ru(fmax(U, 0.0)), 1.0 + eps_ref);
    return U == U ? order_key(d, true) : 0;
  } else if (P == Proof::Cosine) {
    // non-candidate: score <= t  =>  sim <= t bscale / |q| + eps.  DESC (similarity descending): that upper bound;
    // ASC: dist >= 1 - t bscale / |q| - eps
    if (desc) return order_key((double)t * (double)bscale / qm + (double)beps + 1e-9, true);
    return dist_key(1.0 - (double)t * (double)bscale / qm - (double)beps - 1e-9);
  } else {
    // score = 2 dot~ - |x|^2~ <= t  =>  d^2 = |x|^2 - 2 dot + |q|^2 >= -t + |q|^2 - eps_e.  |q|^2 - t is one fused
    // rounding: written out, the product the two thresholds share may be computed once and rounded on its own
    const double L = fma(qm, qm, -(double)t) - (double)beps;
    return L > 0.0 ? dist_key(sqrt(L) * (1.0 - 1e-12)) : 0;
  }
}

template <Proof P>
__global__ void __launch_bounds__(256)
    cand_final_kernel(const uint64_t* __restrict__ rr_key, const double* __restrict__ rr_dist,
                      const uint32_t* __restrict__ rr_row, uint32_t rr_stride, const uint32_t* __restrict__ cnt,
                      uint32_t cap, uint32_t n_special, const float* __restrict__ tau, const double* __restrict__ qmag,
                      const float* __restrict__ bscale, const float* __restrict__ beps, const float* __restrict__ tau2,
                      const float* __restrict__ beps2, uint32_t* __restrict__ flags, const uint32_t* __restrict__ qflags,
                      uint32_t* __restrict__ stat, uint32_t k, uint64_t row_base, uint64_t* __restrict__ out_rows,
                      double* __restrict__ out_dist, uint32_t* __restrict__ out_count, int debug, double eps_ref,
                      bool desc) {
  __shared__ uint64_t s_key[FIN_WIN];  // distance key
  __shared__ uint64_t s_idx[FIN_WIN];  // (row << 32 | entry): secondary order by row (unique), entry = index into rr_*
  const uint32_t q = blockIdx.x;
  const uint32_t n_c = cnt[q] < cap ? cnt[q] : cap;
  const uint32_t n_e = n_c + n_special;
  const uint64_t* qkey = rr_key + (size_t)q * rr_stride;
  const uint32_t* qrow = rr_row + (size_t)q * rr_stride;
  if (n_e <= FIN_WIN) {
    uint32_t p2 = 1;
    while (p2 < n_e) p2 <<= 1;
    for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
      if (i < n_e) {
        s_key[i] = qkey[i];
        s_idx[i] = ((uint64_t)qrow[i] << 32) | i;
      } else {
        s_key[i] = ~0ull;
        s_idx[i] = ~0ull;
      }
    }
    __syncthreads();
    bitonic_pairs(s_key, s_idx, p2);
  } else {
    for (uint32_t i = threadIdx.x; i < FIN_KEEP; i += blockDim.x) {
      s_key[i] = ~0ull;
      s_idx[i] = ~0ull;
    }
    for (uint32_t c0 = 0; c0 < n_e; c0 += FIN_WIN - FIN_KEEP) {
      __syncthreads();
      for (uint32_t i = threadIdx.x; i < FIN_WIN - FIN_KEEP; i += blockDim.x) {
        const uint32_t e = c0 + i;
        s_key[FIN_KEEP + i] = e < n_e ? qkey[e] : ~0ull;
        s_idx[FIN_KEEP + i] = e < n_e ? (((uint64_t)qrow[e] << 32) | e) : ~0ull;
      }
      __syncthreads();
      bitonic_pairs(s_key, s_idx, FIN_WIN);  // the best FIN_KEEP so far end up in front
    }
  }
  const uint32_t n_out = n_e < k ? n_e : k;
  for (uint32_t i = threadIdx.x; i < n_out; i += blockDim.x) {
    const uint32_t e = (uint32_t)s_idx[i];
    out_rows[(size_t)q * k + i] = row_base + (uint64_t)(s_idx[i] >> 32);
    out_dist[(size_t)q * k + i] = rr_dist[(size_t)q * rr_stride + e];
  }
  if (threadIdx.x == 0) {
    out_count[q] = n_out;
    // ---- proof that no row outside the candidate set can enter the top-k ----
    uint32_t fl = flags[q];
    const float t = tau[q];
    if (t > __int_as_float(0xff800000) && n_e >= k && k > 0) {  // tau == -inf: every screened-in row is a candidate
      const double qm = qmag[q];
      const uint64_t kth = s_key[k - 1];
      // proven when the bound sorts strictly after the k-th entry
      bool ok = proof_bound<P>(t, bscale[q], beps[q], qm, eps_ref, desc) > kth;
      // stage B dropped candidates whose f32 score is below tau2: the same proof with the f32 bound (bscale 1)
      const float t2 = tau2[q];
      if (ok && t2 > __int_as_float(0xff800000)) ok = proof_bound<P>(t2, 1.f, beps2[q], qm, eps_ref, desc) > kth;
      if (!ok) fl |= 2u;
      if (debug && q == 0)
        printf("[sdb final] q0 proof=%d tau=%g qmag=%g beps=%g n_e=%u kth_key=%llx ok=%d\n", (int)P, (double)t, qm,
               (double)beps[q], n_e, (unsigned long long)kth, (int)ok);
    }
    if (fl & 1u) fl |= 2u;  // overflowed candidate buffer => exact re-run
    flags[q] = fl;
    if ((fl & 2u) || (qflags[q] & 1u)) atomicAdd(stat + 0, 1u);  // queries the host still has to repair
    atomicAdd(stat + 1, n_e);
    atomicMax(stat + 2, n_e);
  }
}

sdb_status cand_final(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k, uint64_t row_base,
                      uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count, cudaStream_t st,
                      const View& v) {
  if (k > FIN_KEEP) {
    set_error("cand_final: k = %u exceeds the screened path's limit of %u", k, FIN_KEEP);
    return SDB_EINVAL;
  }
  static const int debug = getenv("SDB_DEBUG") != nullptr;
  const uint32_t n_sp = filt.bits ? 0u : view_n_special(c, v);  // filtered: the passing special rows are in the lists
  auto fin = cand_final_kernel<Proof::Euclid>;
  double eps_ref = 0.0;
  switch (family(c)) {
    case Family::Dot:
      if (v.sc == Score::EuclidFar) {
        fin = cand_final_kernel<Proof::EuclidFar>;
        // the reference's distance sqrt(sum (x_i - q_i)^2) in sequential f64: D roundings of differences, squares and
        // sums err by at most (D + 2) 2^-53 relative on the sum (gamma_D), the square root halves that and adds 2^-53
        eps_ref = (c->dim + 4.0) * 0x1p-53;
      } else if (v.sc == Score::Dot) {
        fin = cand_final_kernel<Proof::Dot>;
        // the reference's sequential f64 dot of D terms errs by at most gamma_D sum |x_i q_i| <= gamma_D |x||q|,
        // gamma_D = D 2^-53 / (1 - D 2^-53) <= (D + 2) 2^-53; |x| <= max_norm; (1 + 2^-20) covers the rounding of
        // |q| (qmag) and of this figure
        eps_ref = (c->dim + 2.0) * 0x1p-53 * (double)c->max_norm * (1.0 + 0x1p-20);
      } else if (v.sc == Score::Cosine) {
        fin = v.neg ? cand_final_kernel<Proof::CosineNeg> : cand_final_kernel<Proof::Cosine>;
      }
      break;
    case Family::Count:  // (tau = -inf: nothing to prove)
    case Family::Exact:  // (never reaches cand_final)
      break;
    case Family::Centred:
      fin = cand_final_kernel<Proof::Centred>;
      // |pearson - cos(dx, dq)| <= (2 D + 6) 2^-53 to first order (DESIGN.md section 2); +2 covers the rest
      eps_ref = (2.0 * c->dim + 8.0) * 0x1p-53;
      break;
    case Family::Lp:
      fin = cand_final_kernel<Proof::Lp>;
      break;
  }
  fin<<<nq, 256, 0, st>>>(s.d_rr_key, s.d_rr_dist, s.d_rr_row, s.rr_stride, s.d_cand_cnt, s.sc_cap, n_sp,
                          s.d_tau, s.d_qmag, s.d_bscale, s.d_beps, s.d_tau2, s.d_beps2, s.d_flags, s.d_qflags,
                          s.d_stat, k, row_base, d_out_rows, d_out_dist, d_out_count, debug, eps_ref, v.desc);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

sdb_status candidates_init_device() {
  SDB_CUDA(cudaFuncSetAttribute(cand_rerank_v4_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RRV_SMEM));
  SDB_CUDA(cudaFuncSetAttribute(cand_rerank_v4_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RRV_SMEM));
  return SDB_OK;
}

}  // namespace sdb
