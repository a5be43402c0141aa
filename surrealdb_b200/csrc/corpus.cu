// corpus.cu -- device-resident vector column: per-row exact magnitudes, screening norms, bf16 screen
// copy, special-row list.  Data layout in HBM (DESIGN.md section 4):
//   rows   [cap][dim]        f32|f64  master copy (exact re-rank reads it; the SIMT screen streams it)
//   bf16   [cap][dim_pad]    bf16     screen copy, K-major rows = wgmma "B" operand via TMA (f32 and f64 rows alike)
//   mag    [cap]             f64      sqrt(sum x^2), the reference's `magnitude()` arithmetic
//   snorm  [cap]             f32      cosine: 1/|x|, euclid: |x|^2, NaN => row never screened in
//   xnorm  [cap]             f32      the other metric's screening norm (cross views), NaN wherever snorm is
#include <algorithm>
#include <type_traits>

#include "exactmath.cuh"
#include "internal.cuh"
#include "rowwalk.cuh"

namespace sdb {

// magnitude_squared: v.iter().map(|a| a.to_float().powi(2)).sum::<f64>()   fnc/util/math/vector.rs:301-303
template <typename T, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) finalize_rows_kernel(const T* __restrict__ rows, uint32_t dim, uint64_t n,
                                                            int metric, const uint8_t* __restrict__ skip,
                                                            double* __restrict__ mag, float* __restrict__ snorm,
                                                            uint32_t* __restrict__ special, uint32_t* special_cnt,
                                                            uint32_t* max_norm_bits) {
  __shared__ T tile[WARPS][32][33];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t warps_total = (uint64_t)gridDim.x * WARPS;
  for (uint64_t base = ((uint64_t)blockIdx.x * WARPS + warp) * 32; base < n; base += warps_total * 32) {
    const uint64_t r = base + lane;
    const uint32_t my_row = r < n ? (uint32_t)r : NO_ROW;
    double s = 0.0;
    double amax = 0.0;  // f64 rows: largest |x_i| (an NaN element makes s NaN, which is special anyway)
    warp_walk_rows<T>(rows, dim, my_row, tile[warp], [&](uint32_t, T x) {
      const double xd = (double)x;
      s = __dadd_rn(s, __dmul_rn(xd, xd));
      if constexpr (std::is_same<T, double>::value) amax = fmax(amax, fabs(xd));
    });
    if (my_row == NO_ROW) continue;
    const double m = __dsqrt_rn(s);
    mag[r] = m;
    const bool skipped = skip && skip[r];
    float sn;
    bool is_special;
    if (metric == SDB_COSINE) {
      is_special = !(m > 0.0) || !isfinite(m);  // zero / NaN / inf norm: distance is NaN or needs exact care
      sn = (float)(1.0 / m);
    } else {
      is_special = !isfinite(s);
      sn = (float)s;
      if (!isfinite(sn)) is_special = true;  // |x|^2 overflows f32: rank exactly
    }
    if constexpr (std::is_same<T, double>::value) {
      // f64 rows the f32 / bf16 operands cannot stand for (the screens and stage B see them only through those):
      //  - an element beyond f32 range (its f32 / bf16 copy is inf);
      //  - |x| or the screening norm (1/|x|, |x|^2) not a finite normal f32: the bounds scale by them in f32;
      //  - a non-zero row with |x| < 2^-100 (f64 subnormals, whose squares vanish, included).  Flushing an element to
      //    f32 / bf16 zero or a subnormal errs by at most 2^-150 (f32) or 2^-134 (bf16) absolutely.  The bf16 and
      //    int8 residuals are measured in f64 and include it; stage B's bound is relative (2^-24 per element), and
      //    sqrt(D) 2^-150 |q| <= 2^-142 |q| stays below 2^-42 |q||x| for |x| >= 2^-100 -- far inside the +16 2^-24
      //    slack of beps2.  An all-zero row is exact in every copy (euclidean screens it; cosine never does).
      const bool nonzero = amax > 0.0;
      const float mf = (float)m;
      const bool m_normal = mf >= 1.17549435e-38f && mf <= 3.40282347e38f;
      const bool sn_normal = fabsf(sn) >= 1.17549435e-38f && fabsf(sn) <= 3.40282347e38f;
      if (!(amax <= 3.4028234663852886e38)) is_special = true;
      if (nonzero && (m < 0x1p-100 || !m_normal || !sn_normal)) is_special = true;
    }
    if (skipped) {
      sn = __int_as_float(0x7fc00000);
    } else if (is_special) {
      sn = __int_as_float(0x7fc00000);
      const uint32_t pos = atomicAdd(special_cnt, 1u);
      if (pos < (uint32_t)SPECIAL_CAP) special[pos] = (uint32_t)r;
    } else {
      atomicMax(max_norm_bits, __float_as_uint((float)m) + 1u);  // +1 ulp: upper bound after rounding
    }
    snorm[r] = sn;
  }
}

// MANHATTAN / CHEBYSHEV / MINKOWSKI corpora (screen_lp.cu).  The screen sees every row through its f32 copy x^ = fl32(x), so a
// row with an element whose f32 copy is not finite (NaN, +-inf, or, in f64 rows, beyond f32 range) is special: ranked
// exactly on every query.  snorm is 0 for screened rows (the score is -(s~ + snorm)) and NaN for skipped / special
// ones.  max_norm = the largest norm of the metric over the screened rows, sum_i |x^_i| (MANHATTAN) or max_i |x^_i|
// (CHEBYSHEV, and MINKOWSKI of any order: its bound and scale need the largest element, which no order change moves),
// summed in f64 and rounded up: the error bound of cand_begin_lp_kernel scales with it.  mag keeps the
// reference's magnitude() arithmetic, as finalize_rows_kernel computes it.
template <typename T, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) finalize_lp_kernel(const T* __restrict__ rows, uint32_t dim, uint64_t n,
                                                                 int metric, const uint8_t* __restrict__ skip,
                                                                 double* __restrict__ mag, float* __restrict__ snorm,
                                                                 uint32_t* __restrict__ special, uint32_t* special_cnt,
                                                                 uint32_t* max_norm_bits) {
  __shared__ T tile[WARPS][32][33];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t warps_total = (uint64_t)gridDim.x * WARPS;
  for (uint64_t base = ((uint64_t)blockIdx.x * WARPS + warp) * 32; base < n; base += warps_total * 32) {
    const uint64_t r = base + lane;
    const uint32_t my_row = r < n ? (uint32_t)r : NO_ROW;
    double s = 0.0, l1 = 0.0, amax = 0.0;
    bool bad = false;
    warp_walk_rows<T>(rows, dim, my_row, tile[warp], [&](uint32_t, T x) {
      const double xd = (double)x;
      s = __dadd_rn(s, __dmul_rn(xd, xd));
      const float f = (float)x;
      bad |= !isfinite(f);
      const double a = fabs((double)f);
      l1 += a;
      amax = fmax(amax, a);
    });
    if (my_row == NO_ROW) continue;
    mag[r] = __dsqrt_rn(s);
    float sn = 0.f;
    if (skip && skip[r]) {
      sn = __int_as_float(0x7fc00000);
    } else if (bad) {
      sn = __int_as_float(0x7fc00000);
      const uint32_t pos = atomicAdd(special_cnt, 1u);
      if (pos < (uint32_t)SPECIAL_CAP) special[pos] = (uint32_t)r;
    } else {
      // the f64 sum of dim f32 magnitudes errs by at most dim 2^-53 relative: (1 + 2^-30) covers it up to dim 2^23
      const double nrm = metric == SDB_MANHATTAN ? l1 * (1.0 + 0x1p-30) : amax;
      atomicMax(max_norm_bits, __float_as_uint(__double2float_ru(nrm)));
    }
    snorm[r] = sn;
  }
}

// PEARSON corpora: the reference ranks pearson = covar / (sd1 sd2) of the rows centred in f64 with their own mean, which
// is the cosine of the centred vectors dx_i = x_i - m1 up to f64 rounding (DESIGN.md section 2, "PEARSON screen").
// So the cosine screens run on dx (f32 and f64 rows alike), and this kernel keeps per row, in the exact kernel's own
// arithmetic (RefAcc<SDB_PEARSON>::mean_step, then step_dev's acc2): mom[r] = {m1 = (sum x) / D, S1 = sum (x_i - m1)^2}, both
// sequential f64, and snorm = fl32(1/sqrt(S1)).  mag stays the magnitude (sdb_corpus_project reads it).  Special rows
// (ranked exactly on every query):
//  - S1 = 0: constant rows (zero and -0.0 rows too, every row when D = 1): pearson is a generated NaN (0/0);
//  - m1 or S1 not finite (a NaN or infinite element);
//  - an element of dx beyond f32 range (its f32 / bf16 copy would be infinite);
//  - sqrt(S1) or 1/sqrt(S1) not a normal f32, or sqrt(S1) < 2^-100: the F64 cosine rules of finalize_rows_kernel,
//    applied to dx.
template <typename T, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) finalize_pearson_kernel(const T* __restrict__ rows, uint32_t dim,
                                                                      uint64_t n, const uint8_t* __restrict__ skip,
                                                                      double* __restrict__ mag, double2* __restrict__ mom,
                                                                      float* __restrict__ snorm,
                                                                      uint32_t* __restrict__ special,
                                                                      uint32_t* special_cnt) {
  __shared__ T tile[WARPS][32][33];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t warps_total = (uint64_t)gridDim.x * WARPS;
  for (uint64_t base = ((uint64_t)blockIdx.x * WARPS + warp) * 32; base < n; base += warps_total * 32) {
    const uint64_t r = base + lane;
    const uint32_t my_row = r < n ? (uint32_t)r : NO_ROW;
    double s = 0.0, sum = 0.0;
    warp_walk_rows<T>(rows, dim, my_row, tile[warp], [&](uint32_t, T x) {
      const double xd = (double)x;
      s = __dadd_rn(s, __dmul_rn(xd, xd));
      sum = __dadd_rn(sum, xd);
    });
    const double m1 = __ddiv_rn(sum, (double)dim);
    double s1 = 0.0, amax = 0.0;
    warp_walk_rows<T>(rows, dim, my_row, tile[warp], [&](uint32_t, T x) {
      const double dx = __dsub_rn((double)x, m1);
      s1 = __dadd_rn(s1, __dmul_rn(dx, dx));
      amax = fmax(amax, fabs(dx));
    });
    if (my_row == NO_ROW) continue;
    mag[r] = __dsqrt_rn(s);
    mom[r] = make_double2(m1, s1);
    const double nrm = __dsqrt_rn(s1);
    float sn = (float)(1.0 / nrm);
    const float nf = (float)nrm;
    const bool n_normal = nf >= 1.17549435e-38f && nf <= 3.40282347e38f;
    const bool sn_normal = fabsf(sn) >= 1.17549435e-38f && fabsf(sn) <= 3.40282347e38f;
    const bool is_special = !(s1 > 0.0) || !isfinite(s1) || !isfinite(m1) || !(amax <= 3.4028234663852886e38) ||
                            nrm < 0x1p-100 || !n_normal || !sn_normal;
    if (skip && skip[r]) {
      sn = __int_as_float(0x7fc00000);
    } else if (is_special) {
      sn = __int_as_float(0x7fc00000);
      const uint32_t pos = atomicAdd(special_cnt, 1u);
      if (pos < (uint32_t)SPECIAL_CAP) special[pos] = (uint32_t)r;
    }
    snorm[r] = sn;
  }
}

// JACCARD corpora with the count path's state (sdb_corpus_create): per row the first-occurrence bitmask (bit i of word
// i / 32 set when no earlier element equals x_i under num_eq_f64, compared through eq_key_row) and the number of
// distinct values u_x.  One warp per row, O(D^2 / 32) compares per lane (early exit on the first equal element).
template <typename T>
__global__ void __launch_bounds__(256) finalize_jaccard_kernel(const T* __restrict__ rows, uint32_t dim, uint64_t n,
                                                               uint32_t* __restrict__ first, uint32_t* __restrict__ ux) {
  const uint32_t lane = threadIdx.x & 31u, words = (dim + 31) / 32;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += n_warps) {
    const T* x = rows + r * dim;
    uint32_t u = 0;
    for (uint32_t w = 0; w < words; w++) {
      const uint32_t i = w * 32 + lane;
      bool f = false;
      if (i < dim) {
        const auto key = eq_key_row(x[i]);
        f = true;
        for (uint32_t j = 0; j < i && f; j++) f = eq_key_row(x[j]) != key;
      }
      const uint32_t bits = __ballot_sync(0xffffffffu, f);
      if (lane == 0) first[r * words + w] = bits;
      u += __popc(bits);
    }
    if (lane == 0) ux[r] = u;
  }
}

// rows in [n, cap_pad) are TMA padding of the last screening tile: NaN norm => never a candidate
__global__ void pad_snorm_kernel(float* __restrict__ snorm, uint64_t n, uint64_t n_pad) {
  const uint64_t i = n + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pad) snorm[i] = __int_as_float(0x7fc00000);
}

// bf16 screen copy, one warp per row; also measures e_x = max over valid rows of |x - bf16(x)| / |x| (the residual
// norm that enters the screen's error bound; at most 2^-8 by construction of round-to-nearest, usually ~0.6 of that)
// f64 rows are rounded to bf16 in one step (cvt.rn.bf16.f64: no double rounding through f32), and their residual is
// measured in f64 against the f64 values, then rounded up to f32.
// CENTRED (PEARSON corpora): the copy holds bf16(dx_i), dx_i = x_i - m1 in f64 for f32 and f64 rows alike, and `mag`
// points at the rows' moments {m1, S1} (finalize_pearson_kernel): the residual is measured in f64 against dx, relative
// to |dx| = sqrt(S1).
template <typename T, bool CENTRED = false>
__global__ void __launch_bounds__(256) to_bf16_kernel(const T* __restrict__ rows, uint32_t dim, uint32_t dim_pad, uint64_t n,
                                                      uint64_t n_pad, const double* __restrict__ mag,
                                                      const float* __restrict__ snorm, __nv_bfloat16* __restrict__ out,
                                                      uint32_t* max_rel_bits) {
  using Acc = typename std::conditional<std::is_same<T, double>::value || CENTRED, double, float>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * 8;
  for (uint64_t r = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n_pad; r += warps) {
    __nv_bfloat16* o = out + r * dim_pad;
    Acc err2 = 0;
    const double m1 = (CENTRED && r < n) ? mag[2 * r] : 0.0;
    for (uint32_t c = lane; c < dim_pad; c += 32) {
      if constexpr (CENTRED) {
        const double v = (r < n && c < dim) ? __dsub_rn((double)rows[r * dim + c], m1) : 0.0;
        const __nv_bfloat16 h = __double2bfloat16(v);
        o[c] = h;
        const double d = v - (double)__bfloat162float(h);
        if (d == d) err2 = fma(d, d, err2);
      } else if constexpr (std::is_same<T, double>::value) {
        const double v = (r < n && c < dim) ? rows[r * dim + c] : 0.0;
        const __nv_bfloat16 h = __double2bfloat16(v);
        o[c] = h;
        const double d = v - (double)__bfloat162float(h);
        if (d == d) err2 = fma(d, d, err2);
      } else {
        const float v = (r < n && c < dim) ? rows[r * dim + c] : 0.f;
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        o[c] = h;
        const float d = v - __bfloat162float(h);
        if (d == d) err2 = fmaf(d, d, err2);
      }
    }
#pragma unroll
    for (int o2 = 16; o2 > 0; o2 >>= 1) err2 += __shfl_xor_sync(0xffffffffu, err2, o2);
    if (lane == 0 && r < n) {
      const float sn = snorm[r];
      const double m = CENTRED ? __dsqrt_rn(mag[2 * r + 1]) : mag[r];
      if (sn == sn && m > 0.0 && isfinite(m) && isfinite(err2)) {  // skipped / special rows never reach the screen
        if constexpr (std::is_same<T, double>::value || CENTRED)  // (1 + 2^-30): the f64 rounding of the figure itself
          atomicMax(max_rel_bits, __float_as_uint(__double2float_ru(sqrt(err2) / m * (1.0 + 0x1p-30))));
        else
          atomicMax(max_rel_bits, __float_as_uint((sqrtf(err2) / (float)m) * 1.0001f + 1e-9f));
      }
    }
  }
}

// int8 screen copy (cosine): the NORMALISED rows x/|x| are quantised with ONE global scale s = gmax/127, so the
// integer dot product q8.x8 is itself the screening score (no per-row weight in the epilogue):
//   sim(q,x) = s_q * s * (q8.x8) / |q|  +  err,   |err| <= (1 + e_q) * e_x + e_q,   e_x = |x/|x| - s*x8|  (per row)
// pass 1: gmax = max over valid rows of max_i |x_i| / |x|
// It also keeps every row's figure (rmax[r]) and a 4096-bin histogram of them over the float bit pattern (8 exponent
// + 4 mantissa bits), from which the host picks the scale: a handful of outlier rows (one dominant component) must not
// dictate the quantisation step of the other ten million.
constexpr uint32_t RMAX_BINS = 4096;
__device__ __host__ inline uint32_t rmax_bin(float v) {  // v > 0
  uint32_t u;
#ifdef __CUDA_ARCH__
  u = __float_as_uint(v);
#else
  memcpy(&u, &v, 4);
#endif
  return (u >> 19) & (RMAX_BINS - 1);
}
// (f64 rows: max_i |x_i| / |x| in f64, rounded up to f32; CENTRED: max_i |dx_i| / sqrt(S1), as to_bf16_kernel)
template <typename T, bool CENTRED = false>
__global__ void __launch_bounds__(256) quantize_scan_kernel(const T* __restrict__ rows, uint32_t dim, uint64_t n,
                                                            const double* __restrict__ mag, const float* __restrict__ snorm,
                                                            uint32_t* gmax_bits, float* __restrict__ rmax,
                                                            uint32_t* __restrict__ hist) {
  __shared__ uint32_t s_hist[RMAX_BINS];
  for (uint32_t i = threadIdx.x; i < RMAX_BINS; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * 8;
  float best = 0.f;
  for (uint64_t r = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += warps) {
    const float sn = snorm[r];
    if (!(sn == sn)) {  // skipped / special
      if (lane == 0) rmax[r] = 0.f;
      continue;
    }
    const T* x = rows + r * dim;
    float v;
    if constexpr (CENTRED) {
      const double m1 = mag[2 * r];
      double mx = 0.0;
      for (uint32_t c = lane; c < dim; c += 32) mx = fmax(mx, fabs(__dsub_rn((double)x[c], m1)));
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o2));
      v = __double2float_ru(mx / __dsqrt_rn(mag[2 * r + 1]));
    } else if constexpr (std::is_same<T, double>::value) {
      double mx = 0.0;
      for (uint32_t c = lane; c < dim; c += 32) mx = fmax(mx, fabs(x[c]));
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o2));
      v = __double2float_ru(mx / mag[r]);
    } else {
      float mx = 0.f;
      for (uint32_t c = lane; c < dim; c += 32) mx = fmaxf(mx, fabsf(x[c]));
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o2));
      v = mx / (float)mag[r];
    }
    best = fmaxf(best, v);
    if (lane == 0) {
      rmax[r] = v;
      if (v > 0.f && isfinite(v)) atomicAdd(&s_hist[rmax_bin(v)], 1u);
    }
  }
  if (lane == 0 && best > 0.f) atomicMax(gmax_bits, __float_as_uint(best));
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < RMAX_BINS; i += blockDim.x)
    if (s_hist[i]) atomicAdd(hist + i, s_hist[i]);
}
// rows whose largest normalised component reaches `thr` become special rows (ranked exactly on every query, never a
// screen candidate): the int8 scale is then set by the remaining rows
__global__ void mark_outliers_kernel(const float* __restrict__ rmax, uint64_t n, float thr, float* __restrict__ snorm,
                                     uint32_t* __restrict__ special, uint32_t* special_cnt) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (rmax[r] >= thr) {
    const float sn = snorm[r];
    if (sn == sn) {
      const uint32_t pos = atomicAdd(special_cnt, 1u);
      if (pos < (uint32_t)SPECIAL_CAP) special[pos] = (uint32_t)r;
      snorm[r] = __int_as_float(0x7fc00000);
    }
  }
}
// pass 2: x8 = clamp(rn(x / (|x| s)), +-127), e_x accumulated exactly as the residual norm (clipping included)
// f64 rows: xn = x / |x| and xn / s in f64 (each correctly rounded), the residual xn - s x8 in f64, rounded up to f32
// CENTRED (PEARSON): the same in f64 with xn = dx / sqrt(S1), dx_i = x_i - m1 (`mag` = the moments, as to_bf16_kernel)
template <typename T, bool CENTRED = false>
__global__ void __launch_bounds__(256) quantize_rows_kernel(const T* __restrict__ rows, uint32_t dim, uint32_t dim_pad8,
                                                            uint64_t n, uint64_t n_pad, const double* __restrict__ mag,
                                                            const float* __restrict__ snorm, const uint32_t* gmax_bits,
                                                            int8_t* __restrict__ out, uint32_t* max_rel_bits) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * 8;
  const float gmax = __uint_as_float(*gmax_bits);
  const float s = gmax > 0.f ? gmax / 127.f : 1.f;
  for (uint64_t r = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n_pad; r += warps) {
    int8_t* o = out + r * dim_pad8;
    const float sn = r < n ? snorm[r] : __int_as_float(0x7fc00000);
    const bool ok = (sn == sn) && gmax > 0.f;
    if (!ok) {  // zero row: scores 0, and compaction drops it through its NaN screening norm
      for (uint32_t c = lane; c < dim_pad8; c += 32) o[c] = 0;
      continue;
    }
    const T* x = rows + r * dim;
    if constexpr (std::is_same<T, double>::value || CENTRED) {
      const double m = CENTRED ? __dsqrt_rn(mag[2 * r + 1]) : mag[r], sd = (double)s;
      const double m1 = CENTRED ? mag[2 * r] : 0.0;
      double err2 = 0.0;
      for (uint32_t c = lane; c < dim_pad8; c += 32) {
        int q = 0;
        if (c < dim) {
          const double xn = (CENTRED ? __dsub_rn((double)x[c], m1) : (double)x[c]) / m;
          q = __double2int_rn(xn / sd);
          q = q > 127 ? 127 : (q < -127 ? -127 : q);
          const double d = xn - (double)q * sd;  // q * s is exact (7 x 24 bits)
          err2 = fma(d, d, err2);
        }
        o[c] = (int8_t)q;
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) err2 += __shfl_xor_sync(0xffffffffu, err2, o2);
      // + 2^-40: the f64 normalisation x / |x| is itself rounded (at most 2^-53 in norm); the whole figure rounded up
      if (lane == 0) atomicMax(max_rel_bits, __float_as_uint(__double2float_ru(sqrt(err2) * (1.0 + 0x1p-30) + 0x1p-40)));
    } else {
      const float inv_norm = 1.f / (float)mag[r];
      const float inv = 1.f / s;
      float err2 = 0.f;
      for (uint32_t c = lane; c < dim_pad8; c += 32) {
        int q = 0;
        if (c < dim) {
          const float xn = x[c] * inv_norm;
          q = __float2int_rn(xn * inv);
          q = q > 127 ? 127 : (q < -127 ? -127 : q);
          const float d = xn - (float)q * s;
          err2 = fmaf(d, d, err2);
        }
        o[c] = (int8_t)q;
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) err2 += __shfl_xor_sync(0xffffffffu, err2, o2);
      // + 2^-22: the f32 normalisation x * (1/|x|) is itself rounded; the whole figure is rounded up
      if (lane == 0) atomicMax(max_rel_bits, __float_as_uint(sqrtf(err2) * 1.0001f + 5e-7f));
    }
  }
}

// The cross state of a COSINE or EUCLIDEAN corpus with a bf16 copy, after the own state is final (outliers included):
// per row the other metric's screening norm and special rule, from the exact magnitude m = mag alone (no pass over the
// rows), as finalize_rows_kernel applies them to that metric:
//  - COSINE corpora, for the euclidean views: fl32(m m).  m m is not the reference's sum of squares s, only m = sqrt(s)
//    is stored: m = sqrt(s) (1 + d1) and fl64(m m) = s (1 + d1)^2 (1 + d2), |d1|, |d2| <= 2^-53, so fl32(m m) is within
//    2^-24 + 3.01 2^-53 of s relatively -- inside the 8 2^-24 |x|^2 (stage A) and 4 2^-24 |x|^2 (stage B) that the
//    euclidean bounds give the screening norm (cand_begin_kernel).  Special: m m or its f32 copy not finite;
//  - EUCLIDEAN corpora, for the cosine views: fl32(1 / m), exactly the COSINE corpus' d_snorm.  Special: m not finite or
//    not above 0 (zero rows: their cosine is the generated NaN, which sorts first in the ascending orders);
//  - f64 rows, either metric: a non-zero row whose |x| or screening norm is not a normal f32 or whose |x| < 2^-100.
// xnorm is NaN wherever snorm is (skipped, removed, own special and outlier rows, padding up to n_pad), and the cross
// special list is the own list (already in xspecial[0, n_own)) plus the rows only the cross rule makes special.
template <bool F64>
__global__ void finalize_cross_kernel(const double* __restrict__ mag, const float* __restrict__ snorm, uint64_t n,
                                      uint64_t n_pad, int metric, float* __restrict__ xnorm,
                                      uint32_t* __restrict__ xspecial, uint32_t* xcnt) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_pad) return;
  float xn = __int_as_float(0x7fc00000);
  if (r < n && snorm[r] == snorm[r]) {
    const double m = mag[r];
    bool special;
    if (metric == SDB_COSINE) {
      const double s = __dmul_rn(m, m);
      xn = (float)s;
      special = !isfinite(s) || !isfinite(xn);
    } else {
      special = !(m > 0.0) || !isfinite(m);
      xn = (float)(1.0 / m);
    }
    if (F64) {
      const float mf = (float)m;
      const bool m_normal = mf >= 1.17549435e-38f && mf <= 3.40282347e38f;
      const bool xn_normal = fabsf(xn) >= 1.17549435e-38f && fabsf(xn) <= 3.40282347e38f;
      if (m > 0.0 && (m < 0x1p-100 || !m_normal || !xn_normal)) special = true;
    }
    if (special) {
      xn = __int_as_float(0x7fc00000);
      const uint32_t pos = atomicAdd(xcnt, 1u);
      if (pos < (uint32_t)SPECIAL_CAP) xspecial[pos] = (uint32_t)r;
    }
  }
  xnorm[r] = xn;
}

// tombstones (sdb_corpus_remove): the row is skipped by every path from now on -- skip mask for the exact kernel, NaN
// screening norms (own and cross) for the screens and the re-rank's special lists, and an all-zero int8 row so that the integer screen
// scores it exactly 0 (the only score for which that screen looks up a row's validity).  No re-finalize needed.
__global__ void or_mask_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint64_t n) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && src[i]) dst[i] = 1;
}
sdb_status corpus_reapply_tombstones(Corpus* c, cudaStream_t st) {  // after the caller replaced the skip mask
  if (!c->d_removed || !c->n) return SDB_OK;
  if (!c->d_skip) {
    SDB_CUDA(c->d_skip.reserve(c->cap));
    SDB_CUDA(cudaMemsetAsync(c->d_skip, 0, c->cap, st));
  }
  or_mask_kernel<<<(unsigned)((c->n + 255) / 256), 256, 0, st>>>(c->d_skip, c->d_removed, c->n);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}
__global__ void remove_rows_kernel(const uint64_t* __restrict__ ids, uint64_t n, uint8_t* __restrict__ skip,
                                   uint8_t* __restrict__ removed, float* __restrict__ snorm, float* __restrict__ xnorm,
                                   int8_t* __restrict__ i8, uint32_t dim_pad8) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= n) return;
  const uint64_t r = ids[w];
  if (lane == 0) {
    skip[r] = 1;
    removed[r] = 1;
    if (snorm) snorm[r] = __int_as_float(0x7fc00000);
    if (xnorm) xnorm[r] = __int_as_float(0x7fc00000);
  }
  if (i8)
    for (uint32_t c = lane; c < dim_pad8; c += 32) i8[r * dim_pad8 + c] = 0;
}
sdb_status corpus_remove_device(Corpus* c, const uint64_t* h_ids, uint64_t n) {
  Ctx* ctx = c->ctx;
  cudaStream_t st = ctx->stream;
  if (!c->d_skip) {
    SDB_CUDA(c->d_skip.reserve(c->cap));
    SDB_CUDA(cudaMemsetAsync(c->d_skip, 0, c->cap, st));
  }
  if (!c->d_removed) {
    SDB_CUDA(c->d_removed.reserve(c->cap));
    SDB_CUDA(cudaMemsetAsync(c->d_removed, 0, c->cap, st));
  }
  AsyncBuf<uint64_t> d_ids;
  SDB_CUDA(d_ids.reserve(n, st));
  SDB_CUDA(cudaMemcpyAsync(d_ids, h_ids, sizeof(uint64_t) * n, cudaMemcpyHostToDevice, st));
  remove_rows_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(
      d_ids, n, c->d_skip, c->d_removed, c->finalized ? c->d_snorm.get() : nullptr,
      c->finalized && c->d_xnorm ? c->d_xnorm.get() : nullptr, c->finalized ? c->d_i8.get() : nullptr, c->dim_pad8);
  count_launch(ctx);
  d_ids.reset();
  std::vector<uint64_t> sorted(h_ids, h_ids + n);
  std::sort(sorted.begin(), sorted.end());
  // a removed special row leaves the always-exact lists (own and cross)
  auto compact = [&](DevBuf<uint32_t>& d_list, uint32_t& n_list) -> sdb_status {
    if (!c->finalized || !n_list) return SDB_OK;
    std::vector<uint32_t> sp(n_list);
    SDB_CUDA(cudaMemcpyAsync(sp.data(), d_list, sizeof(uint32_t) * n_list, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    std::vector<uint32_t> keep;
    for (uint32_t r : sp)
      if (!std::binary_search(sorted.begin(), sorted.end(), (uint64_t)r)) keep.push_back(r);
    if (keep.size() != sp.size()) {
      if (!keep.empty())
        SDB_CUDA(cudaMemcpyAsync(d_list, keep.data(), sizeof(uint32_t) * keep.size(), cudaMemcpyHostToDevice, st));
      SDB_CUDA(cudaStreamSynchronize(st));  // `keep` lives in this frame
      n_list = (uint32_t)keep.size();
    }
    return SDB_OK;
  };
  SDB_TRY(compact(c->d_special, c->n_special));
  if (c->d_xnorm) SDB_TRY(compact(c->d_xspecial, c->n_xspecial));
  SDB_CUDA(cudaStreamSynchronize(st));
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

sdb_status corpus_finalize_device(Corpus* c) {
  Ctx* ctx = c->ctx;
  cudaStream_t st = ctx->stream;
  DevBuf<uint32_t> d_tmp;  // [0] special count, [1] max-norm bits, [2] max relative int8 error bits, [3] int8 gmax
  SDB_CUDA(d_tmp.reserve(8));                                            // [4] max relative bf16 residual bits
  SDB_CUDA(cudaMemsetAsync(d_tmp, 0, 32, st));
  SDB_CUDA(c->d_special.reserve(SPECIAL_CAP));
  {
    const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
    if (n_pad > c->n) {
      pad_snorm_kernel<<<(unsigned)((n_pad - c->n + 255) / 256), 256, 0, st>>>(c->d_snorm, c->n, n_pad);
      count_launch(ctx);
    }
  }
  // Centred corpora (PEARSON with their screen copies, sdb_corpus_create): moments, centred copies; without them the
  // exact kernel serves every query and the corpus is finalized as before
  const bool centred = family(c) == Family::Centred;
  if (c->n) {
    const int grid = ctx->sm_count * 8;
    if (centred) {
      if (c->dtype == SDB_F32)
        finalize_pearson_kernel<float, 8><<<grid, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n, c->d_skip,
                                                                c->d_mag, c->d_mom, c->d_snorm, c->d_special, d_tmp);
      else
        finalize_pearson_kernel<double, 4><<<grid * 2, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n,
                                                                     c->d_skip, c->d_mag, c->d_mom, c->d_snorm,
                                                                     c->d_special, d_tmp);
    } else if (c->metric == SDB_MANHATTAN || c->metric == SDB_CHEBYSHEV || c->metric == SDB_MINKOWSKI) {
      // (MINKOWSKI of every order, not only Family::Lp: the order may change after finalize)
      if (c->dtype == SDB_F32)
        finalize_lp_kernel<float, 8><<<grid, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n, (int)c->metric,
                                                           c->d_skip, c->d_mag, c->d_snorm, c->d_special, d_tmp,
                                                           d_tmp + 1);
      else
        finalize_lp_kernel<double, 4><<<grid * 2, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n,
                                                                (int)c->metric, c->d_skip, c->d_mag, c->d_snorm,
                                                                c->d_special, d_tmp, d_tmp + 1);
    } else if (c->dtype == SDB_F32)
      finalize_rows_kernel<float, 8><<<grid, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n, (int)c->metric,
                                                        c->d_skip, c->d_mag, c->d_snorm, c->d_special, d_tmp,
                                                        d_tmp + 1);
    else
      finalize_rows_kernel<double, 4><<<grid * 2, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n, (int)c->metric,
                                                         c->d_skip, c->d_mag, c->d_snorm, c->d_special, d_tmp,
                                                         d_tmp + 1);
    count_launch(ctx);
    SDB_CUDA(cudaGetLastError());
    if (c->d_bf16) {
      const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
      const double* mom = (const double*)c->d_mom.get();
      if (centred && c->dtype == SDB_F32)
        to_bf16_kernel<float, true><<<ctx->sm_count * 16, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->dim_pad,
                                                                        c->n, n_pad, mom, c->d_snorm, c->d_bf16, d_tmp + 4);
      else if (centred)
        to_bf16_kernel<double, true><<<ctx->sm_count * 16, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim,
                                                                         c->dim_pad, c->n, n_pad, mom, c->d_snorm,
                                                                         c->d_bf16, d_tmp + 4);
      else if (c->dtype == SDB_F32)
        to_bf16_kernel<float><<<ctx->sm_count * 16, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->dim_pad, c->n,
                                                                  n_pad, c->d_mag, c->d_snorm, c->d_bf16, d_tmp + 4);
      else
        to_bf16_kernel<double><<<ctx->sm_count * 16, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->dim_pad,
                                                                   c->n, n_pad, c->d_mag, c->d_snorm, c->d_bf16, d_tmp + 4);
      count_launch(ctx);
      SDB_CUDA(cudaGetLastError());
    }
  }
  if (c->n && c->d_jfirst) {  // JACCARD corpora that hold their first-occurrence state
    if (c->dtype == SDB_F32)
      finalize_jaccard_kernel<float><<<ctx->sm_count * 8, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n,
                                                                       c->d_jfirst, c->d_jux);
    else
      finalize_jaccard_kernel<double><<<ctx->sm_count * 8, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n,
                                                                        c->d_jfirst, c->d_jux);
    count_launch(ctx);
    SDB_CUDA(cudaGetLastError());
  }
  c->n_outliers = 0;
  if (c->n && c->d_i8 && (c->metric == SDB_COSINE || centred)) {
    const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
    const double* mom = (const double*)c->d_mom.get();
    AsyncBuf<float> d_rmax;
    AsyncBuf<uint32_t> d_hist;
    SDB_CUDA(d_rmax.reserve(c->n, st));
    SDB_CUDA(d_hist.reserve(RMAX_BINS, st));
    SDB_CUDA(cudaMemsetAsync(d_hist, 0, sizeof(uint32_t) * RMAX_BINS, st));
    if (centred && c->dtype == SDB_F32)
      quantize_scan_kernel<float, true><<<ctx->sm_count * 8, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n,
                                                                           mom, c->d_snorm, d_tmp + 3, d_rmax, d_hist);
    else if (centred)
      quantize_scan_kernel<double, true><<<ctx->sm_count * 8, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n,
                                                                            mom, c->d_snorm, d_tmp + 3, d_rmax, d_hist);
    else if (c->dtype == SDB_F32)
      quantize_scan_kernel<float><<<ctx->sm_count * 8, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n, c->d_mag,
                                                                     c->d_snorm, d_tmp + 3, d_rmax, d_hist);
    else
      quantize_scan_kernel<double><<<ctx->sm_count * 8, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n, c->d_mag,
                                                                      c->d_snorm, d_tmp + 3, d_rmax, d_hist);
    count_launch(ctx);
    // ---- pick the scale: if at most 64 rows sit far above the rest (their largest normalised component is more
    //      than 1.5 x that of the 65th), make THEM special rows and quantise for the others ----
    std::vector<uint32_t> h_hist(RMAX_BINS);
    uint32_t h4[4] = {0, 0, 0, 0};
    SDB_CUDA(cudaMemcpyAsync(h_hist.data(), d_hist, sizeof(uint32_t) * RMAX_BINS, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaMemcpyAsync(h4, d_tmp, 16, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    float gmax;
    memcpy(&gmax, &h4[3], 4);
    if (gmax > 0.f && !getenv("SDB_NO_OUTLIER_ROWS")) {
      // walk the occupied bins from the top while at most 64 rows lie above; an outlier group ends at a GAP: the next
      // occupied bin below starts at less than 2/3 of the group's lowest bin.  The lowest such gap wins (largest
      // group of rows that are all clearly detached from the bulk); without a gap nothing is special.
      uint32_t cum = 0;
      int cut = -1, below = -1;
      int last = -1;  // lowest occupied bin seen so far
      for (int b = (int)RMAX_BINS - 1; b >= 0; b--) {
        if (!h_hist[b]) continue;
        if (last >= 0 && cum <= 64u) {
          // edges: bin x covers [edge(x), edge(x+1)); gap test between the top of bin b and the bottom of bin `last`
          uint32_t ul = (uint32_t)last << 19, ub = (uint32_t)(b + 1) << 19;
          float lo_last, hi_b;
          memcpy(&lo_last, &ul, 4);
          memcpy(&hi_b, &ub, 4);
          if (lo_last > 1.5f * hi_b) {
            cut = last;
            below = b;
          }
        }
        cum += h_hist[b];
        if (cum > 64u) break;
        last = b;
      }
      if (cut >= 0) {
        uint32_t n_out = 0;
        for (int b = cut; b < (int)RMAX_BINS; b++) n_out += h_hist[b];
        if (n_out > 0 && h4[0] + n_out <= (uint32_t)SPECIAL_CAP) {
          const uint32_t ut = (uint32_t)cut << 19, us = (uint32_t)(below + 1) << 19;
          float thr, new_gmax;
          memcpy(&thr, &ut, 4);        // rows with rmax >= thr are the outliers
          memcpy(&new_gmax, &us, 4);   // every remaining row has rmax < this: the scale of the int8 copy
          mark_outliers_kernel<<<(unsigned)((c->n + 255) / 256), 256, 0, st>>>(d_rmax, c->n, thr, c->d_snorm, c->d_special, d_tmp);
          count_launch(ctx);
          SDB_CUDA(cudaMemcpyAsync(d_tmp + 3, &new_gmax, 4, cudaMemcpyHostToDevice, st));
          SDB_CUDA(cudaStreamSynchronize(st));  // `new_gmax` lives on this stack frame
          c->n_outliers = n_out;
        }
      }
    }
    if (centred && c->dtype == SDB_F32)
      quantize_rows_kernel<float, true><<<ctx->sm_count * 8, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim,
                                                                           c->dim_pad8, c->n, n_pad, mom, c->d_snorm,
                                                                           d_tmp + 3, c->d_i8, d_tmp + 2);
    else if (centred)
      quantize_rows_kernel<double, true><<<ctx->sm_count * 8, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim,
                                                                            c->dim_pad8, c->n, n_pad, mom, c->d_snorm,
                                                                            d_tmp + 3, c->d_i8, d_tmp + 2);
    else if (c->dtype == SDB_F32)
      quantize_rows_kernel<float><<<ctx->sm_count * 8, 256, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->dim_pad8, c->n,
                                                                     n_pad, c->d_mag, c->d_snorm, d_tmp + 3, c->d_i8, d_tmp + 2);
    else
      quantize_rows_kernel<double><<<ctx->sm_count * 8, 256, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->dim_pad8,
                                                                      c->n, n_pad, c->d_mag, c->d_snorm, d_tmp + 3, c->d_i8,
                                                                      d_tmp + 2);
    count_launch(ctx);
    SDB_CUDA(cudaGetLastError());
  }
  uint32_t h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  SDB_CUDA(cudaMemcpyAsync(h, d_tmp, 32, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  // no special rows: zero, NaN and +-inf are ordinary values for equality (a fact of the metric, whatever the family)
  if (c->metric == SDB_HAMMING || c->metric == SDB_JACCARD) h[0] = 0;
  c->special_overflow = h[0] > (uint32_t)SPECIAL_CAP;
  c->n_special = h[0] > (uint32_t)SPECIAL_CAP ? (uint32_t)SPECIAL_CAP : h[0];
  float mn;
  memcpy(&mn, &h[1], 4);
  c->max_norm = mn;
  memcpy(&c->max_rel_qerr, &h[2], 4);
  {
    float e;
    memcpy(&e, &h[4], 4);
    // never trust a figure above the analytic worst case of round-to-nearest (2^-8 per element => 2^-8 in norm)
    c->bf16_rel_err = (e > 0.f && e < 0.00390625f) ? e : 0.00390625f;
  }
  {
    float gmax;
    memcpy(&gmax, &h[3], 4);
    c->i8_scale = gmax > 0.f ? gmax / 127.f : 1.f;
  }
  // the cross state (cross_ranking): after the own state is final, so that it follows every own NaN norm and special
  // row; the union overflowing SPECIAL_CAP sends the cross views to the exact kernel, and KNN keeps its own state
  c->n_xspecial = 0;
  c->xspecial_overflow = false;
  if (family(c) == Family::Dot && c->d_bf16) {
    const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
    const uint64_t cap_pad = (c->cap + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
    if (c->d_xnorm.reserve(cap_pad) != cudaSuccess || c->d_xspecial.reserve(SPECIAL_CAP) != cudaSuccess) {
      c->d_xnorm.reset();  // no cross state: the cross views take the exact kernel
      c->d_xspecial.reset();
    } else {
      if (c->n_special)
        SDB_CUDA(cudaMemcpyAsync(c->d_xspecial, c->d_special, sizeof(uint32_t) * c->n_special, cudaMemcpyDeviceToDevice, st));
      const uint32_t own = c->special_overflow ? (uint32_t)SPECIAL_CAP + 1u : c->n_special;
      SDB_CUDA(cudaMemcpyAsync(d_tmp, &own, 4, cudaMemcpyHostToDevice, st));
      if (n_pad) {
        auto kern = c->dtype == SDB_F64 ? finalize_cross_kernel<true> : finalize_cross_kernel<false>;
        kern<<<(unsigned)((n_pad + 255) / 256), 256, 0, st>>>(c->d_mag, c->d_snorm, c->n, n_pad, (int)c->metric,
                                                              c->d_xnorm, c->d_xspecial, d_tmp);
        count_launch(ctx);
        SDB_CUDA(cudaGetLastError());
      }
      uint32_t nx = 0;
      SDB_CUDA(cudaMemcpyAsync(&nx, d_tmp, 4, cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaStreamSynchronize(st));  // (`own` and `nx` live in this frame)
      c->xspecial_overflow = nx > (uint32_t)SPECIAL_CAP;
      c->n_xspecial = nx > (uint32_t)SPECIAL_CAP ? (uint32_t)SPECIAL_CAP : nx;
    }
  }
  c->finalized = true;
  return SDB_OK;
}

}  // namespace sdb
