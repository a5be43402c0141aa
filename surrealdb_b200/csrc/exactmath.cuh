// exactmath.cuh -- the reference's f64 arithmetic, op for op, with explicit round-to-nearest
// intrinsics so nvcc can never contract a*b+c into an FMA (Rust/LLVM does not fuse either).
// RefAcc<M> below holds each metric's whole definition, cited there; every kernel that ends in the reference's value
// (exact.cu's exact kernel, candidates.cu's re-ranks) takes its steps and finish from it.
// NaN sign convention = x86-64 hardware (where the reference runs): a GENERATED NaN (0/0, inf-inf,
// inf*0) is the negative "real indefinite" 0xFFF8000000000000 and therefore sorts FIRST under
// Number::cmp's total_cmp; a NaN that came in through the data (Rust f64::NAN, positive) propagates
// as a positive NaN and sorts LAST.  Mixed cases are unpinned (DESIGN.md section 3).
#pragma once
#include <cstdint>
#include <type_traits>

#include "../../include/sdbgpu.h"

namespace sdb {

// Number equality of two elements after the widening to f64 (val/number.rs PartialEq): the same bits, or both zero, so
// 0.0 == -0.0 and NaN == NaN exactly when the bits agree.  HAMMING and JACCARD count with it everywhere.
__device__ __forceinline__ bool num_eq_f64(double a, double b) {
  return __double_as_longlong(a) == __double_as_longlong(b) || (a == 0.0 && b == 0.0);
}
// Keys that turn num_eq_f64 into one integer compare (the HAMMING count kernel, count.cu).
//  - f64 rows and queries: the bits, -0.0 folded onto 0.0.
//  - f32 rows: the key of (double)x, the exact kernel's widening, in 32 bits: x's own bits for a number (the widening
//    is exact; -0.0 folded onto 0.0), sign | 0x7f800000 | fraction bits 51..29 of the widened value for a NaN, so that
//    two NaNs get one key exactly when the device widens them to the same bits.
//  - an f64 query element against f32 rows: the key of the f32 that widens to it bit for bit, or EQ_KEY_NONE when no
//    f32 does; EQ_KEY_NONE is -0.0's pattern, which no row key takes.
constexpr uint32_t EQ_KEY_NONE = 0x80000000u;
__device__ __forceinline__ unsigned long long eq_key_f64(double x) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(x);
  return (b << 1) == 0 ? 0ull : b;
}
__device__ __forceinline__ uint32_t eq_key_f32(float x) {
  const double w = (double)x;
  const unsigned long long b = (unsigned long long)__double_as_longlong(w);
  if ((b << 1) == 0) return 0u;
  if (w != w) return ((uint32_t)(b >> 32) & 0x80000000u) | 0x7f800000u | ((uint32_t)(b >> 29) & 0x7fffffu);
  return __float_as_uint(x);
}
__device__ __forceinline__ uint32_t eq_qkey_f32(double q) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(q);
  if ((b << 1) == 0) return 0u;
  // the only f32 that can widen to q: q rounded for a number, q's sign and top fraction bits for a NaN
  const uint32_t fb = q != q ? ((uint32_t)(b >> 32) & 0x80000000u) | 0x7f800000u | ((uint32_t)(b >> 29) & 0x7fffffu)
                             : __float_as_uint(__double2float_rn(q));
  const float f = __uint_as_float(fb);
  if ((unsigned long long)__double_as_longlong((double)f) != b) return EQ_KEY_NONE;
  return eq_key_f32(f);
}

template <typename T>
using EqKey = typename std::conditional<sizeof(T) == 8, unsigned long long, uint32_t>::type;
__device__ __forceinline__ uint32_t eq_key_row(float x) { return eq_key_f32(x); }
__device__ __forceinline__ unsigned long long eq_key_row(double x) { return eq_key_f64(x); }

// JACCARD (vector.rs:121-127 with v1 = the row, v2 = the query) from counts, as jaccard_keys_kernel computes it:
// u_x / u_q = distinct values of the row / the query, m = values both share; inter = D - u_q + m,
// union = u_x + u_q - m, result inter / union in one f64 division.  first: the row's first-occurrence bitmask (bit i
// set when x_i is the first element of its value; popcount = u_x, finalize_jaccard_kernel); qk: the query's distinct
// keys that some row element can have, sorted ascending (n_look of them).  m = first-occurrence elements of the row
// whose key is among them: O(u_x log u_q) per pair.
template <typename T>
__device__ __forceinline__ double jaccard_counts(const T* __restrict__ x, uint32_t dim, const uint32_t* __restrict__ first,
                                                 uint32_t ux, const EqKey<T>* __restrict__ qk, uint32_t n_look,
                                                 uint32_t uq) {
  uint32_t m = 0;
  for (uint32_t w = 0; w * 32 < dim; w++) {
    uint32_t b = __ldg(first + w);
    while (b) {
      const uint32_t i = w * 32 + (uint32_t)(__ffs(b) - 1);
      b &= b - 1;
      const EqKey<T> key = eq_key_row(__ldg(x + i));
      uint32_t lo = 0, hi = n_look;
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(qk + mid) < key) lo = mid + 1;
        else hi = mid;
      }
      m += (lo < n_look && __ldg(qk + lo) == key) ? 1u : 0u;
    }
  }
  return __ddiv_rn((double)(dim - uq + m), (double)(ux + uq - m));
}

// ---- the reference's per-metric arithmetic --------------------------------------------------------------------------
// RefSum is one row's running state; RefAcc<M> is metric M with its parameters (MINKOWSKI's order, PEARSON's means):
// its start value, step(s, x, q) over the elements x of the row and q of the query, left to right, and finish(s, ...),
// which carries the metric's whole rule for the result.  M is a metric id or one of the projections SDB_FN_*.
struct RefSum {
  double acc = 0.0;
  double acc2 = 0.0;    // PEARSON's exact-kernel pass B: sum (x - m1)^2
  bool nan_in = false;  // a NaN element of the row came in
};

// NaN sign rule (header comment): a NaN result is positive when a NaN came in through the data (the row's elements,
// nan_in, or the query's, q_nan), else the negative generated NaN
__device__ __forceinline__ double canon_nan(double r, bool nan_in) {
  if (r != r) return __longlong_as_double(nan_in ? 0x7FF8000000000000ll : (long long)0xFFF8000000000000ull);
  return r;
}

template <int M>
struct RefAcc;

//   cosine: 1 - similarity, vector.rs:65-71 with dot vector.rs:279-281 and the row's magnitude (vector.rs:301-314) from
//           finalize
template <>
struct RefAcc<SDB_COSINE> {
  static constexpr double start = 0.0;
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const {
    s.nan_in |= (x != x);
    s.acc = __dadd_rn(s.acc, __dmul_rn(x, q));
  }
  __device__ __forceinline__ double finish(const RefSum& s, double row_mag, double q_mag, bool q_nan) const {
    return canon_nan(__dsub_rn(1.0, __ddiv_rn(s.acc, __dmul_rn(row_mag, q_mag))), s.nan_in || q_nan);
  }
};
//   similarity::cosine: vector.rs:65-71
template <>
struct RefAcc<SDB_FN_SIMILARITY_COSINE> : RefAcc<SDB_COSINE> {
  __device__ __forceinline__ double finish(const RefSum& s, double row_mag, double q_mag, bool q_nan) const {
    return canon_nan(__ddiv_rn(s.acc, __dmul_rn(row_mag, q_mag)), s.nan_in || q_nan);
  }
};
//   dot: vector.rs:279-281
template <>
struct RefAcc<SDB_FN_DOT> : RefAcc<SDB_COSINE> {
  __device__ __forceinline__ double finish(const RefSum& s, bool q_nan) const { return canon_nan(s.acc, s.nan_in || q_nan); }
};
//   magnitude: vector.rs:301-314, computed at finalize; no steps
template <>
struct RefAcc<SDB_FN_MAGNITUDE> {
  __device__ __forceinline__ double finish(double row_mag) const { return row_mag; }
};
//   euclidean: vector.rs:288-299   sqrt(sum (x - q)^2)
template <>
struct RefAcc<SDB_EUCLIDEAN> {
  static constexpr double start = 0.0;
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const {
    s.nan_in |= (x != x);
    const double d = __dsub_rn(x, q);
    s.acc = __dadd_rn(s.acc, __dmul_rn(d, d));
  }
  __device__ __forceinline__ double finish(const RefSum& s, bool q_nan) const {
    return canon_nan(__dsqrt_rn(s.acc), s.nan_in || q_nan);
  }
};
//   manhattan: vector.rs:152-157   acc = acc + |x - q|        (Number add, Int(0) start == 0.0 + ...)
template <>
struct RefAcc<SDB_MANHATTAN> {
  static constexpr double start = 0.0;
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const {
    s.nan_in |= (x != x);
    s.acc = __dadd_rn(s.acc, fabs(__dsub_rn(x, q)));
  }
  __device__ __forceinline__ double finish(const RefSum& s, bool q_nan) const { return canon_nan(s.acc, s.nan_in || q_nan); }
};
//   chebyshev: vector.rs:215-225   fold(f64::MIN, f64::max)  -- f64::max returns the non-NaN operand, as fmax does, so
//              the result is never NaN and needs no NaN rule
template <>
struct RefAcc<SDB_CHEBYSHEV> {
  static constexpr double start = -1.7976931348623157e308;  // f64::MIN
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const { s.acc = fmax(s.acc, fabs(__dsub_rn(x, q))); }
  __device__ __forceinline__ double finish(const RefSum& s, bool) const { return s.acc; }
};
//   hamming  : vector.rs:111-116   count of a != b under Number's PartialEq (0.0 == -0.0, NaN == NaN bitwise)
template <>
struct RefAcc<SDB_HAMMING> {
  static constexpr double start = 0.0;
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const {
    s.acc = __dadd_rn(s.acc, num_eq_f64(x, q) ? 0.0 : 1.0);  // exact: an integer count below 2^53
  }
  __device__ __forceinline__ double finish(const RefSum& s, bool) const { return s.acc; }
};
//   minkowski: vector.rs:163-174   acc = acc + |x - q|^p ; finish: acc^(1/p).  pow() is CUDA's libm here and the
//              platform libm in the reference: each call agrees to within an ulp or two, not bit for bit.
template <>
struct RefAcc<SDB_MINKOWSKI> {
  static constexpr double start = 0.0;
  double p;
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const {
    s.nan_in |= (x != x);
    s.acc = __dadd_rn(s.acc, pow(fabs(__dsub_rn(x, q)), p));
  }
  __device__ __forceinline__ double finish(const RefSum& s, bool q_nan) const {
    return canon_nan(pow(s.acc, __ddiv_rn(1.0, p)), s.nan_in || q_nan);
  }
};
//   pearson  : vector.rs:133-146   covar / (sd1 * sd2), covar = sum (x - m1)(q - m2) / len, sd = deviation(sample =
//              false) (vector.rs:9-21), each mean sequential (fnc/util/math/mod.rs:54-69).  The exact kernel runs two
//              passes (mean_step, then step_dev from the row's mean); the re-rank runs step from the stored means.
template <>
struct RefAcc<SDB_PEARSON> {
  static constexpr double start = 0.0;
  double m1, m2;  // the row's and the query's mean
  // pass A: sum x
  __device__ __forceinline__ static void mean_step(RefSum& s, double x) {
    s.nan_in |= (x != x);
    s.acc = __dadd_rn(s.acc, x);
  }
  // pass B: covar and the row's deviation sum (pass A saw the row's NaN)
  __device__ __forceinline__ void step_dev(RefSum& s, double x, double q) const {
    const double dx = __dsub_rn(x, m1);
    s.acc = __dadd_rn(s.acc, __dmul_rn(dx, __dsub_rn(q, m2)));
    s.acc2 = __dadd_rn(s.acc2, __dmul_rn(dx, dx));
  }
  // one pass from the stored means: covar, and the row's NaN as pass A sees it
  __device__ __forceinline__ void step(RefSum& s, double x, double q) const {
    s.nan_in |= (x != x);
    step_dev(s, x, q);
  }
  // the deviation from S = sum (x_i - m)^2: 0 when dim == 1 (the reference's deviation of one element)
  __device__ __forceinline__ static double sd(double S, uint32_t dim) {
    return dim == 1 ? 0.0 : __dsqrt_rn(__ddiv_rn(S, (double)dim));
  }
  // a row whose mean is a generated NaN (+inf and -inf) and no NaN element sorts first
  __device__ __forceinline__ static double finish(const RefSum& s, uint32_t dim, double sd1, double sd2, bool q_nan) {
    const double covar = __ddiv_rn(s.acc, (double)dim);
    return canon_nan(__ddiv_rn(covar, __dmul_rn(sd1, sd2)), s.nan_in || q_nan);
  }
};
// (m, S) of a contiguous vector in the sequential arithmetic above: m = (sum v) / dim, S = sum (v_i - m)^2
__device__ __forceinline__ double2 pearson_moments(const double* v, uint32_t dim) {
  double s = 0.0;
  for (uint32_t i = 0; i < dim; i++) s = __dadd_rn(s, v[i]);
  const double m = __ddiv_rn(s, (double)dim);
  double S = 0.0;
  for (uint32_t i = 0; i < dim; i++) {
    const double d = __dsub_rn(v[i], m);
    S = __dadd_rn(S, __dmul_rn(d, d));
  }
  return make_double2(m, S);
}

}  // namespace sdb
