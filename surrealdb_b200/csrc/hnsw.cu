// hnsw.cu -- K3: HNSW layer walk, one warp per query, strict-parity with the reference's sequential search.
//
// Replaces Hnsw::knn_search (idx/trees/hnsw/mod.rs:459-482): search_ep greedy descent (mod.rs:521-548) and
// HnswLayer::search (hnsw/layer.rs:184-223) with its two DoublePriorityQueues (idx/trees/knn.rs:15-123) and
// visited set.  Parity rules reproduced exactly:
//   * candidates popped nearest-first, FIFO among equal distances; stop when nearest candidate > farthest kept
//   * neighbours visited in STORED order; admitted iff d < f or |w| < ef; w trimmed with pop_last (newest of
//     the farthest); f re-read after every admission
//   * distances are the typed-f32 kernels of idx/trees/vector.rs:243-289: cosine = ndarray 8-lane f32 dot and
//     sums, finished in f64; euclid = sequential f32 sum of squares, f64 sqrt (same op order as the oracle)
// Batched candidate expansion: the <=32 neighbours of the popped candidate are de-duplicated against the
// per-query visited table with warp-parallel CAS, their vectors are gathered with coalesced transposed loads
// (one lane per neighbour walks its row in order), and only the admission step is serial.
// Queue trick (result-neutral): once w is full, candidates farther than f can never be expanded (f only
// shrinks), so they are dropped from the candidate array, which bounds it to 2*ef entries.
//
// Algorithmic bytes per query = visited * (4*dim + 4) + expanded * 4*deg, both counters are returned.
#include <algorithm>
#include <type_traits>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "internal.cuh"
#include "rowwalk.cuh"

namespace sdb {

// Per-vector state of the metrics that carry it (vec_state_make); null where the metric needs none.  K fixes how it is
// allocated: an index's elements in device memory (Mem::Device), freed with the index; the queries or pending vectors of
// one call from the stream's pool (Mem::Async), freed on the stream once the call's kernels are queued.
template <Mem K>
struct VecState {
  Buf<double, K> norm;      // COSINE: the vector's factor of the denominator: sqrt((double)sumsq) (F32, vector.rs:246),
                            // sqrt of the 8-lane f64 sum of f64(x)^2 (the other types, vector.rs:238,257)
  Buf<double, K> mean;      // PEARSON: mean (in the type's arithmetic, widened) and sum of squared deviations
  Buf<double, K> sx2;       // (vector.rs:412-451)
  Buf<char, K> bits;        // JACCARD: sorted distinct keys (JKey, dim-strided rows) ...
  Buf<uint32_t, K> nbits;   // ... and how many there are (vector.rs:316-356)
};

constexpr int HN_WARPS = 4;

// The queues' order (FloatKey, idx/trees/knn.rs:129-160): f64::total_cmp, so -0.0 sorts before 0.0.  Unlike the
// brute-force path's dist_key (Number::cmp, where -0.0 equals 0.0) this key is one-to-one, and key_to_double gives back
// the distance itself, sign of zero included.
__device__ __forceinline__ uint64_t walk_key(double d) {
  const uint64_t b = f64_bits(d);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
// the key with -0.0 and 0.0 made equal, where the reference compares the two distances as f64
__device__ __forceinline__ uint64_t zero_tie(uint64_t key) {
  return key == 0x7fffffffffffffffull ? 0x8000000000000000ull : key;  // walk_key(-0.0) -> walk_key(0.0)
}
__device__ __forceinline__ double key_to_double(uint64_t key) {
  const uint64_t b = (key >> 63) ? (key & 0x7fffffffffffffffull) : ~key;
  return __longlong_as_double((long long)b);
}

// ---- element types (sdb_vector_type -> T): F64 double, F32 float, I64 long long, I32 int, I16 short
template <typename T> constexpr bool is_f32_v = std::is_same<T, float>::value;
template <typename T> constexpr bool is_f64_v = std::is_same<T, double>::value;
template <typename T> constexpr bool is_i16_v = std::is_same<T, short>::value;
template <typename T> constexpr bool is_wint_v = std::is_same<T, long long>::value || std::is_same<T, int>::value;  // I64, I32
// JACCARD key of an element: its bit pattern (F32, F64, vector.rs:316-340) or its value (integers, :342-356); u64 for the
// 8-byte types, u32 for the others
template <typename T> using JKey = typename std::conditional<sizeof(T) == 8, unsigned long long, uint32_t>::type;
// Wrapping integer arithmetic in T (the reference is a release build without overflow checks, so `+ - * abs` wrap):
// computed in an unsigned type of at least 32 bits, truncated to T.
template <typename T> using Wide = typename std::conditional<sizeof(T) == 8, unsigned long long, uint32_t>::type;
template <typename T> __device__ __forceinline__ Wide<T> wide(T v) { return (Wide<T>)(typename std::make_unsigned<T>::type)v; }
template <typename T> __device__ __forceinline__ T wrap(Wide<T> v) { return (T)(typename std::make_unsigned<T>::type)v; }
template <typename T> __device__ __forceinline__ T wsub(T a, T b) { return wrap<T>(wide(a) - wide(b)); }
template <typename T> __device__ __forceinline__ T wabs(T a) { return a < 0 ? wrap<T>(Wide<T>(0) - wide(a)) : a; }  // abs(MIN) = MIN
// The float type the reference's float arithmetic runs in for T: f32 for F32, f64 for every other type
template <typename T> using Real = typename std::conditional<is_f32_v<T>, float, double>::type;
// IEEE round-to-nearest + - * in f32 or f64 (never contracted into an FMA, as in the reference)
__device__ __forceinline__ float rn_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double rn_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float rn_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double rn_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float rn_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double rn_mul(double a, double b) { return __dmul_rn(a, b); }

// ndarray's fold of 8 partial sums p_j (p_j = the sequential chain over the columns 8i+j of unrolled_fold / unrolled_dot):
// ((((0+(p0+p4))+(p1+p5))+(p2+p6))+(p3+p7)).  S = float (F32) or double.
template <typename S>
__device__ __forceinline__ S fold8(const S p[8]) {
  S s = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) s = rn_add(s, rn_add(p[j], p[j + 4]));
  return s;
}
// The same fold when the 8 chains of a row live on 8 consecutive lanes (lane 8g+j holds p_j): the result is on lane 8g.
// All 32 lanes must call; only the lanes with `take` add up (the others return 0).
__device__ __forceinline__ float quad_fold8(float p, bool take) {
  const float sj = __fadd_rn(p, __shfl_down_sync(0xffffffffu, p, 4));
  const float s1 = __shfl_down_sync(0xffffffffu, sj, 1);
  const float s2 = __shfl_down_sync(0xffffffffu, sj, 2);
  const float s3 = __shfl_down_sync(0xffffffffu, sj, 3);
  float s = 0.f;
  if (take) {
    s = __fadd_rn(0.f, sj);
    s = __fadd_rn(s, s1);
    s = __fadd_rn(s, s2);
    s = __fadd_rn(s, s3);
  }
  return s;
}
// ndarray's 8-lane sum of a row in S (unrolled_fold: fold8 of the 8 chains, then the < 8 tail columns in order) of S(x)^2
// (SQ) or of S(x).  S = float: F32's sums (tests/hnsw_metric_ref.py nd_sum_f32); S = double: the f64 sums of the other
// types (tests/hnsw_types_ref.py nd_sum_f64), the cosine norms (vector.rs:238,257) and the F64 mean.  One thread per row.
template <typename S, bool SQ, typename T>
__device__ __forceinline__ S nd_sum(const T* a, uint32_t dim) {
  S p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  uint32_t i = 0;
  for (; i + 8 <= dim; i += 8)
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const S v = (S)a[i + j];
      p[j] = rn_add(p[j], SQ ? rn_mul(v, v) : v);
    }
  S s = fold8(p);
  for (; i < dim; i++) {
    const S v = (S)a[i];
    s = rn_add(s, SQ ? rn_mul(v, v) : v);
  }
  return s;
}

// cosine norms of the types other than F32 (load time, and once per query batch)
template <typename T>
__global__ void hnsw_norm_kernel(const T* __restrict__ vec, uint32_t dim, uint64_t n, double* __restrict__ norm) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) norm[r] = __dsqrt_rn(nd_sum<double, true>(vec + r * dim, dim));
}

// cosine norms of F32 elements (load time): sqrt((double)sumsq), sumsq = ndarray's 8-lane f32 sum of squares
// (vector.rs:246).  8 threads per row, thread j owns the chain over the columns 8i+j; the 8 threads of a row read one
// 32-byte sector per step.
__global__ void hnsw_norm_f32_kernel(const float* __restrict__ vec, uint32_t dim, uint64_t n, double* __restrict__ norm) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t r = t >> 3;
  const uint32_t j = (uint32_t)t & 7u;
  const bool valid = r < n;
  const float* a = vec + (valid ? r : 0) * dim + j;
  const uint32_t steps = dim >> 3;
  float p = 0.f;
  if (valid)
    for (uint32_t i = 0; i < steps; i++) {
      const float v = __ldg(a + 8u * i);
      p = __fadd_rn(p, __fmul_rn(v, v));
    }
  float sum = quad_fold8(p, valid && j == 0);
  if (valid && j == 0) {
    const float* row = vec + r * dim;
    for (uint32_t c = dim & ~7u; c < dim; c++) sum = __fadd_rn(sum, __fmul_rn(__ldg(row + c), __ldg(row + c)));
    norm[r] = __dsqrt_rn((double)sum);
  }
}

// ---- per-vector state of PEARSON and JACCARD (load time for the elements, per batch for queries and pending vectors)

// PEARSON (vector.rs:412-451): mean = ndarray's mean in T, widened to f64 -- F32: nd_sum in f32 divided by n as f32;
// F64: the same in f64; integers: the wrapping sum divided by n in T (truncating toward zero).  sx2 = sequential f64
// sum of (f64(x_i) - mean)^2.  Only the cross term is left per pair.  One thread per vector (load time, and once per
// query batch).
template <typename T>
__global__ void pearson_stats_kernel(const T* __restrict__ vec, uint32_t dim, uint64_t n, double* __restrict__ mean,
                                     double* __restrict__ sx2) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const T* a = vec + r * dim;
  double m;
  if constexpr (is_f32_v<T>) {
    m = (double)__fdiv_rn(nd_sum<float, false>(a, dim), (float)dim);
  } else if constexpr (is_f64_v<T>) {
    m = __ddiv_rn(nd_sum<double, false>(a, dim), (double)dim);
  } else {  // the wrapping sum is the same in any order
    Wide<T> w = 0;
    for (uint32_t c = 0; c < dim; c++) w += wide(a[c]);
    m = (double)(T)(wrap<T>(w) / (T)dim);
  }
  double d2 = 0.0;
  for (uint32_t c = 0; c < dim; c++) {
    const double d = __dsub_rn((double)a[c], m);
    d2 = __dadd_rn(d2, __dmul_rn(d, d));
  }
  mean[r] = m;
  sx2[r] = d2;
}

// JACCARD compares f32 / f64 BIT PATTERNS (vector.rs:316-340) and integer values (:342-356), as JKey<T>.  A vector's
// state is its sorted list of distinct keys: after a segmented sort of each row (one row = one segment), this drops the
// repeats in place and records the count.
template <typename K>
__global__ void distinct_sorted_kernel(K* __restrict__ bits, uint32_t dim, uint64_t n, uint32_t* __restrict__ nbits) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  K* row = bits + r * dim;
  uint32_t u = 1;
  K prev = row[0];
  for (uint32_t i = 1; i < dim; i++) {
    const K v = row[i];
    if (v != prev) row[u++] = v;
    prev = v;
  }
  nbits[r] = u;
}
__global__ void segment_offsets_kernel(int* __restrict__ off, uint32_t rows, uint32_t dim) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= rows) off[i] = (int)(i * dim);
}
// I16: the values widened to u32 keys (any injective map keeps the distinct count and the intersection)
__global__ void widen_keys_kernel(const short* __restrict__ v, uint64_t count, uint32_t* __restrict__ keys) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) keys[i] = (uint32_t)(int)v[i];
}

// rows x dim keys -> per row: sorted distinct keys (bits, rows x dim, caller-allocated) and their count (nbits)
template <typename K>
sdb_status jaccard_prepare(Ctx* ctx, const K* keys, uint64_t rows, uint32_t dim, K* bits, uint32_t* nbits,
                           cudaStream_t st) {
  if (!rows) return SDB_OK;
  const uint64_t chunk = std::max<uint64_t>(1, std::min<uint64_t>(rows, (1u << 30) / dim));  // CUB counts items in int
  AsyncBuf<int> d_off;
  AsyncBuf<char> d_tmp;
  size_t tmp_bytes = 0;
  if (cub::DeviceSegmentedSort::SortKeys(nullptr, tmp_bytes, keys, bits, (int)(chunk * dim), (int)chunk, d_off.get(),
                                         d_off + 1, st) != cudaSuccess)
    return SDB_ECUDA;
  if (d_off.reserve(chunk + 1, st) != cudaSuccess || d_tmp.reserve(tmp_bytes ? tmp_bytes : 1, st) != cudaSuccess) {
    set_error("hnsw jaccard: %zu bytes of sort scratch could not be allocated", tmp_bytes + 4 * (chunk + 1));
    return SDB_ENOMEM;
  }
  sdb_status rc = SDB_OK;
  for (uint64_t r0 = 0; r0 < rows && rc == SDB_OK; r0 += chunk) {
    const uint32_t nr = (uint32_t)std::min<uint64_t>(chunk, rows - r0);
    segment_offsets_kernel<<<(nr + 256) / 256, 256, 0, st>>>(d_off, nr, dim);
    count_launch(ctx);
    size_t b = tmp_bytes;
    if (cub::DeviceSegmentedSort::SortKeys(d_tmp.get(), b, keys + r0 * dim, bits + r0 * dim, (int)(nr * dim), (int)nr,
                                           d_off.get(), d_off + 1, st) != cudaSuccess)
      rc = SDB_ECUDA;
    count_launch(ctx);
  }
  if (rc == SDB_OK) {
    distinct_sorted_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, st>>>(bits, dim, rows, nbits);
    count_launch(ctx);
  }
  if (rc != SDB_OK) set_error("hnsw jaccard: segmented sort failed: %s", cudaGetErrorString(cudaGetLastError()));
  return rc;
}

// rows x dim elements of type vt -> their JACCARD state (bits: rows x dim JKey, caller-allocated)
sdb_status jaccard_prepare_typed(Ctx* ctx, sdb_vector_type vt, const void* d_vec, uint64_t rows, uint32_t dim, void* bits,
                                 uint32_t* nbits, cudaStream_t st) {
  if (vt == SDB_VT_F64 || vt == SDB_VT_I64)
    return jaccard_prepare(ctx, static_cast<const unsigned long long*>(d_vec), rows, dim,
                           static_cast<unsigned long long*>(bits), nbits, st);
  if (vt != SDB_VT_I16)
    return jaccard_prepare(ctx, static_cast<const uint32_t*>(d_vec), rows, dim, static_cast<uint32_t*>(bits), nbits, st);
  if (!rows) return SDB_OK;
  AsyncBuf<uint32_t> keys;
  if (keys.reserve(rows * dim, st) != cudaSuccess) {
    set_error("hnsw jaccard: %llu bytes of key scratch could not be allocated", (unsigned long long)(4 * rows * dim));
    return SDB_ENOMEM;
  }
  widen_keys_kernel<<<(unsigned)((rows * dim + 255) / 256), 256, 0, st>>>(static_cast<const short*>(d_vec), rows * dim, keys);
  count_launch(ctx);
  return jaccard_prepare(ctx, static_cast<const uint32_t*>(keys), rows, dim, static_cast<uint32_t*>(bits), nbits, st);
}

// per-query operands of the metrics that carry state (staged once per query, the same arithmetic as the elements')
struct MetricQ {
  double mean = 0.0, sx2 = 0.0;  // PEARSON: the query's mean and sum of squared deviations
  double p = 3.0;                // MINKOWSKI: the order
  uint32_t u = 0;                // JACCARD: number of distinct bit patterns of the query
};

// Per-column accumulators of the metrics that fold ONE sequential chain per row (ndarray-stats' Zip folds, the explicit
// loops of vector.rs).  step(x, q): x = the element / pending vector, q = the query.  All of them are symmetric in their
// two arguments (|x-q| = |q-x| exactly, products commute), so the walk's calculate(element, query) and the pending log's
// calculate(query, vector) share them.  row_mean / row_sx2: the row's PEARSON state.
// Each metric is in the element type's own arithmetic (vector.rs:206-451).  The integer l1_dist / l2_dist / linf_dist
// are ndarray-stats' DeviationExt (not vendored): they accumulate in T, with wrapping `+ - * abs`, and cast to f64 at
// the end.  to_float() is `as f64` (round to nearest for I64).  A sum that is exact (integers below 2^53) or wraps is
// the same in any order; the others are the reference's sequential folds.
template <int MET, typename T>
struct RowAcc;
// l2_dist: the sum of squares in T (F32: f32, then an f64 sqrt); I16: euclidean(), the f64 sum of exact squares
template <typename T>
struct RowAcc<SDB_EUCLIDEAN, T> {
  typename std::conditional<is_wint_v<T>, Wide<T>, Real<T>>::type s = 0;
  __device__ __forceinline__ RowAcc(const MetricQ&, double, double, uint32_t) {}
  __device__ __forceinline__ void step(T x, T q) {
    if constexpr (is_wint_v<T>) {
      const Wide<T> d = wide(x) - wide(q);
      s += d * d;
    } else {
      const Real<T> d = rn_sub((Real<T>)x, (Real<T>)q);
      s = rn_add(s, rn_mul(d, d));
    }
  }
  __device__ __forceinline__ double finish() const {
    if constexpr (is_wint_v<T>) return __dsqrt_rn((double)wrap<T>(s));
    else return __dsqrt_rn((double)s);
  }
};
// l1_dist (vector.rs:377-386): the sum of |x-q| in T, then as f64 (integers: the wrapping abs of a wrapping difference);
// I16: the f64 sum of |f64(x - q)|, x - q wrapping in i16
template <typename T>
struct RowAcc<SDB_MANHATTAN, T> {
  typename std::conditional<is_wint_v<T>, Wide<T>, Real<T>>::type s = 0;
  __device__ __forceinline__ RowAcc(const MetricQ&, double, double, uint32_t) {}
  __device__ __forceinline__ void step(T x, T q) {
    if constexpr (is_wint_v<T>) s += wide(wabs(wsub(x, q)));
    else if constexpr (is_i16_v<T>) s = __dadd_rn(s, fabs((double)wsub(x, q)));
    else s = rn_add(s, fabs(rn_sub(x, q)));
  }
  __device__ __forceinline__ double finish() const {
    if constexpr (is_wint_v<T>) return (double)wrap<T>(s);
    else return (double)s;
  }
};
// linf_dist (vector.rs:218-233): in T, max starts at 0, `if d > max` (a NaN never wins; abs(MIN) stays negative and
// never wins); I16: fold(0.0, f64::max) of |f64(x) - f64(q)|
template <typename T>
struct RowAcc<SDB_CHEBYSHEV, T> {
  typename std::conditional<is_i16_v<T>, double, T>::type m = 0;
  __device__ __forceinline__ RowAcc(const MetricQ&, double, double, uint32_t) {}
  __device__ __forceinline__ void step(T x, T q) {
    if constexpr (is_i16_v<T>) {
      m = fmax(m, fabs(__dsub_rn((double)x, (double)q)));
    } else if constexpr (std::is_floating_point<T>::value) {
      const T d = fabs(rn_sub(x, q));
      if (d > m) m = d;
    } else {
      const T d = wabs(wsub(x, q));
      if (d > m) m = d;
    }
  }
  __device__ __forceinline__ double finish() const { return (double)m; }
};
template <typename T>
struct RowAcc<SDB_HAMMING, T> {  // vector.rs:291-314: count of x != q (F32, F64: IEEE `!=`, NaN != NaN, 0.0 == -0.0)
  uint32_t c = 0;
  __device__ __forceinline__ RowAcc(const MetricQ&, double, double, uint32_t) {}
  __device__ __forceinline__ void step(T x, T q) { c += x != q; }
  __device__ __forceinline__ double finish() const { return (double)c; }
};
template <typename T>
struct RowAcc<SDB_MINKOWSKI, T> {  // vector.rs:388-410: f64 sum of |f64(x) - f64(q)|^p, then ^(1/p), for every type
  double s = 0.0, p;
  __device__ __forceinline__ RowAcc(const MetricQ& mq, double, double, uint32_t) : p(mq.p) {}
  __device__ __forceinline__ void step(T x, T q) { s = __dadd_rn(s, pow(fabs(__dsub_rn((double)x, (double)q)), p)); }
  __device__ __forceinline__ double finish() const { return pow(s, __ddiv_rn(1.0, p)); }
};
// vector.rs:412-451: sxy / sqrt(sx2 * sy2), 0.0 when that is 0 (a similarity).  The means come from
// pearson_stats_kernel<T>; the loop is f64 for every type.
template <typename T>
struct RowAcc<SDB_PEARSON, T> {
  double sxy = 0.0, mx, sx2, my, sy2;
  __device__ __forceinline__ RowAcc(const MetricQ& mq, double row_mean, double row_sx2, uint32_t)
      : mx(row_mean), sx2(row_sx2), my(mq.mean), sy2(mq.sx2) {}
  __device__ __forceinline__ void step(T x, T q) {
    sxy = __dadd_rn(sxy, __dmul_rn(__dsub_rn((double)x, mx), __dsub_rn((double)q, my)));
  }
  __device__ __forceinline__ double finish() const {
    const double den = __dsqrt_rn(__dmul_rn(sx2, sy2));
    return den == 0.0 ? 0.0 : __ddiv_rn(sxy, den);
  }
};
// COSINE of the types other than F32 (F32 has its own 8-lane paths), 1 - dot / (na * nb) with the norms of
// hnsw_norm_kernel.  F64: dot is ndarray's 8-lane f64 dot (the chain of column c is c mod 8; the 8 chains rotate through
// p[] so that every index is static), folded by fold8, then the < 8 tail columns.  Integers: a.dot(b) is a wrapping sum
// of wrapping products in T -- I16 wraps in i16 -- so any order gives it.  row_norm / q_norm: the two norms (the product
// commutes, so either argument order).
template <typename T>
struct RowAcc<SDB_COSINE, T> {
  double p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  double s = 0.0, na, nb;
  Wide<T> w = 0;
  uint32_t i = 0, d8;
  __device__ __forceinline__ RowAcc(const MetricQ&, double row_norm, double q_norm, uint32_t dim)
      : na(row_norm), nb(q_norm), d8(dim & ~7u) {}
  __device__ __forceinline__ void step(T x, T q) {
    if constexpr (is_f64_v<T>) {
      const double pr = __dmul_rn(x, q);
      if (i < d8) {
        const double t = __dadd_rn(p[0], pr);
#pragma unroll
        for (int j = 0; j < 7; j++) p[j] = p[j + 1];
        p[7] = t;
      } else {
        if (i == d8) s = fold8(p);
        s = __dadd_rn(s, pr);
      }
      i++;
    } else {
      w += wide(x) * wide(q);
    }
  }
  __device__ __forceinline__ double finish() const {
    double dot;
    if constexpr (is_f64_v<T>) dot = i == d8 ? fold8(p) : s;
    else dot = (double)wrap<T>(w);
    return __dsub_rn(1.0, __ddiv_rn(dot, __dmul_rn(na, nb)));
  }
};

// JACCARD from counts.  calculate(a, b): union = the distinct patterns of a; every b_i whose pattern is already in the
// set counts -- all occurrences of a pattern a has, and the 2nd.. occurrences of one it lacks.  With u_a, u_b distinct
// patterns and m shared: inter = dim - (u_b - m), |union| = u_a + u_b - m.  Asymmetric: the caller fixes (a, b).
__device__ __forceinline__ double jaccard_from_counts(uint32_t dim, uint32_t ua, uint32_t ub, uint32_t m) {
  return __ddiv_rn((double)(dim - (ub - m)), (double)(ua + ub - m));
}
// jaccard_f64 (vector.rs:316-327) alone returns 1 - inter / union, a distance; every other type the similarity
template <typename T>
__device__ __forceinline__ double jaccard_typed(uint32_t dim, uint32_t ua, uint32_t ub, uint32_t m) {
  if constexpr (is_f64_v<T>) return __dsub_rn(1.0, jaccard_from_counts(dim, ua, ub, m));
  else return jaccard_from_counts(dim, ua, ub, m);
}
template <typename K>
__device__ __forceinline__ bool sorted_contains(const K* s, uint32_t n, K v) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (s[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && s[lo] == v;
}

// Distance::calculate for VectorType::F32 (idx/trees/vector.rs:218-451,659-672), one thread per vector: the typed
// metric of the walk applied to vectors that are NOT part of the graph -- the new_vectors of pending updates that
// HnswIndex::search_pendings ranks by brute force (hnsw/index.rs:398-404) as calculate(&search.pt, &vector).  Same
// arithmetic as the walk, so a vector gets the same distance whether it is reached through the graph or through the
// pending log.
// The other element types use the same kernel with T and their RowAcc / JACCARD keys.
struct TypedArgs {
  const float* q;          // dim elements of T (typed as F32's: as const void*, the F32 kernels compile to other loads)
  const float* vecs;       // n x dim elements of T
  uint32_t dim;
  uint64_t n;
  double* out;
  MetricQ mq;
  const double* v_mean;    // PEARSON: state of every vector
  const double* v_sx2;
  const void* q_bits;      // JACCARD: the query's sorted distinct keys (mq.u of them, JKey<T>) ...
  const void* v_bits;      // ... and every vector's
  const uint32_t* v_nbits;
  const double* v_norm;    // COSINE, types other than F32: the norms of every vector ...
  const double* q_norm;    // ... and of the query
};
template <int MET, typename T>
__global__ void typed_distance_kernel(TypedArgs A) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= A.n) return;
  const uint32_t dim = A.dim;
  const T* __restrict__ q = reinterpret_cast<const T*>(A.q);
  const T* a = reinterpret_cast<const T*>(A.vecs) + r * dim;
  if constexpr (MET == SDB_COSINE && is_f32_v<T>) {
    float p[8] = {0, 0, 0, 0, 0, 0, 0, 0}, pa[8] = {0, 0, 0, 0, 0, 0, 0, 0}, pq[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t i = 0;
    for (; i + 8 <= dim; i += 8)
#pragma unroll
      for (int j = 0; j < 8; j++) {
        p[j] = __fadd_rn(p[j], __fmul_rn(a[i + j], q[i + j]));
        pa[j] = __fadd_rn(pa[j], __fmul_rn(a[i + j], a[i + j]));
        pq[j] = __fadd_rn(pq[j], __fmul_rn(q[i + j], q[i + j]));
      }
    // fold8 of p, pa and pq, interleaved (three separate fold8 calls schedule differently)
    float dot = 0.f, sa = 0.f, sq = 0.f;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      dot = __fadd_rn(dot, __fadd_rn(p[j], p[j + 4]));
      sa = __fadd_rn(sa, __fadd_rn(pa[j], pa[j + 4]));
      sq = __fadd_rn(sq, __fadd_rn(pq[j], pq[j + 4]));
    }
    for (; i < dim; i++) {
      dot = __fadd_rn(dot, __fmul_rn(a[i], q[i]));
      sa = __fadd_rn(sa, __fmul_rn(a[i], a[i]));
      sq = __fadd_rn(sq, __fmul_rn(q[i], q[i]));
    }
    const double na = __dsqrt_rn((double)sa), nb = __dsqrt_rn((double)sq);
    // calculate(a = search.pt, b = vector): dot and the product of norms are symmetric
    A.out[r] = __dsub_rn(1.0, __ddiv_rn((double)dot, __dmul_rn(na, nb)));
  } else if constexpr (MET == SDB_JACCARD) {
    // calculate(a = query, b = vector)
    using K = JKey<T>;
    const uint32_t ub = A.v_nbits[r];
    const K* vb = static_cast<const K*>(A.v_bits) + r * dim;
    uint32_t m = 0;
    for (uint32_t i = 0; i < ub; i++) m += sorted_contains(static_cast<const K*>(A.q_bits), A.mq.u, vb[i]);
    A.out[r] = jaccard_typed<T>(dim, A.mq.u, ub, m);
  } else {
    RowAcc<MET, T> acc(A.mq, MET == SDB_PEARSON ? A.v_mean[r] : MET == SDB_COSINE ? A.v_norm[r] : 0.0,
                       MET == SDB_PEARSON ? A.v_sx2[r] : MET == SDB_COSINE ? *A.q_norm : 0.0, dim);
    for (uint32_t i = 0; i < dim; i++) acc.step(a[i], q[i]);
    A.out[r] = acc.finish();
  }
}

// ---- the walk's per-warp shared memory: the staged query, the distance scratch, then the 8-byte keys and 4-byte ids of
// the candidate (ccap entries) and result (wcap entries) queues.  f32_cosine: the index is F32 COSINE (the 8-lane path).
// F32 cosine keeps the query TRANSPOSED: qT[j * qs + i] = q[8i + j] (chain j contiguous), qs = hn_q_stride = 4 mod 32
// words so the 8 lanes of a row read 8 different bank groups with one LDS.128 per 4 steps; the < 8 tail columns follow
// at qT[8 * qs ...].
__host__ __device__ constexpr uint32_t hn_q_stride(uint32_t dim) { return (((dim >> 3) + 27u) / 32u) * 32u + 4u; }
// F32's other metrics keep the query as dim floats (JACCARD: its <= dim sorted distinct bit patterns).
__host__ __device__ constexpr size_t hn_q_floats(uint32_t dim, bool cosine) {
  return cosine ? (size_t)8 * hn_q_stride(dim) + 8 : (size_t)((dim + 3) & ~3u);
}
// Bytes of the staged query, a multiple of 16.  f32: the index is F32, counted in floats; every other type keeps dim
// elements of elem bytes (its own type, or its JACCARD keys), cosine included: it walks the one-chain tile path there.
__host__ __device__ constexpr size_t hn_q_bytes(uint32_t dim, bool f32, bool cosine, size_t elem) {
  return f32 ? sizeof(float) * hn_q_floats(dim, cosine) : ((size_t)dim * elem + 15) & ~size_t(15);
}
// Scratch of the distance phase.  F32 cosine: 32 compacted row ids + 32 f64 results (the rows are read straight from
// global memory, see warp_distance_cosine_f32).  Every other cell: a 32 x 33 float transposing tile (JACCARD uses 32
// compacted row ids + 32 f64 results of it).
__host__ __device__ constexpr size_t hn_tile_bytes(bool f32_cosine) { return f32_cosine ? 32 * 4 + 32 * 8 : sizeof(float) * 32 * 33; }

// distance of this lane's row (or NO_ROW) to the query held in shared memory; all 32 lanes must call.
// F32 COSINE.  ndarray's f32 dot (a6; oracle orc_nd_dot_f32) keeps 8 running sums p_j over the columns 8i+j, each one a
// strictly sequential chain over i, and folds them with fold8 followed by the <8 tail columns.  The 8 chains of a row
// are independent, so a row is given to 8 LANES (lane j = chain j) and a warp works on 4 rows at a time -- two such
// quads interleaved when more than 4 rows are new, so every lane carries two independent chains.  Lane (g, j) reads
// x[row_g][8i+j] directly from global memory: the 8 lanes of a row cover one 32-byte sector and the 4 rows of a quad 4
// sectors, i.e. a request moves as many bytes as a fully coalesced one; no shared-memory transposition, 8 x fewer
// dependent steps per row than one lane per row (the walk was bound by issue latency: ncu r1, 30 % issue-active at 13
// cycles per instruction, ~6.7k instructions per expanded node).
__device__ __forceinline__ double warp_distance_cosine_f32(const float* __restrict__ vec, const double* __restrict__ norm,
                                                           uint32_t dim, uint32_t my_row, const float* s_q, double q_norm,
                                                           float (*tile)[33]) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t d8 = dim & ~7u, steps = dim >> 3, qs = hn_q_stride(dim);
  uint32_t* ids = reinterpret_cast<uint32_t*>(tile);
  double* res = reinterpret_cast<double*>(ids + 32);
  const uint32_t vmask = __ballot_sync(0xffffffffu, my_row != NO_ROW);
  const uint32_t n_rows = __popc(vmask);
  const uint32_t ci = __popc(vmask & ((1u << lane) - 1u));  // compact index of this lane's row
  if (my_row != NO_ROW) ids[ci] = my_row;
  __syncwarp();
  const uint32_t grp = lane >> 3, j = lane & 7u;
  const float* qj = s_q + j * qs;
  const uint32_t row_bytes = dim * 4u;
  for (uint32_t g0 = 0; g0 < n_rows; g0 += 8) {
    const uint32_t ia = g0 + grp, ib = g0 + 4 + grp;
    const bool va = ia < n_rows, vb = ib < n_rows;
    const uint32_t ra = va ? ids[ia] : 0u, rb = vb ? ids[ib] : 0u;
    const float* xa = vec + (size_t)ra * dim + j;
    const float* xb = vec + (size_t)rb * dim + j;
    // ask L2 for every line of the rows of this round up front (lane j: lines j, j+8, ...): the first loads below pay
    // the DRAM latency once, the later ones find their sectors in L2
    if (va)
      for (uint32_t off = j * 128u; off < row_bytes; off += 8u * 128u)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(xa - j) + off));
    if (vb)
      for (uint32_t off = j * 128u; off < row_bytes; off += 8u * 128u)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(xb - j) + off));
    double na = 0.0, nb = 0.0;
    if (va && j == 0) na = __ldg(norm + ra);
    if (vb && j == 0) nb = __ldg(norm + rb);
    float pa = 0.f, pb = 0.f;
    uint32_t i = 0;
    if (g0 + 4 < n_rows) {  // (warp-uniform) two quads
      for (; i + 8 <= steps; i += 8) {
        float a[8], b[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
          a[u] = va ? __ldg(xa + 8u * (i + u)) : 0.f;
          b[u] = vb ? __ldg(xb + 8u * (i + u)) : 0.f;
        }
        const float4 q0 = *reinterpret_cast<const float4*>(qj + i), q1 = *reinterpret_cast<const float4*>(qj + i + 4);
        const float qv[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
        for (int u = 0; u < 8; u++) {
          pa = __fadd_rn(pa, __fmul_rn(a[u], qv[u]));
          pb = __fadd_rn(pb, __fmul_rn(b[u], qv[u]));
        }
      }
      for (; i < steps; i++) {
        const float qv = qj[i];
        pa = __fadd_rn(pa, __fmul_rn(va ? __ldg(xa + 8u * i) : 0.f, qv));
        pb = __fadd_rn(pb, __fmul_rn(vb ? __ldg(xb + 8u * i) : 0.f, qv));
      }
    } else {  // one quad: deeper unroll for the same number of loads in flight
      for (; i + 16 <= steps; i += 16) {
        float a[16];
#pragma unroll
        for (int u = 0; u < 16; u++) a[u] = va ? __ldg(xa + 8u * (i + u)) : 0.f;
#pragma unroll
        for (int v4 = 0; v4 < 4; v4++) {
          const float4 q4 = *reinterpret_cast<const float4*>(qj + i + 4 * v4);
          pa = __fadd_rn(pa, __fmul_rn(a[4 * v4 + 0], q4.x));
          pa = __fadd_rn(pa, __fmul_rn(a[4 * v4 + 1], q4.y));
          pa = __fadd_rn(pa, __fmul_rn(a[4 * v4 + 2], q4.z));
          pa = __fadd_rn(pa, __fmul_rn(a[4 * v4 + 3], q4.w));
        }
      }
      for (; i < steps; i++) pa = __fadd_rn(pa, __fmul_rn(va ? __ldg(xa + 8u * i) : 0.f, qj[i]));
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const bool v = h ? vb : va;
      float dot = quad_fold8(h ? pb : pa, v && j == 0);
      if (v && j == 0) {
        const uint32_t row = h ? rb : ra;
        for (uint32_t c = d8; c < dim; c++)
          dot = __fadd_rn(dot, __fmul_rn(__ldg(vec + (size_t)row * dim + c), s_q[8u * qs + (c - d8)]));
        res[h ? ib : ia] = __dsub_rn(1.0, __ddiv_rn((double)dot, __dmul_rn(h ? nb : na, q_norm)));
      }
    }
  }
  __syncwarp();
  return my_row != NO_ROW ? res[ci] : 0.0;
}

// EUCLID and the other one-chain metrics (MANHATTAN, CHEBYSHEV, HAMMING in f32; MINKOWSKI, PEARSON in f64, see RowAcc),
// and every metric but JACCARD for the other element types (COSINE there: RowAcc<SDB_COSINE, T>).
// ndarray-stats' l2_dist folds (a-b)^2 strictly sequentially over the columns: one chain per row, so a row stays on ONE
// lane and the rows of a round are transposed through shared memory (coalesced fetches, 256 bytes of a row a step).
// row_mean / row_sx2: the PEARSON state of the elements (null for the other metrics); COSINE: row_mean = the element
// norms, q_norm the query's.
template <int MET, typename T>
__device__ __forceinline__ double warp_distance_rows(const T* __restrict__ vec, uint32_t dim, uint32_t my_row,
                                                     const T* s_q, float (*tile)[33], const MetricQ& mq,
                                                     const double* __restrict__ row_mean, const double* __restrict__ row_sx2,
                                                     double q_norm = 0.0) {
  constexpr uint32_t CW = 256u / sizeof(T);  // columns per step (f32: 64)
  const uint32_t lane = threadIdx.x & 31u;
  RowAcc<MET, T> acc(mq, (MET == SDB_PEARSON || MET == SDB_COSINE) && my_row != NO_ROW ? __ldg(row_mean + my_row) : 0.0,
                     MET == SDB_PEARSON && my_row != NO_ROW ? __ldg(row_sx2 + my_row) : MET == SDB_COSINE ? q_norm : 0.0, dim);
  // Only a handful of the <=32 neighbours of an expanded node are new (6 on average): the valid rows are compacted and
  // handled in rounds of 16; the 32 x 33 float scratch is viewed as 16 rows x (256 bytes + 2 padding words), so one
  // step moves 64 f32 columns of every row of the round -- up to 32 independent loads per lane in flight per wait
  // instead of 4.  The padding words park the compacted row ids.
  float(*t)[66] = reinterpret_cast<float(*)[66]>(tile);
  const uint32_t vmask = __ballot_sync(0xffffffffu, my_row != NO_ROW);
  const uint32_t n_rows = __popc(vmask);
  const uint32_t ci = __popc(vmask & ((1u << lane) - 1u));  // compact index of this lane's row
  if (my_row != NO_ROW) t[ci & 15u][64 + (ci >> 4)] = __uint_as_float(my_row);
  __syncwarp();
  {
    const uint32_t row_bytes = dim * (uint32_t)sizeof(T);
    for (uint32_t r = 0; r < n_rows; r++) {
      const char* base = reinterpret_cast<const char*>(vec + (size_t)__float_as_uint(t[r & 15u][64 + (r >> 4)]) * dim);
      for (uint32_t off = lane * 128u; off < row_bytes; off += 32u * 128u)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(base + off));
    }
  }
  for (uint32_t g0 = 0; g0 < n_rows; g0 += 16) {
    const uint32_t nr = n_rows - g0 < 16u ? n_rows - g0 : 16u;
    const bool mine = my_row != NO_ROW && (ci >> 4) == (g0 >> 4);
    const T* x = reinterpret_cast<const T*>(t[ci & 15u]);
    for (uint32_t c0 = 0; c0 < dim; c0 += CW) {
      if constexpr (is_f32_v<T>) {
        const bool in0 = c0 + lane < dim, in1 = c0 + 32 + lane < dim;
#pragma unroll 4
        for (uint32_t r = 0; r < nr; r++) {
          const float* src = vec + (size_t)__float_as_uint(t[r][64 + (g0 >> 4)]) * dim + c0 + lane;  // broadcast id read
          const float v0 = in0 ? __ldg(src) : 0.f;
          const float v1 = in1 ? __ldg(src + 32) : 0.f;
          t[r][lane] = v0;
          t[r][lane + 32] = v1;
        }
      } else {
#pragma unroll 4
        for (uint32_t r = 0; r < nr; r++) {
          const T* src = vec + (size_t)__float_as_uint(t[r][64 + (g0 >> 4)]) * dim + c0 + lane;
          T v[CW / 32];
#pragma unroll
          for (uint32_t u = 0; u < CW / 32; u++) v[u] = c0 + 32u * u + lane < dim ? __ldg(src + 32u * u) : T(0);
#pragma unroll
          for (uint32_t u = 0; u < CW / 32; u++) reinterpret_cast<T*>(t[r])[lane + 32u * u] = v[u];
        }
      }
      __syncwarp();
      if (mine) {
        const uint32_t lim = dim - c0 < CW ? dim - c0 : CW;
        for (uint32_t jj = 0; jj < lim; jj++) acc.step(x[jj], s_q[c0 + jj]);
      }
      __syncwarp();
    }
  }
  if (my_row == NO_ROW) return 0.0;
  return acc.finish();
}

// JACCARD, calculate(a = element, b = query): only m = |distinct(element) & distinct(query)| is per pair.  The query's
// sorted distinct keys (q_u of them) are in shared memory; the warp takes one new row at a time, every lane binary-
// searching a 32-key slice of the row's distinct list.  QFIRST: calculate(a = query, b = element) instead, from the same
// counts (the re-sort mode of the neighbour selection).
template <typename T, bool QFIRST = false>
__device__ __forceinline__ double warp_distance_jaccard(const JKey<T>* __restrict__ bits, const uint32_t* __restrict__ nbits,
                                                        uint32_t dim, uint32_t my_row, const JKey<T>* s_qb, uint32_t q_u,
                                                        float (*tile)[33]) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t* ids = reinterpret_cast<uint32_t*>(tile);
  double* res = reinterpret_cast<double*>(ids + 32);
  const uint32_t vmask = __ballot_sync(0xffffffffu, my_row != NO_ROW);
  const uint32_t n_rows = __popc(vmask);
  const uint32_t ci = __popc(vmask & ((1u << lane) - 1u));
  if (my_row != NO_ROW) ids[ci] = my_row;
  __syncwarp();
  for (uint32_t r = 0; r < n_rows; r++) {
    const uint32_t row = ids[r];
    const uint32_t ua = __ldg(nbits + row);
    const JKey<T>* eb = bits + (size_t)row * dim;
    uint32_t m = 0;
    for (uint32_t i = lane; i < ua; i += 32) m += sorted_contains(s_qb, q_u, __ldg(eb + i));
    m = __reduce_add_sync(0xffffffffu, m);
    if (lane == 0) res[r] = QFIRST ? jaccard_typed<T>(dim, q_u, ua, m) : jaccard_typed<T>(dim, ua, q_u, m);
  }
  __syncwarp();
  return my_row != NO_ROW ? res[ci] : 0.0;
}

// sorted (ascending key, FIFO inside a key) array insert by the whole warp; entries live in [head, n).  One pass from
// the top: every 32-entry chunk above the insertion point moves up by one; the chunk that holds an entry <= key fixes the
// position (the new entry goes AFTER its equals).
__device__ __forceinline__ uint32_t sorted_insert(uint64_t* keys, uint32_t* ids, uint32_t head, uint32_t n, uint64_t key,
                                                  uint32_t id) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t pos = head;
  for (uint32_t hi = n; hi > head;) {
    const uint32_t lo = hi - head > 32u ? hi - 32u : head;
    const uint32_t i = lo + lane;
    uint64_t k = 0;
    uint32_t v = 0;
    const bool in = i < hi;
    if (in) {
      k = keys[i];
      v = ids[i];
    }
    const uint32_t le = __ballot_sync(0xffffffffu, in && k <= key);
    __syncwarp();  // every lane has read its entry before a neighbour overwrites it
    if (in && k > key) {
      keys[i + 1] = k;
      ids[i + 1] = v;
    }
    __syncwarp();
    if (le) {
      pos = lo + __popc(le);
      break;
    }
    hi = lo;
  }
  if (lane == 0) {
    keys[pos] = key;
    ids[pos] = id;
  }
  __syncwarp();
  return n + 1;
}

struct HnswParams {
  const void* vec;        // n x dim elements of the index's type
  const double* norm;     // sqrt((double)sumsq) per element (cosine)
  const uint64_t* const* rp;
  const uint32_t* const* ci;
  uint32_t dim, n_layers;
  int64_t entry;
  const void* queries;    // nq x dim elements of the index's type
  uint32_t nq, k, ef;
  uint32_t ccap;          // capacity of the candidate window (entries)
  const uint8_t* truthy;  // non-null: knn_search_with_filter -- one byte per element (layer 0 only)
  const uint8_t* noexp;   // non-null: pending docs -- noexp[e] != 0: every document of element e has a pending update;
                          // the element still enters w but is never expanded (layer.rs:209, every layer)
  uint64_t* visited;
  uint32_t table_log2;
  uint32_t gen_base, gens_per_warp;
  uint64_t* out_elems;
  double* out_dist;
  uint32_t* out_count;
  uint64_t* out_counters;
  uint32_t* overflow;
  const int* cancel;  // mapped host flag (sdb_ctx_cancel): polled before every query
  // state of the metrics that carry it (unused by cosine / euclid)
  double mink_p;              // MINKOWSKI order
  const double* e_mean;       // PEARSON: per element / per query mean and sum of squared deviations
  const double* e_sx2;
  const double* q_mean;
  const double* q_sx2;
  const void* e_bits;         // JACCARD: per element / per query sorted distinct keys (JKey, dim-strided) and count
  const uint32_t* e_nbits;
  const void* q_bits;
  const uint32_t* q_nbits;
  const double* q_norm;       // COSINE of the types other than F32: per query norm (the elements' are `norm`)
  // the batch-filtered walk (hnsw_search_kernel<.., BITS = true>, hnsw_spill_kernel): per-query element bitmaps
  const uint32_t* filters;       // bitmaps of fwords words: element e passes iff bit e % 32 of word e / 32 is set
  const uint32_t* query_filter;  // nq bitmap indices (null: every query uses bitmap 0)
  uint32_t fwords;
  uint32_t* spill_list;  // the queries the on-chip walk gave up on (candidate window or visited table full) ...
  uint32_t* n_spill;     // ... and how many there are
};

// bit e of a filter bitmap
__device__ __forceinline__ bool filter_bit(const uint32_t* bits, uint32_t e) { return (__ldg(bits + (e >> 5)) >> (e & 31u)) & 1u; }
// the bitmap query q tests
__device__ __forceinline__ const uint32_t* query_bits(const HnswParams& P, uint32_t q) {
  return P.filters + (size_t)(P.query_filter ? P.query_filter[q] : 0u) * P.fwords;
}

// Stages vector r of a set (the queries of a walk, or an element) in shared memory as the distance functions above read
// it: F32 COSINE transposed (hn_q_stride) with its 8-lane norm computed here (the same arithmetic as the elements'
// hnsw_norm_f32_kernel), JACCARD its sorted distinct keys, every other cell its dim elements; the set's metric state at
// r goes to q_norm / mq.  All 32 lanes must call.  The same steps as the staging in hnsw_search_kernel, which keeps its
// own inline copy, so that the walk's generated code stays as it was (calling this from there schedules it differently).
template <int MET, typename T, typename I>
__device__ __forceinline__ void stage_vector(uint32_t dim, const void* vecs, const double* norm, const double* mean,
                                             const double* sx2, const void* bits, const uint32_t* nbits, double mink_p,
                                             I r, float* s_q, double& q_norm, MetricQ& mq) {
  constexpr bool COSINE = MET == SDB_COSINE && is_f32_v<T>;
  const uint32_t lane = threadIdx.x & 31;
  if (COSINE) {
    const uint32_t qs = hn_q_stride(dim), d8 = dim & ~7u, steps = dim >> 3;
    const float* qg = static_cast<const float*>(vecs) + (size_t)r * dim;
    for (uint32_t c = lane; c < dim; c += 32) {
      const float v = qg[c];
      if (c < d8) s_q[(c & 7u) * qs + (c >> 3)] = v;
      else s_q[8u * qs + (c - d8)] = v;
    }
    __syncwarp();
    float p = 0.f;
    if (lane < 8)
      for (uint32_t i = 0; i < steps; i++) {
        const float v = s_q[lane * qs + i];
        p = __fadd_rn(p, __fmul_rn(v, v));
      }
    float q_sumsq = quad_fold8(p, true);
    for (uint32_t c = d8; c < dim; c++) {
      const float v = s_q[8u * qs + (c - d8)];
      q_sumsq = __fadd_rn(q_sumsq, __fmul_rn(v, v));
    }
    q_norm = __dsqrt_rn((double)__shfl_sync(0xffffffffu, q_sumsq, 0));
  } else if (MET == SDB_JACCARD) {
    mq.u = nbits[r];
    JKey<T>* s_qb = reinterpret_cast<JKey<T>*>(s_q);
    for (uint32_t c = lane; c < mq.u; c += 32) s_qb[c] = static_cast<const JKey<T>*>(bits)[(size_t)r * dim + c];
    __syncwarp();
  } else {
    T* s_qt = reinterpret_cast<T*>(s_q);
    for (uint32_t c = lane; c < dim; c += 32) s_qt[c] = static_cast<const T*>(vecs)[(size_t)r * dim + c];
    __syncwarp();
    if (MET == SDB_PEARSON) {
      mq.mean = mean[r];
      mq.sx2 = sx2[r];
    }
    if (MET == SDB_MINKOWSKI) mq.p = mink_p;
    if (MET == SDB_COSINE) q_norm = norm[r];
  }
}

template <int MET, typename T>
__device__ __forceinline__ double walk_distance(const HnswParams& P, uint32_t my_row, const float* s_q, double q_norm,
                                                const MetricQ& mq, float (*tile)[33]) {
  if constexpr (MET == SDB_COSINE && is_f32_v<T>)
    return warp_distance_cosine_f32(static_cast<const float*>(P.vec), P.norm, P.dim, my_row, s_q, q_norm, tile);
  else if constexpr (MET == SDB_JACCARD)
    return warp_distance_jaccard<T>(static_cast<const JKey<T>*>(P.e_bits), P.e_nbits, P.dim, my_row,
                                    reinterpret_cast<const JKey<T>*>(s_q), mq.u, tile);
  else
    return warp_distance_rows<MET, T>(static_cast<const T*>(P.vec), P.dim, my_row, reinterpret_cast<const T*>(s_q), tile,
                                      mq, MET == SDB_COSINE ? P.norm : P.e_mean, P.e_sx2, q_norm);
}

// T: the element type of the index (float = F32; double, long long, int, short = F64, I64, I32, I16)
// BITS: the batch-filtered walk.  Layer 0 tests bit e of the query's own bitmap (query_bits) where the single-mask walk
// reads truthy[e], and a query that fills its candidate window or its visited table stops at once and is appended to
// the spill list (hnsw_spill_kernel walks it again and writes its outputs) instead of raising the batch's overflow word.
template <int MET, int MINB, typename T, bool BITS = false>
__global__ void __launch_bounds__(HN_WARPS * 32, MINB) hnsw_search_kernel(HnswParams P) {
  constexpr bool COSINE = MET == SDB_COSINE && is_f32_v<T>;  // the 8-lane transposed path of F32 cosine
  constexpr size_t ELEM = MET == SDB_JACCARD ? sizeof(JKey<T>) : sizeof(T);  // bytes of a staged query element
  extern __shared__ uint8_t smem_raw[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ccap = P.ccap, wcap = P.ef + 2;
  // per-warp shared layout
  const size_t per_warp = hn_q_bytes(P.dim, is_f32_v<T>, MET == SDB_COSINE, ELEM) + hn_tile_bytes(COSINE) + (sizeof(uint64_t) + sizeof(uint32_t)) * (ccap + wcap) + 64;
  uint8_t* base = smem_raw + (size_t)warp * ((per_warp + 15) & ~size_t(15));
  // query first (16-byte aligned: LDS.128), then the distance scratch, the 8-byte keys, the 4-byte ids
  float* s_q = reinterpret_cast<float*>(base);
  float(*tile)[33] = reinterpret_cast<float(*)[33]>(is_f32_v<T> ? s_q + ((hn_q_floats(P.dim, COSINE) + 3) & ~size_t(3))
                                                                : reinterpret_cast<float*>(base + hn_q_bytes(P.dim, false, false, ELEM)));
  uint64_t* c_key = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(tile) + hn_tile_bytes(COSINE));
  uint64_t* w_key = c_key + ccap;
  uint32_t* c_id = reinterpret_cast<uint32_t*>(w_key + wcap);
  uint32_t* w_id = c_id + ccap;

  const uint32_t gwarp = blockIdx.x * HN_WARPS + warp;
  const uint32_t n_warps = gridDim.x * HN_WARPS;
  uint64_t* table = P.visited + ((size_t)gwarp << P.table_log2);
  const uint32_t mask = (1u << P.table_log2) - 1u;
  uint32_t gen = P.gen_base + gwarp * P.gens_per_warp;

  for (uint32_t q = gwarp; q < P.nq; q += n_warps) {
    if (*reinterpret_cast<const volatile int*>(P.cancel)) break;  // uniform per warp: every lane reads the same word
    // stage the query (cosine: transposed, see hn_q_stride) and its 8-lane sum of squares
    double q_norm = 0.0;
    MetricQ mq;
    if (COSINE) {
      const uint32_t qs = hn_q_stride(P.dim), d8 = P.dim & ~7u, steps = P.dim >> 3;
      const float* qg = static_cast<const float*>(P.queries) + (size_t)q * P.dim;
      for (uint32_t c = lane; c < P.dim; c += 32) {
        const float v = qg[c];
        if (c < d8) s_q[(c & 7u) * qs + (c >> 3)] = v;
        else s_q[8u * qs + (c - d8)] = v;
      }
      __syncwarp();
      float p = 0.f;
      if (lane < 8)
        for (uint32_t i = 0; i < steps; i++) {
          const float v = s_q[lane * qs + i];
          p = __fadd_rn(p, __fmul_rn(v, v));
        }
      float q_sumsq = quad_fold8(p, true);
      for (uint32_t c = d8; c < P.dim; c++) {
        const float v = s_q[8u * qs + (c - d8)];
        q_sumsq = __fadd_rn(q_sumsq, __fmul_rn(v, v));
      }
      q_norm = __dsqrt_rn((double)__shfl_sync(0xffffffffu, q_sumsq, 0));
    } else if (MET == SDB_JACCARD) {
      mq.u = P.q_nbits[q];
      JKey<T>* s_qb = reinterpret_cast<JKey<T>*>(s_q);
      for (uint32_t c = lane; c < mq.u; c += 32) s_qb[c] = static_cast<const JKey<T>*>(P.q_bits)[(size_t)q * P.dim + c];
      __syncwarp();
    } else {
      T* s_qt = reinterpret_cast<T*>(s_q);
      for (uint32_t c = lane; c < P.dim; c += 32) s_qt[c] = static_cast<const T*>(P.queries)[(size_t)q * P.dim + c];
      __syncwarp();
      if (MET == SDB_PEARSON) {
        mq.mean = P.q_mean[q];
        mq.sx2 = P.q_sx2[q];
      }
      if (MET == SDB_MINKOWSKI) mq.p = P.mink_p;
      if (MET == SDB_COSINE) q_norm = P.q_norm[q];
    }
    uint64_t n_visited = 0, n_expanded = 0;
    uint32_t n_out = 0;
    const uint32_t* qbits = BITS ? query_bits(P, q) : nullptr;
    bool spill = false;  // BITS: this query goes to the spill tier (warp-uniform once set)
    if (P.entry >= 0) {
      uint32_t ep = (uint32_t)P.entry;
      double ep_d = walk_distance<MET, T>(P, lane == 0 ? ep : NO_ROW, s_q, q_norm, mq, tile);
      ep_d = __shfl_sync(0xffffffffu, ep_d, 0);
      n_visited++;
      for (int32_t layer = (int32_t)P.n_layers - 1; layer >= 0; layer--) {
        const uint32_t ef = layer == 0 ? P.ef : 1u;
        const uint64_t* rp = P.rp[layer];
        const uint32_t* ci = P.ci[layer];
        gen++;
        // search_single: visited = {ep}; candidates = w = {(ep_d, ep)}        layer.rs:76-90
        uint32_t head = 0, cn = 0, wn = 0;
        {
          const uint64_t my = ((uint64_t)gen << 32) | ep;
          if (lane == 0) {
            uint32_t slot = (ep * 2654435761u) & mask;
            while ((table[slot] >> 32) == gen) slot = (slot + 1) & mask;
            table[slot] = my;
          }
          __syncwarp();
        }
        // search_single_with_filter (layer.rs:111-149): w starts with ep only if one of its documents is truthy
        const uint8_t* truthy = layer == 0 ? P.truthy : nullptr;
        cn = sorted_insert(c_key, c_id, head, cn, walk_key(ep_d), ep);
        double fd = 1.7976931348623157e308;  // w.peek_last_dist().unwrap_or(f64::MAX)
        if (BITS ? layer != 0 || filter_bit(qbits, ep) : !truthy || truthy[ep]) {
          wn = sorted_insert(w_key, w_id, 0, wn, walk_key(ep_d), ep);
          fd = ep_d;
        }
        while (head < cn) {
          const uint64_t ckey = c_key[head];
          const uint32_t cid = c_id[head];
          head++;
          if (key_to_double(ckey) > fd) break;  // cq_dist > fq_dist
          n_expanded++;
          const uint64_t beg = rp[cid], end = rp[cid + 1];
          for (uint64_t b0 = beg; b0 < end; b0 += 32) {
            const uint32_t nb = b0 + lane < end ? __ldg(ci + b0 + lane) : NO_ROW;
            bool is_new = false;
            if (nb != NO_ROW) {  // visited.insert(e_id)
              const uint64_t my = ((uint64_t)gen << 32) | nb;
              uint32_t slot = (nb * 2654435761u) & mask;
              for (uint32_t probes = 0;; probes++) {
                const uint64_t cur = *reinterpret_cast<volatile uint64_t*>(table + slot);
                if (cur == my) break;
                if ((uint32_t)(cur >> 32) != gen) {
                  const uint64_t old = atomicCAS(reinterpret_cast<unsigned long long*>(table + slot),
                                                 (unsigned long long)cur, (unsigned long long)my);
                  if (old == cur) {
                    is_new = true;
                    break;
                  }
                  if (old == my) break;
                  if ((uint32_t)(old >> 32) != gen) continue;
                }
                if (probes > mask) {  // table full: report, treat as visited
                  if (BITS) spill = true;
                  else *P.overflow = 1;
                  break;
                }
                slot = (slot + 1) & mask;
              }
            }
            const uint32_t new_mask = __ballot_sync(0xffffffffu, is_new);
            if (BITS && __any_sync(0xffffffffu, spill)) {
              spill = true;
              break;
            }
            if (!new_mask) continue;
            n_visited += __popc(new_mask);
            const double d = walk_distance<MET, T>(P, is_new ? nb : NO_ROW, s_q, q_norm, mq, tile);
            // admission in stored order                                     layer.rs:205-217
            uint32_t m = new_mask;
            while (m) {
              const int i = __ffs(m) - 1;
              m &= m - 1;
              const double di = __shfl_sync(0xffffffffu, d, i);
              const uint32_t idi = __shfl_sync(0xffffffffu, nb, i);
              if (di < fd || wn < ef) {
                const uint64_t key = walk_key(di);
                if (cn >= ccap) {  // slide the live window down (or, if truly full, drop the farthest tie)
                  if (head > 0) {
                    for (uint32_t lo = head; lo < cn; lo += 32) {
                      const uint32_t j = lo + lane;
                      uint64_t kk = 0;
                      uint32_t vv = 0;
                      if (j < cn) { kk = c_key[j]; vv = c_id[j]; }
                      __syncwarp();
                      if (j < cn) { c_key[j - head] = kk; c_id[j - head] = vv; }
                      __syncwarp();
                    }
                    cn -= head;
                    head = 0;
                  }
                  if (cn >= ccap) {
                    if (BITS) {
                      spill = true;
                      break;
                    }
                    cn = ccap - 1;
                    *P.overflow = 2;
                  }
                }
                if (!P.noexp || !P.noexp[idi]) cn = sorted_insert(c_key, c_id, head, cn, key, idi);
                if (BITS ? layer != 0 || filter_bit(qbits, idi) : !truthy || truthy[idi]) {  // add_if_truthy  layer.rs:277-306
                  wn = sorted_insert(w_key, w_id, 0, wn, key, idi);
                  if (wn > ef) wn--;  // pop_last
                  fd = key_to_double(w_key[wn - 1]);
                }
                if (wn == ef) {  // candidates beyond f can never be expanded any more
                  // (cq_dist > fq_dist is an f64 comparison: a 0.0 candidate is not beyond a -0.0 f)
                  const uint64_t fkey = zero_tie(w_key[wn - 1]);
                  while (cn > head && zero_tie(c_key[cn - 1]) > fkey) cn--;
                }
              }
            }
            if (BITS && spill) break;
          }
          if (BITS && spill) break;
        }
        if (BITS && spill) break;
        // next layer starts from w.peek_first()                                mod.rs:530-538
        if (wn) {
          ep = w_id[0];
          ep_d = key_to_double(w_key[0]);
        }
        if (layer == 0) {
          n_out = wn < P.k ? wn : P.k;  // to_vec_limit(k)
          for (uint32_t i = lane; i < n_out; i += 32) {
            P.out_elems[(size_t)q * P.k + i] = w_id[i];
            P.out_dist[(size_t)q * P.k + i] = key_to_double(w_key[i]);
          }
        }
        __syncwarp();
      }
    }
    if (BITS && spill) {  // outputs and counters come from the spill tier
      if (lane == 0) P.spill_list[atomicAdd(P.n_spill, 1u)] = q;
      continue;
    }
    if (lane == 0) {
      P.out_count[q] = n_out;
      if (P.out_counters) {
        P.out_counters[2 * (size_t)q] = n_visited;
        P.out_counters[2 * (size_t)q + 1] = n_expanded;
      }
    }
  }
}

// Bytes of one warp's staged vector and distance scratch in the kernels that share the walk's distance code.
static size_t hn_stage_bytes(uint32_t dim, sdb_metric metric, sdb_vector_type vt) {
  const size_t elem = metric == SDB_JACCARD ? (vt == SDB_VT_F64 || vt == SDB_VT_I64 ? 8 : 4)
                                            : (vt == SDB_VT_F64 || vt == SDB_VT_I64 ? 8 : vt == SDB_VT_I16 ? 2 : 4);
  return hn_q_bytes(dim, vt == SDB_VT_F32, metric == SDB_COSINE, elem) + hn_tile_bytes(vt == SDB_VT_F32 && metric == SDB_COSINE);
}
// the staged vector and the distance scratch of one warp (hnsw_search_kernel's layout), then `rest`
template <int MET, typename T>
__device__ __forceinline__ void hn_warp_layout(uint8_t* base, uint32_t dim, float*& s_q, float (*&tile)[33], uint8_t*& rest) {
  constexpr bool COSINE = MET == SDB_COSINE && is_f32_v<T>;
  constexpr size_t ELEM = MET == SDB_JACCARD ? sizeof(JKey<T>) : sizeof(T);
  s_q = reinterpret_cast<float*>(base);
  tile = reinterpret_cast<float(*)[33]>(is_f32_v<T> ? s_q + ((hn_q_floats(dim, COSINE) + 3) & ~size_t(3))
                                                    : reinterpret_cast<float*>(base + hn_q_bytes(dim, false, false, ELEM)));
  rest = reinterpret_cast<uint8_t*>(tile) + hn_tile_bytes(COSINE);
}

// ---- spill tier of the batch-filtered walk: the queries hnsw_search_kernel<.., BITS> gave up on, walked again from the
// top layer with no capacity limit.  One warp per slot; a slot is
//   heap:  a binary min-heap of (walk_key, tag = insertion sequence << 32 | element) in global memory, n entries: an
//          element enters a layer's candidates at most once (it is visited once), so n is a hard bound.  Popping by
//          (key, sequence) is sorted_insert's order -- nearest first, FIFO among equal keys -- without the window.
//   stamp: one u32 per element, the slot's layer generation that last visited it (an exact visited set; 0 = never).
// w (ef + 2 entries) stays in shared memory, as in the on-chip walk.  Lane 0 owns the heap; the other lanes wait.
struct SpillSlots {
  ulonglong2* heap;   // n_slots x n
  uint32_t* stamp;    // n_slots x n
  uint64_t n;
  uint32_t n_slots;
  uint32_t* next;     // the next spill-list entry to take
};

__device__ __forceinline__ bool heap_less(ulonglong2 a, ulonglong2 b) { return a.x < b.x || (a.x == b.x && a.y < b.y); }
// adds v to the heap of hn entries (the caller counts it)
__device__ __forceinline__ void heap_push(ulonglong2* hp, uint32_t hn, ulonglong2 v) {
  uint32_t i = hn;
  while (i) {
    const uint32_t p = (i - 1) >> 1;
    const ulonglong2 pv = hp[p];
    if (!heap_less(v, pv)) break;
    hp[i] = pv;
    i = p;
  }
  hp[i] = v;
}
// removes and returns the smallest entry; hn = the number of entries left (the caller has counted the removal)
__device__ __forceinline__ ulonglong2 heap_pop(ulonglong2* hp, uint32_t hn) {
  const ulonglong2 top = hp[0];
  const ulonglong2 last = hp[hn];
  uint32_t i = 0;
  for (;;) {
    uint32_t c = 2 * i + 1;
    if (c >= hn) break;
    ulonglong2 cv = hp[c];
    if (c + 1 < hn) {
      const ulonglong2 rv = hp[c + 1];
      if (heap_less(rv, cv)) cv = rv, c++;
    }
    if (!heap_less(cv, last)) break;
    hp[i] = cv;
    i = c;
  }
  if (hn) hp[i] = last;
  return top;
}

// The same walk as hnsw_search_kernel<MET, .., T, true> (layer 0 filtered by the query's bitmap, the descent above
// unfiltered), for the queries of P.spill_list: each warp takes the next one until the list is done.  The cancel word is
// polled per query and every 32 expansions, since one walk may cover the whole reachable layer 0.
template <int MET, typename T>
__global__ void __launch_bounds__(HN_WARPS * 32, 1) hnsw_spill_kernel(HnswParams P, SpillSlots S, uint32_t per_warp) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t slot = blockIdx.x * HN_WARPS + warp;
  if (slot >= S.n_slots) return;
  float* s_q;
  float(*tile)[33];
  uint8_t* rest;
  hn_warp_layout<MET, T>(smem_raw + (size_t)warp * per_warp, P.dim, s_q, tile, rest);
  const uint32_t wcap = P.ef + 2;
  uint64_t* w_key = reinterpret_cast<uint64_t*>(rest);
  uint32_t* w_id = reinterpret_cast<uint32_t*>(w_key + wcap);
  ulonglong2* hp = S.heap + slot * S.n;
  uint32_t* stamp = S.stamp + slot * S.n;
  const volatile int* cancel = reinterpret_cast<const volatile int*>(P.cancel);
  const uint32_t n_spill = *P.n_spill;
  uint32_t gen = 0;
  // lane 0 reads the cancel word for the warp, so that every lane takes the same branch
  auto cancelled = [&]() { return __shfl_sync(0xffffffffu, lane == 0 ? *cancel : 0, 0) != 0; };
  for (;;) {
    uint32_t i = 0;
    if (lane == 0) i = atomicAdd(S.next, 1u);
    i = __shfl_sync(0xffffffffu, i, 0);
    if (i >= n_spill || cancelled()) break;
    const uint32_t q = P.spill_list[i];
    double q_norm = 0.0;
    MetricQ mq;
    stage_vector<MET, T>(P.dim, P.queries, P.q_norm, P.q_mean, P.q_sx2, P.q_bits, P.q_nbits, P.mink_p, q, s_q, q_norm, mq);
    const uint32_t* qbits = query_bits(P, q);
    uint64_t n_visited = 0, n_expanded = 0;
    uint32_t n_out = 0;
    bool stop = false;
    if (P.entry >= 0) {
      uint32_t ep = (uint32_t)P.entry;
      double ep_d = walk_distance<MET, T>(P, lane == 0 ? ep : NO_ROW, s_q, q_norm, mq, tile);
      ep_d = __shfl_sync(0xffffffffu, ep_d, 0);
      n_visited++;
      for (int32_t layer = (int32_t)P.n_layers - 1; layer >= 0; layer--) {
        const uint32_t ef = layer == 0 ? P.ef : 1u;
        const uint64_t* rp = P.rp[layer];
        const uint32_t* ci = P.ci[layer];
        if (++gen == 0) {  // the generations wrapped: forget every stamp
          for (uint64_t e = lane; e < S.n; e += 32) stamp[e] = 0;
          gen = 1;
        }
        __syncwarp();
        // search_single(_with_filter): visited = {ep}; candidates = {(ep_d, ep)}; w = {(ep_d, ep)} if ep passes
        uint32_t wn = 0;
        if (lane == 0) {
          stamp[ep] = gen;
          heap_push(hp, 0, make_ulonglong2(walk_key(ep_d), ep));
        }
        uint32_t hn = 1, seq = 1;  // heap entries, insertions so far
        __syncwarp();
        double fd = 1.7976931348623157e308;
        if (layer != 0 || filter_bit(qbits, ep)) {
          wn = sorted_insert(w_key, w_id, 0, wn, walk_key(ep_d), ep);
          fd = ep_d;
        }
        while (hn) {
          hn--;
          ulonglong2 top = make_ulonglong2(0, 0);
          if (lane == 0) top = heap_pop(hp, hn);
          const uint64_t ckey = __shfl_sync(0xffffffffu, top.x, 0);
          const uint32_t cid = (uint32_t)__shfl_sync(0xffffffffu, top.y, 0);
          if (key_to_double(ckey) > fd) break;  // cq_dist > fq_dist
          n_expanded++;
          if ((n_expanded & 31) == 0 && cancelled()) {
            stop = true;
            break;
          }
          const uint64_t beg = rp[cid], end = rp[cid + 1];
          for (uint64_t b0 = beg; b0 < end; b0 += 32) {
            const uint32_t nb = b0 + lane < end ? __ldg(ci + b0 + lane) : NO_ROW;
            // visited.insert in stored order: of repeats inside the chunk only the first can be new
            const uint32_t dup = __match_any_sync(0xffffffffu, nb);
            bool is_new = false;
            if (nb != NO_ROW && (dup & ((1u << lane) - 1u)) == 0 && stamp[nb] != gen) {
              stamp[nb] = gen;
              is_new = true;
            }
            __syncwarp();  // the stamps are seen by every lane of the next chunk
            const uint32_t new_mask = __ballot_sync(0xffffffffu, is_new);
            if (!new_mask) continue;
            n_visited += __popc(new_mask);
            const double d = walk_distance<MET, T>(P, is_new ? nb : NO_ROW, s_q, q_norm, mq, tile);
            uint32_t m = new_mask;
            while (m) {  // admission in stored order                      layer.rs:205-217,277-306
              const int j = __ffs(m) - 1;
              m &= m - 1;
              const double dj = __shfl_sync(0xffffffffu, d, j);
              const uint32_t idj = __shfl_sync(0xffffffffu, nb, j);
              if (dj < fd || wn < ef) {
                const uint64_t key = walk_key(dj);
                if (lane == 0) heap_push(hp, hn, make_ulonglong2(key, ((uint64_t)seq << 32) | idj));
                hn++, seq++;
                if (layer != 0 || filter_bit(qbits, idj)) {
                  wn = sorted_insert(w_key, w_id, 0, wn, key, idj);
                  if (wn > ef) wn--;  // pop_last
                  fd = key_to_double(w_key[wn - 1]);
                }
              }
            }
          }
        }
        __syncwarp();
        if (stop) break;
        if (wn) {
          ep = w_id[0];
          ep_d = key_to_double(w_key[0]);
        }
        if (layer == 0) {
          n_out = wn < P.k ? wn : P.k;
          for (uint32_t o = lane; o < n_out; o += 32) {
            P.out_elems[(size_t)q * P.k + o] = w_id[o];
            P.out_dist[(size_t)q * P.k + o] = key_to_double(w_key[o]);
          }
        }
        __syncwarp();
      }
    }
    if (stop) break;  // cancelled: the caller reports SDB_ECANCELLED
    if (lane == 0) {
      P.out_count[q] = n_out;
      if (P.out_counters) {
        P.out_counters[2 * (size_t)q] = n_visited;
        P.out_counters[2 * (size_t)q + 1] = n_expanded;
      }
    }
  }
}

// ---- exact kNN over the elements in the walk's arithmetic (TestCollection::knn, idx/trees/hnsw/mod.rs:1186-1197) ----
// For every query q: d = calculate(element, q) for every member element (the walk's argument order and distance code,
// so a distance equals the one sdb_hnsw_search reports for that pair), and the k smallest in (key, element id) order,
// the order of KnnResultBuilder.  One warp per query streams the members 32 at a time through walk_distance and keeps
// a sorted top-k in shared memory.  members: ascending element ids (null: every element); ties then stay in id order,
// because sorted_insert puts a new entry after its equals and a tie of the k-th entry is not admitted.
template <int MET, typename T>
__global__ void __launch_bounds__(HN_WARPS * 32, 1) hnsw_knn_exact_kernel(HnswParams P, const uint32_t* __restrict__ members,
                                                                       uint64_t n_members, uint32_t per_warp) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t k = P.k;
  float* s_q;
  float(*tile)[33];
  uint8_t* rest;
  hn_warp_layout<MET, T>(smem_raw + (size_t)warp * per_warp, P.dim, s_q, tile, rest);
  uint64_t* w_key = reinterpret_cast<uint64_t*>(rest);
  uint32_t* w_id = reinterpret_cast<uint32_t*>(w_key + k + 1);
  const uint32_t gwarp = blockIdx.x * HN_WARPS + warp, n_warps = gridDim.x * HN_WARPS;
  for (uint32_t q = gwarp; q < P.nq; q += n_warps) {
    double q_norm = 0.0;
    MetricQ mq;
    stage_vector<MET, T>(P.dim, P.queries, P.q_norm, P.q_mean, P.q_sx2, P.q_bits, P.q_nbits, P.mink_p, q, s_q, q_norm, mq);
    uint32_t wn = 0;
    for (uint64_t b0 = 0; b0 < n_members; b0 += 32) {
      const uint64_t i = b0 + lane;
      const uint32_t row = i < n_members ? (members ? __ldg(members + i) : (uint32_t)i) : NO_ROW;
      const double d = walk_distance<MET, T>(P, row, s_q, q_norm, mq, tile);
      const uint64_t key = walk_key(d);
      uint32_t m = __ballot_sync(0xffffffffu, row != NO_ROW && (wn < k || key < w_key[k - 1]));
      while (m) {  // in member order: the admission of a later lane sees the earlier ones
        const int j = __ffs(m) - 1;
        m &= m - 1;
        const uint64_t kj = __shfl_sync(0xffffffffu, key, j);
        const uint32_t idj = __shfl_sync(0xffffffffu, row, j);
        if (wn == k) {
          if (kj >= w_key[k - 1]) continue;
          wn--;  // the farthest leaves
        }
        wn = sorted_insert(w_key, w_id, 0, wn, kj, idj);
      }
    }
    for (uint32_t i = lane; i < wn; i += 32) {
      P.out_elems[(size_t)q * k + i] = w_id[i];
      P.out_dist[(size_t)q * k + i] = key_to_double(w_key[i]);
    }
    if (lane == 0) P.out_count[q] = wn;
    __syncwarp();
  }
}

// ---- Heuristic::select in the walk's arithmetic (standard variant, heuristic.rs:61-81,201-216), one warp per element.
// Every distance is walk_distance with one vector staged as the walk stages a query, so each is the distance the walk
// would compute for the pair, in the reference's argument order:
//   e_dist, presorted: calculate(candidate, element) -- the distance the candidate list was ranked by (an insertion
//     search or the exact kNN above, both element-first with the new element as the query);
//   e_dist, re-sort (build_priority_list, layer.rs:389-405): calculate(element, candidate), the visiting order then by
//     (key, list position), i.e. FIFO among equal distances;
//   r_dist = calculate(r, e) for every accepted r (elements.rs:133-140), with e staged.
// Only JACCARD is asymmetric; its re-sort e_dist swaps the two counts of the same intersection.  e is rejected when
// e_dist > r_dist for some accepted r; all candidates (other than the element) are taken when there are <= m_max.
// Shared memory per warp: the staged vector and scratch, then kc f64 e_dist, kc u32 visiting order, m_max u32 picks.
template <int MET, typename T>
__global__ void __launch_bounds__(HN_WARPS * 32, 1) hnsw_select_typed_kernel(HnswParams P, const uint32_t* __restrict__ elem_ids,
                                                                          uint64_t row0, uint64_t n,
                                                                          const uint64_t* __restrict__ cand,
                                                                          const uint32_t* __restrict__ cand_cnt, uint32_t kc,
                                                                          uint32_t m_max, int presorted,
                                                                          uint32_t* __restrict__ out,
                                                                          uint32_t* __restrict__ out_cnt, uint32_t per_warp) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* s_q;
  float(*tile)[33];
  uint8_t* rest;
  hn_warp_layout<MET, T>(smem_raw + (size_t)warp * per_warp, P.dim, s_q, tile, rest);
  double* s_ed = reinterpret_cast<double*>(rest);
  uint32_t* s_ord = reinterpret_cast<uint32_t*>(s_ed + kc);
  uint32_t* s_acc = s_ord + kc;
  const uint64_t n_warps = (uint64_t)gridDim.x * HN_WARPS;
  for (uint64_t i = (uint64_t)blockIdx.x * HN_WARPS + warp; i < n; i += n_warps) {
    const uint64_t self = elem_ids ? (uint64_t)elem_ids[i] : row0 + i;
    const uint64_t* cl = cand + i * kc;
    const uint32_t nc = cand_cnt[i] < kc ? cand_cnt[i] : kc;
    uint32_t n_real = 0;  // candidates other than the element itself
    for (uint32_t j = lane; j < nc; j += 32) n_real += cl[j] != self;
    n_real = __reduce_add_sync(0xffffffffu, n_real);
    const bool take_all = n_real <= m_max;
    double q_norm = 0.0;
    MetricQ mq;
    if (!(presorted && take_all)) {  // e_dist of every candidate, the element staged
      stage_vector<MET, T>(P.dim, P.vec, P.norm, P.e_mean, P.e_sx2, P.e_bits, P.e_nbits, P.mink_p, self, s_q, q_norm, mq);
      for (uint32_t j0 = 0; j0 < nc; j0 += 32) {
        const uint32_t j = j0 + lane;
        const uint32_t row = j < nc && cl[j] != self ? (uint32_t)cl[j] : NO_ROW;
        double d;
        if constexpr (MET == SDB_JACCARD)
          d = presorted ? walk_distance<MET, T>(P, row, s_q, q_norm, mq, tile)
                        : warp_distance_jaccard<T, true>(static_cast<const JKey<T>*>(P.e_bits), P.e_nbits, P.dim, row,
                                                         reinterpret_cast<const JKey<T>*>(s_q), mq.u, tile);
        else
          d = walk_distance<MET, T>(P, row, s_q, q_norm, mq, tile);
        if (j < nc) s_ed[j] = d;
      }
      __syncwarp();
    }
    // visiting order: as given, or by (key of e_dist, position); the element itself goes last (it is skipped)
    if (presorted) {
      for (uint32_t j = lane; j < nc; j += 32) s_ord[j] = j;
    } else {
      for (uint32_t j = lane; j < nc; j += 32) {
        const bool sj = cl[j] == self;
        const uint64_t kj = walk_key(s_ed[j]);
        uint32_t rank = 0;
        for (uint32_t t = 0; t < nc; t++) {
          const bool st = cl[t] == self;
          const uint64_t kt = walk_key(s_ed[t]);
          rank += st == sj ? (kt < kj || (kt == kj && t < j)) : (uint32_t)sj;
        }
        s_ord[rank] = j;
      }
    }
    __syncwarp();
    uint32_t acc = 0;
    for (uint32_t jj = 0; jj < nc && acc < m_max; jj++) {
      const uint32_t j = s_ord[jj];
      const uint64_t e = cl[j];
      if (e == self) continue;
      bool ok = true;
      if (!take_all) {
        const double e_dist = s_ed[j];
        stage_vector<MET, T>(P.dim, P.vec, P.norm, P.e_mean, P.e_sx2, P.e_bits, P.e_nbits, P.mink_p, e, s_q, q_norm, mq);
        for (uint32_t r0 = 0; r0 < acc && ok; r0 += 32) {
          const uint32_t row = r0 + lane < acc ? s_acc[r0 + lane] : NO_ROW;
          const double r_dist = walk_distance<MET, T>(P, row, s_q, q_norm, mq, tile);
          ok = !__any_sync(0xffffffffu, row != NO_ROW && e_dist > r_dist);  // is_closer: heuristic.rs:209-211
        }
      }
      if (ok) {
        if (lane == 0) s_acc[acc] = (uint32_t)e;
        acc++;
        __syncwarp();
      }
    }
    for (uint32_t a = lane; a < acc; a += 32) out[i * m_max + a] = s_acc[a];
    if (lane == 0) out_cnt[i] = acc;
    __syncwarp();
  }
}

// ---- construction helper: Heuristic::select over pre-ranked candidates, one warp per element ------------------------
// The F32 COSINE / EUCLIDEAN GPU builder's selection (fmaf, f32, squared euclidean), kept as it is so that the graphs that
// builder makes do not change; every other metric and type selects with hnsw_select_typed_kernel above.
template <bool COSINE>
__device__ __forceinline__ float warp_pair_dist(const float* a_smem, float a_n2, const float* __restrict__ b, uint32_t dim) {
  const uint32_t lane = threadIdx.x & 31u;
  float dot = 0.f, n2 = 0.f;
  for (uint32_t c = lane; c < dim; c += 32) {
    const float x = a_smem[c], y = __ldg(b + c);
    if (COSINE) {
      dot = fmaf(x, y, dot);
      n2 = fmaf(y, y, n2);
    } else {
      const float d = x - y;
      dot = fmaf(d, d, dot);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (COSINE) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
  }
  return COSINE ? 1.f - dot * rsqrtf(a_n2 * n2) : dot;  // euclid: squared distance (same ordering)
}

template <bool COSINE>
__global__ void __launch_bounds__(128) hnsw_select_kernel(const float* __restrict__ vec, uint32_t dim, uint64_t row0, uint64_t n,
                                                          const uint32_t* __restrict__ elem_ids,
                                                          const uint64_t* __restrict__ cand, const uint32_t* __restrict__ cand_cnt,
                                                          uint32_t kc, uint32_t m_max, int presorted, uint32_t* __restrict__ out,
                                                          uint32_t* __restrict__ out_cnt) {
  extern __shared__ float s_sel[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* s_q = s_sel + (size_t)warp * (2 * dim + 2 * kc);
  float* s_e = s_q + dim;
  float* s_d = s_e + dim;                                   // [kc] distances (unsorted mode)
  uint32_t* s_ord = reinterpret_cast<uint32_t*>(s_d + kc);  // [kc] visiting order
  const uint64_t i = (uint64_t)blockIdx.x * 4 + warp;  // element index inside this batch
  if (i >= n) return;
  const uint64_t self = elem_ids ? (uint64_t)elem_ids[i] : row0 + i;
  const float* q = vec + self * dim;
  float qn2 = 0.f;
  for (uint32_t c = lane; c < dim; c += 32) {
    const float x = __ldg(q + c);
    s_q[c] = x;
    qn2 = fmaf(x, x, qn2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) qn2 += __shfl_xor_sync(0xffffffffu, qn2, o);
  __syncwarp();
  const uint64_t* cl = cand + i * kc;
  uint32_t nc = cand_cnt[i] < kc ? cand_cnt[i] : kc;
  uint32_t n_real = 0;  // candidates other than the element itself
  for (uint32_t j = 0; j < nc; j++) n_real += cl[j] != self;
  // visiting order: as given (nearest first) or by computed distance (build_priority_list, layer.rs:389-405)
  if (presorted) {
    for (uint32_t j = lane; j < nc; j += 32) s_ord[j] = j;
  } else {
    for (uint32_t j = 0; j < nc; j++) {
      const float d = cl[j] == self ? 3.0e38f : warp_pair_dist<COSINE>(s_q, qn2, vec + cl[j] * dim, dim);
      if (lane == 0) s_d[j] = d;
    }
    __syncwarp();
    // a total order, so that the ranks are a permutation: numbers by value, equal ones in list order; NaN (a zero
    // row under cosine, a NaN or inf element) after every number and the self marker, NaNs in list order
    for (uint32_t j = lane; j < nc; j += 32) {
      const float dj = s_d[j];
      const bool nj = dj != dj;
      uint32_t rank = 0;
      for (uint32_t t = 0; t < nc; t++) {
        const float dt = s_d[t];
        rank += (dt != dt) != nj ? nj : (dt < dj || ((dt == dj || nj) && t < j));
      }
      s_ord[rank] = j;
    }
  }
  __syncwarp();
  uint32_t* o = out + i * m_max;
  uint32_t acc = 0;
  const bool take_all = n_real <= m_max;
  for (uint32_t jj = 0; jj < nc && acc < m_max; jj++) {
    const uint32_t j = s_ord[jj];
    const uint64_t e = cl[j];
    if (e == self) continue;
    bool ok = true;
    if (!take_all) {
      const float* ev = vec + e * dim;
      float en2 = 0.f;
      for (uint32_t c = lane; c < dim; c += 32) {
        const float x = __ldg(ev + c);
        s_e[c] = x;
        en2 = fmaf(x, x, en2);
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) en2 += __shfl_xor_sync(0xffffffffu, en2, o2);
      __syncwarp();
      const float e_dist = warp_pair_dist<COSINE>(s_q, qn2, ev, dim);
      for (uint32_t r = 0; r < acc && ok; r++) {
        const float r_dist = warp_pair_dist<COSINE>(s_e, en2, vec + (uint64_t)o[r] * dim, dim);
        if (e_dist > r_dist) ok = false;  // is_closer: heuristic.rs:209-211
      }
      __syncwarp();
    }
    if (ok) {
      if (lane == 0) o[acc] = (uint32_t)e;
      acc++;
      __syncwarp();
    }
  }
  if (lane == 0) out_cnt[i] = acc;
}

// ---- load-time validation (ADVICE r1): adjacency supplied across the ABI is used for device indexing, so it is
// range-checked once here instead of trusted.  bad[0] counts row_ptr violations (non-monotone / beyond the edge count),
// bad[1] counts neighbour ids >= n_elems.
__global__ void csr_validate_kernel(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ ci, uint64_t n_rows,
                                    uint64_t n_edges, uint64_t id_limit, unsigned long long* __restrict__ bad) {
  const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t t0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (uint64_t r = t0; r < n_rows; r += step)
    if (rp[r] > rp[r + 1] || rp[r + 1] > n_edges) atomicAdd(bad, 1ull);
  if (t0 == 0 && n_rows && rp[0] != 0) atomicAdd(bad, 1ull);
  for (uint64_t e = t0; e < n_edges; e += step)
    if ((uint64_t)ci[e] >= id_limit) atomicAdd(bad + 1, 1ull);
}

sdb_status csr_check(Ctx* ctx, const uint64_t* d_rp, const uint32_t* d_ci, uint64_t n_rows, uint64_t n_edges,
                     uint64_t id_limit, unsigned long long counts[2], const char* what, cudaStream_t st) {
  AsyncBuf<unsigned long long> d_bad;
  SDB_CUDA(d_bad.reserve(2, st));
  cudaMemsetAsync(d_bad, 0, 16, st);
  const uint64_t work = n_rows > n_edges ? n_rows : n_edges;
  const unsigned grid = (unsigned)std::min<uint64_t>((work + 255) / 256 + 1, (uint64_t)ctx->sm_count * 16);
  csr_validate_kernel<<<grid, 256, 0, st>>>(d_rp, d_ci, n_rows, n_edges, id_limit, d_bad);
  count_launch(ctx);
  unsigned long long h_bad[2] = {0, 0};
  cudaError_t e = cudaMemcpyAsync(h_bad, d_bad, 16, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  d_bad.reset();
  if (e != cudaSuccess) {
    set_error("%s: validation failed to run: %s", what, cudaGetErrorString(e));
    return SDB_ECUDA;
  }
  counts[0] = h_bad[0];
  counts[1] = h_bad[1];
  return SDB_OK;
}
sdb_status csr_validate(Ctx* ctx, const uint64_t* d_rp, const uint32_t* d_ci, uint64_t n_rows, uint64_t n_edges,
                        uint64_t id_limit, const char* what, cudaStream_t st) {
  unsigned long long h_bad[2] = {0, 0};
  SDB_TRY(csr_check(ctx, d_rp, d_ci, n_rows, n_edges, id_limit, h_bad, what, st));
  if (h_bad[0] || h_bad[1]) {
    set_error("%s: malformed CSR (%llu row_ptr violations, %llu neighbour ids out of range)", what, h_bad[0], h_bad[1]);
    return SDB_EINVAL;
  }
  return SDB_OK;
}

// ---- edges to elements without a vector: the reference marks such a neighbour visited and computes nothing
// (elements.get_vector -> None, hnsw/layer.rs:204), which is equivalent to the edge not being there.  Staged loads
// therefore drop them from the device CSR: count, scan, fill.
__global__ void csr_present_degree_kernel(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ ci,
                                          const uint8_t* __restrict__ present, uint64_t n_rows,
                                          uint64_t* __restrict__ deg) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_rows) return;
  uint64_t d = 0;
  if (r < n_rows && present[r])  // an absent element is never expanded either
    for (uint64_t e = rp[r]; e < rp[r + 1]; e++) d += present[ci[e]] ? 1 : 0;
  deg[r] = d;  // deg[n_rows] = 0: the scan's total
}
__global__ void csr_present_fill_kernel(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ ci,
                                        const uint8_t* __restrict__ present, uint64_t n_rows,
                                        const uint64_t* __restrict__ rp2, uint32_t* __restrict__ ci2) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows || !present[r]) return;
  uint64_t o = rp2[r];
  for (uint64_t e = rp[r]; e < rp[r + 1]; e++) {
    const uint32_t v = ci[e];
    if (present[v]) ci2[o++] = v;  // stored order kept
  }
}

// The visited tables of the walks queued on one stream (one table per resident warp) and their generation counter.
// Each of the context's two streams has its own set, so a re-size or a generation wrap is ordered after the walks
// already queued on that set by the stream itself: the table is an AsyncBuf of that stream, freed there.
struct VisitSet {
  AsyncBuf<uint64_t> tab;
  uint32_t table_log2 = 0, n_tables = 0;
  uint32_t gen = 1;  // generations consumed so far (each warp uses gen_base + its own counter)
};

// One search between the two halves of the walk driver (hnsw_enqueue, hnsw_complete): an asynchronous ticket of
// sdb_hnsw_submit* or a blocking call.  It owns everything the completion half still reads: the staged queries and
// their metric state, the staged bitmaps or pending mask, the copied query_filter, the device outputs of the host
// variants, the counters, the spill list and the spill tier's slots.
struct HnswTicket {
  bool busy = false;
  bool waiting = false;  // a sdb_hnsw_wait has taken it
  uint32_t id = 0;
  cudaStream_t st = nullptr;
  VisitSet* vis = nullptr;  // the visited-table set of st
  HnswParams P{};
  bool walked = false;      // the walk was launched (false: an empty batch)
  bool batch_filter = false;
  bool device_io = false;
  uint32_t nq = 0, k = 0;
  uint64_t* out_elems = nullptr;  // the caller's outputs
  double* out_dist = nullptr;
  uint32_t* out_count = nullptr;
  uint64_t* out_counters = nullptr;
  uint32_t* h_word = nullptr;  // pinned, 2 words: [0] the spill count, [1] the overflow flag, copied after the walk
  cudaEvent_t ev = nullptr;    // the last work of the search queued so far
  AsyncBuf<char> q_buf;
  AsyncBuf<uint64_t> elems_buf, d_ctr;
  AsyncBuf<double> dist_buf;
  AsyncBuf<uint32_t> cnt_buf, d_ovf;
  AsyncBuf<uint8_t> d_noexp, d_truthy;
  AsyncBuf<uint32_t> d_filters, d_qf, d_spill;
  VecState<Mem::Async> qs;
  std::vector<uint32_t> h_qf;  // the caller's query_filter, copied at submit
  DevBuf<ulonglong2> spill_heap;
  DevBuf<uint32_t> spill_stamp;
  AsyncBuf<uint32_t> spill_next;
  // frees the per-search buffers (the AsyncBufs on the stream, after the search's own work) and frees the slot
  void release() {
    q_buf.reset(), elems_buf.reset(), d_ctr.reset(), dist_buf.reset(), cnt_buf.reset(), d_ovf.reset();
    d_noexp.reset(), d_truthy.reset(), d_filters.reset(), d_qf.reset(), d_spill.reset();
    qs = VecState<Mem::Async>();
    h_qf = std::vector<uint32_t>();
    spill_heap.reset(), spill_stamp.reset(), spill_next.reset();
    busy = waiting = walked = false;
  }
  ~HnswTicket() {
    if (ev) cudaEventDestroy(ev);
  }
};

struct Hnsw {
  Ctx* ctx = nullptr;
  uint32_t dim = 0;
  sdb_metric metric = SDB_EUCLIDEAN;
  sdb_vector_type vt = SDB_VT_F32;  // element type of the vectors (and of the queries a search takes)
  uint64_t n = 0;
  uint32_t n_layers = 0;
  int64_t entry = -1;
  void* d_vec = nullptr;     // n x dim elements of type vt (own_vec's, or the caller's for a borrowed handle)
  double minkowski_p = 3.0;  // order of SDB_MINKOWSKI (sdb_hnsw_set_minkowski_order)
  VecState<Mem::Device> elems;  // the elements' metric state
  std::vector<uint64_t*> rp;    // per layer CSR (own_rp / own_ci's, or the caller's for a borrowed handle)
  std::vector<uint32_t*> ci;
  DevBuf<char> own_vec;         // empty for a borrowed handle
  std::vector<DevBuf<uint64_t>> own_rp;
  std::vector<DevBuf<uint32_t>> own_ci;
  DevBuf<const uint64_t*> d_rp;  // device tables of the rp / ci pointers
  DevBuf<const uint32_t*> d_ci;
  VisitSet vis[2];             // the walks of the context's stream / stream2
  uint32_t last_spilled = 0;  // queries of the last batch-filtered call (or waited ticket) that the spill tier finished
  // slots 0 .. N_TICKETS - 1: the asynchronous tickets (even slots on the context's stream, odd ones on stream2);
  // slot N_TICKETS: the blocking calls, which hold `mu` from their enqueue to their completion
  HnswTicket slots[N_TICKETS + 1];
  PinnedBuf<uint32_t> h_words;  // 2 words per slot (HnswTicket::h_word), allocated with the first search
  uint32_t next_ticket = 1;
  bool borrowed = false;  // sdb_hnsw_load_device: vectors and CSR arrays belong to the caller
  std::mutex mu;
};

}  // namespace sdb

struct sdb_hnsw : sdb::Hnsw {};
using namespace sdb;

extern "C" void sdb_hnsw_destroy(sdb_hnsw* h);

static size_t vt_size(sdb_vector_type vt) { return vt == SDB_VT_F64 || vt == SDB_VT_I64 ? 8 : vt == SDB_VT_I16 ? 2 : 4; }
static size_t jkey_size(sdb_vector_type vt) { return vt == SDB_VT_F64 || vt == SDB_VT_I64 ? 8 : 4; }
// calls f(T()) with the C++ element type of vt
template <typename F>
static auto with_vt(sdb_vector_type vt, F&& f) {
  switch (vt) {
    case SDB_VT_F64: return f(double());
    case SDB_VT_I64: return f((long long)0);
    case SDB_VT_I32: return f(int());
    case SDB_VT_I16: return f(short());
    default: return f(float());
  }
}
// calls f(std::integral_constant<int, MET>()) with the metric as a compile-time constant
template <typename F>
static auto with_metric(sdb_metric metric, F&& f) {
  switch (metric) {
    case SDB_CHEBYSHEV: return f(std::integral_constant<int, SDB_CHEBYSHEV>());
    case SDB_COSINE: return f(std::integral_constant<int, SDB_COSINE>());
    case SDB_HAMMING: return f(std::integral_constant<int, SDB_HAMMING>());
    case SDB_JACCARD: return f(std::integral_constant<int, SDB_JACCARD>());
    case SDB_MANHATTAN: return f(std::integral_constant<int, SDB_MANHATTAN>());
    case SDB_MINKOWSKI: return f(std::integral_constant<int, SDB_MINKOWSKI>());
    case SDB_PEARSON: return f(std::integral_constant<int, SDB_PEARSON>());
    default: return f(std::integral_constant<int, SDB_EUCLIDEAN>());
  }
}
// The checks every loader shares, after its own pointer checks: the shape of the index, then the refusals of an
// unknown metric or type and of I16 PEARSON beyond the reference's i16 divisor.
static sdb_status check_load(const char* what, sdb_ctx* ctx, sdb_hnsw** out, uint32_t dim, sdb_metric metric, int vt,
                             uint64_t n_elems, uint32_t n_layers, int64_t entry_point) {
  if (!ctx || !out || dim == 0 || dim > 65535 || n_elems >= 0xFFFFFFF0ull || !n_layers || entry_point >= (int64_t)n_elems)
    return SDB_EINVAL;
  if ((unsigned)metric > SDB_PEARSON) {
    set_error("hnsw: unknown metric %d", (int)metric);
    return SDB_EUNSUPPORTED;
  }
  if ((unsigned)vt > SDB_VT_I16) {
    set_error("%s: unknown vector type %d", what, vt);
    return SDB_EINVAL;
  }
  if (vt == SDB_VT_I16 && metric == SDB_PEARSON && dim > 32767) {  // A::from_usize(n) fails: the reference panics
    set_error("%s: an I16 PEARSON index of dimension %u cannot be searched (the mean's divisor does not fit i16)", what, dim);
    return SDB_EUNSUPPORTED;
  }
  *out = nullptr;
  return SDB_OK;
}

// a handle with the index's shape; the loader adds the vectors and the adjacency, hnsw_finish the rest
static sdb_hnsw* new_hnsw(Ctx* ctx, uint32_t dim, sdb_metric metric, sdb_vector_type vt, uint64_t n, uint32_t n_layers,
                          int64_t entry) {
  sdb_hnsw* h = new sdb_hnsw();
  h->ctx = ctx;
  h->dim = dim;
  h->metric = metric;
  h->vt = vt;
  h->n = n;
  h->n_layers = n_layers;
  h->entry = entry;
  return h;
}

// The state `metric` needs for rows x dim vectors d_v of type vt, allocated into s and computed on st: COSINE the norms
// (none for an F32 batch: the walk computes the query's own, typed_distance_kernel both), PEARSON the mean and sx2,
// JACCARD the sorted distinct keys.
template <Mem K>
static sdb_status vec_state_make(Ctx* ctx, sdb_metric metric, sdb_vector_type vt, const void* d_v, uint64_t rows,
                                 uint32_t dim, VecState<K>& s, cudaStream_t st) {
  if (!rows) return SDB_OK;
  cudaError_t e = cudaSuccess;
  auto oom = [&](const char* what, size_t bytes) {
    set_error("hnsw: %s (%zu bytes) could not be allocated: %s", what, bytes, cudaGetErrorString(e));
    return K == Mem::Async ? SDB_ECUDA : SDB_ENOMEM;
  };
  const unsigned grid = (unsigned)((rows + 127) / 128);
  if (metric == SDB_COSINE && !(vt == SDB_VT_F32 && K == Mem::Async)) {
    if ((e = s.norm.reserve(rows, st)) != cudaSuccess) return oom("cosine norms", sizeof(double) * rows);
    with_vt(vt, [&](auto tag) {
      using T = decltype(tag);
      if constexpr (is_f32_v<T>)
        hnsw_norm_f32_kernel<<<(unsigned)((rows * 8 + 127) / 128), 128, 0, st>>>(static_cast<const float*>(d_v), dim,
                                                                                  rows, s.norm);
      else
        hnsw_norm_kernel<T><<<grid, 128, 0, st>>>(static_cast<const T*>(d_v), dim, rows, s.norm);
    });
    count_launch(ctx);
  } else if (metric == SDB_PEARSON) {
    if ((e = s.mean.reserve(rows, st)) != cudaSuccess || (e = s.sx2.reserve(rows, st)) != cudaSuccess)
      return oom("pearson state", 2 * sizeof(double) * rows);
    with_vt(vt, [&](auto tag) {
      using T = decltype(tag);
      pearson_stats_kernel<T><<<grid, 128, 0, st>>>(static_cast<const T*>(d_v), dim, rows, s.mean, s.sx2);
    });
    count_launch(ctx);
  } else if (metric == SDB_JACCARD) {  // key bytes * rows * dim: the sorted distinct keys of every vector
    const size_t kb = jkey_size(vt) * rows * dim;
    if ((e = s.bits.reserve(kb, st)) != cudaSuccess || (e = s.nbits.reserve(rows, st)) != cudaSuccess)
      return oom("jaccard state", kb + sizeof(uint32_t) * rows);
    return jaccard_prepare_typed(ctx, vt, d_v, rows, dim, s.bits, s.nbits, st);
  }
  return SDB_OK;
}

// the device tables of per-layer CSR pointers (h->rp, h->ci), (re)allocated for h->n_layers; the copy is queued on st
static sdb_status upload_layer_tables(sdb_hnsw* h, cudaStream_t st) {
  const uint32_t n_layers = h->n_layers;
  h->d_rp.reset();
  h->d_ci.reset();
  cudaError_t e = h->d_rp.reserve(n_layers);
  if (e == cudaSuccess) e = h->d_ci.reserve(n_layers);
  if (e != cudaSuccess) {
    set_error("hnsw: layer table allocation failed: %s", cudaGetErrorString(e));
    return SDB_ENOMEM;
  }
  if (cudaMemcpyAsync(h->d_rp, h->rp.data(), sizeof(void*) * n_layers, cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(h->d_ci, h->ci.data(), sizeof(void*) * n_layers, cudaMemcpyHostToDevice, st) != cudaSuccess) {
    set_error("hnsw: layer table copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    return SDB_ECUDA;
  }
  return SDB_OK;
}

// common tail of the loaders: per-layer pointer tables + the elements' metric state
static sdb_status hnsw_finish(sdb_hnsw* h, sdb_hnsw** out) {
  Ctx* ctx = h->ctx;
  cudaStream_t st = ctx->stream;
  auto fail = [&](const char* what, sdb_status rc) {
    set_error("hnsw load: %s failed: %s", what, cudaGetErrorString(cudaGetLastError()));
    sdb_hnsw_destroy(h);
    return rc;
  };
  sdb_status rc = upload_layer_tables(h, st);
  if (rc != SDB_OK) {
    sdb_hnsw_destroy(h);
    return rc;
  }
  rc = vec_state_make(ctx, h->metric, h->vt, h->d_vec, h->n, h->dim, h->elems, st);
  if (rc != SDB_OK) {
    sdb_hnsw_destroy(h);
    return rc;
  }
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail("finish", SDB_ECUDA);
  *out = h;
  return SDB_OK;
}

// the element side of HnswParams: vectors, their metric state, the Minkowski order
static HnswParams element_params(const sdb_hnsw* h) {
  HnswParams P{};
  P.vec = h->d_vec;
  P.norm = h->elems.norm;
  P.dim = h->dim;
  P.mink_p = h->minkowski_p;
  P.e_mean = h->elems.mean;
  P.e_sx2 = h->elems.sx2;
  P.e_bits = h->elems.bits;
  P.e_nbits = h->elems.nbits;
  return P;
}

// launches kern (4 warps per block, `per_warp` bytes of shared memory each) with enough blocks for `items` warps, at most
// as many as are resident at once (the kernels loop)
template <typename K, typename... A>
static sdb_status launch_warps(Ctx* ctx, K kern, size_t per_warp, uint64_t items, const char* what, A... args) {
  per_warp = (per_warp + 15) & ~size_t(15);
  const size_t smem = per_warp * HN_WARPS;
  if (smem > 220 * 1024) {
    set_error("%s: %zu bytes of shared memory per block needed (dimension, k or candidate count too large)", what, smem);
    return SDB_EUNSUPPORTED;
  }
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  SDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, HN_WARPS * 32, smem));
  const uint64_t grid = std::min<uint64_t>((uint64_t)ctx->sm_count * std::max(per_sm, 1), (items + HN_WARPS - 1) / HN_WARPS);
  kern<<<(unsigned)grid, HN_WARPS * 32, smem, ctx->stream>>>(args..., (uint32_t)per_warp);
  count_launch(ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

__global__ void members_max_kernel(const uint32_t* __restrict__ m, uint64_t n, unsigned int* __restrict__ mx) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicMax(mx, m[i]);
}

extern "C" {

void sdb_hnsw_destroy(sdb_hnsw* h) {
  if (!h) return;
  cudaSetDevice(h->ctx->device);
  for (const HnswTicket& t : h->slots)  // tickets never waited for: their work ends before their buffers go
    if (t.busy) cudaEventSynchronize(t.ev);
  delete h;
}

sdb_status sdb_hnsw_load(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, uint64_t n_elems, const float* vectors,
                         uint32_t n_layers, const uint64_t* const* row_ptr, const uint32_t* const* col_idx,
                         int64_t entry_point, sdb_hnsw** out) {
  return sdb_hnsw_load_typed(ctx, dim, metric, SDB_VT_F32, n_elems, vectors, n_layers, row_ptr, col_idx, entry_point, out);
}

sdb_status sdb_hnsw_load_typed(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, sdb_vector_type vt, uint64_t n_elems,
                               const void* vectors, uint32_t n_layers, const uint64_t* const* row_ptr,
                               const uint32_t* const* col_idx, int64_t entry_point, sdb_hnsw** out) {
  if ((n_elems && !vectors) || !row_ptr || !col_idx) return SDB_EINVAL;
  SDB_TRY(check_load("sdb_hnsw_load_typed", ctx, out, dim, metric, (int)vt, n_elems, n_layers, entry_point));
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  sdb_hnsw* h = new_hnsw(ctx, dim, metric, vt, n_elems, n_layers, entry_point);
  cudaStream_t st = ctx->stream;
  const sdb_status rc = [&]() -> sdb_status {
    auto fail = [&](const char* what, cudaError_t e) {
      set_error("hnsw load: %s failed: %s", what, cudaGetErrorString(e));
      return SDB_ENOMEM;
    };
    const uint64_t nn = n_elems ? n_elems : 1;
    const size_t esz = vt_size(vt);
    cudaError_t e = h->own_vec.reserve(esz * nn * dim);
    if (e != cudaSuccess) return fail("vectors", e);
    h->d_vec = h->own_vec;
    if (n_elems) SDB_CUDA(cudaMemcpyAsync(h->d_vec, vectors, esz * n_elems * dim, cudaMemcpyHostToDevice, st));
    for (uint32_t l = 0; l < n_layers; l++) {
      const uint64_t ne = n_elems ? row_ptr[l][n_elems] : 0;
      DevBuf<uint64_t> drp;
      DevBuf<uint32_t> dci;
      if ((e = drp.reserve(n_elems + 1)) != cudaSuccess) return fail("row_ptr", e);
      if ((e = dci.reserve(ne ? ne : 1)) != cudaSuccess) return fail("col_idx", e);
      h->rp.push_back(drp);
      h->ci.push_back(dci);
      h->own_rp.push_back(std::move(drp));
      h->own_ci.push_back(std::move(dci));
      SDB_CUDA(cudaMemcpyAsync(h->rp[l], row_ptr[l], sizeof(uint64_t) * (n_elems + 1), cudaMemcpyHostToDevice, st));
      if (ne) SDB_CUDA(cudaMemcpyAsync(h->ci[l], col_idx[l], sizeof(uint32_t) * ne, cudaMemcpyHostToDevice, st));
      SDB_TRY(csr_validate(ctx, h->rp[l], h->ci[l], n_elems, ne, n_elems, "sdb_hnsw_load", st));
    }
    return SDB_OK;
  }();
  if (rc != SDB_OK) {
    sdb_hnsw_destroy(h);
    return rc;
  }
  return hnsw_finish(h, out);
}

sdb_status sdb_hnsw_load_device(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, uint64_t n_elems, const float* d_vectors,
                                uint32_t n_layers, const uint64_t* const* d_row_ptr, const uint32_t* const* d_col_idx,
                                int64_t entry_point, sdb_hnsw** out) {
  return sdb_hnsw_load_device_typed(ctx, dim, metric, SDB_VT_F32, n_elems, d_vectors, n_layers, d_row_ptr, d_col_idx,
                                    entry_point, out);
}

sdb_status sdb_hnsw_load_device_typed(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, sdb_vector_type vt, uint64_t n_elems,
                                      const void* d_vectors, uint32_t n_layers, const uint64_t* const* d_row_ptr,
                                      const uint32_t* const* d_col_idx, int64_t entry_point, sdb_hnsw** out) {
  if ((n_elems && !d_vectors) || !d_row_ptr || !d_col_idx) return SDB_EINVAL;
  SDB_TRY(check_load("sdb_hnsw_load_device_typed", ctx, out, dim, metric, (int)vt, n_elems, n_layers, entry_point));
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  sdb_hnsw* h = new_hnsw(ctx, dim, metric, vt, n_elems, n_layers, entry_point);
  h->borrowed = true;  // nothing is copied: the caller keeps vectors and adjacency alive while the handle exists
  h->d_vec = const_cast<void*>(d_vectors);
  for (uint32_t l = 0; l < n_layers; l++) {
    h->rp.push_back(const_cast<uint64_t*>(d_row_ptr[l]));
    h->ci.push_back(const_cast<uint32_t*>(d_col_idx[l]));
  }
  return hnsw_finish(h, out);
}

sdb_status sdb_hnsw_set_layers_device(sdb_hnsw* h, uint32_t n_layers, const uint64_t* const* d_row_ptr,
                                      const uint32_t* const* d_col_idx, int64_t entry_point) {
  if (!h || !n_layers || !d_row_ptr || !d_col_idx || entry_point >= (int64_t)h->n) return SDB_EINVAL;
  if (!h->borrowed) {
    set_error("sdb_hnsw_set_layers_device: the handle owns its arrays (only a handle of sdb_hnsw_load_device[_typed] can "
              "swap its adjacency)");
    return SDB_EINVAL;
  }
  std::lock_guard<std::mutex> guard(h->mu);  // blocking searches hold it for their whole run
  for (const HnswTicket& t : h->slots)  // a ticket's spill tier reads the layers it was submitted against
    if (t.busy) {
      set_error("sdb_hnsw_set_layers_device: tickets in flight (call sdb_hnsw_wait first)");
      return SDB_EINVAL;
    }
  SDB_CUDA(cudaSetDevice(h->ctx->device));
  h->rp.clear();
  h->ci.clear();
  for (uint32_t l = 0; l < n_layers; l++) {
    h->rp.push_back(const_cast<uint64_t*>(d_row_ptr[l]));
    h->ci.push_back(const_cast<uint32_t*>(d_col_idx[l]));
  }
  h->n_layers = n_layers;
  h->entry = entry_point;
  SDB_TRY(upload_layer_tables(h, h->ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(h->ctx->stream));
  return SDB_OK;
}

// native < 0: sdb_hnsw_load_staged, an F32 index: He values of another variant are refused, F32 ones converted; otherwise
// sdb_hnsw_load_staged_typed, native = the variant number of the index's type: values are decoded as they are stored and
// any other variant counts as bad.
static sdb_status hnsw_load_staged_impl(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, sdb_vector_type vt, int native,
                                        uint64_t n_elems, const uint8_t* vec_blob, const uint64_t* vec_off,
                                        const uint64_t* vec_ids, uint64_t n_vec, uint32_t n_layers,
                                        const uint8_t* const* node_blob, const uint64_t* const* node_off,
                                        const uint64_t* const* node_ids, const uint64_t* n_nodes, int64_t entry_point,
                                        sdb_hnsw** out, uint64_t* n_bad) {
  if (!node_blob || !node_off || !node_ids || !n_nodes || (n_vec && (!vec_blob || !vec_off))) return SDB_EINVAL;
  SDB_TRY(check_load(native < 0 ? "sdb_hnsw_load_staged" : "sdb_hnsw_load_staged_typed", ctx, out, dim, metric, (int)vt,
                     n_elems, n_layers, entry_point));
  // An F32 index refuses a value of another SerializedVector variant.  It would load -- the decoder converts it -- but
  // be searched in F32 arithmetic where the reference computes in the value's own type (idx/trees/vector.rs:206-451).
  // Header = revision varint (1) + variant varint: one byte each.
  for (uint64_t v = 0; native < 0 && v < n_vec; v++) {
    const uint64_t a = vec_off[v], b = vec_off[v + 1];
    if (b >= a + 2 && vec_blob[a] == 1 && vec_blob[a + 1] != 1 && vec_blob[a + 1] <= 4) {
      static const char* names[] = {"F64", "F32", "I64", "I32", "I16"};
      set_error("sdb_hnsw_load_staged: He value %llu holds a %s vector; this loader builds F32 indexes "
                "(sdb_hnsw_load_staged_typed loads an index of that type)", (unsigned long long)v, names[vec_blob[a + 1]]);
      return SDB_EUNSUPPORTED;
    }
  }
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  sdb_hnsw* h = new_hnsw(ctx, dim, metric, vt, n_elems, n_layers, entry_point);
  cudaStream_t st = ctx->stream;
  const uint64_t nn = n_elems ? n_elems : 1;
  uint64_t bad_total = 0, bad = 0;
  sdb_status rc = SDB_OK;
  DevBuf<uint8_t> d_present;
  cudaError_t e = d_present.reserve(nn);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_present, 0, nn, st);
  if (e != cudaSuccess) {
    set_error("hnsw load: present-mask allocation failed: %s", cudaGetErrorString(e));
    rc = SDB_ENOMEM;
  }
  const size_t esz = vt_size(vt);
  if ((e = h->own_vec.reserve(esz * nn * dim)) != cudaSuccess) {
    set_error("hnsw load: vector allocation failed: %s", cudaGetErrorString(e));
    rc = SDB_ENOMEM;
  }
  h->d_vec = h->own_vec;
  // elements without an He value keep all-zero vectors; they are unreachable unless an Hn value names them
  if (rc == SDB_OK && cudaMemsetAsync(h->d_vec, 0, esz * nn * dim, st) != cudaSuccess) rc = SDB_ECUDA;
  if (rc == SDB_OK)
    rc = stage_decode_vectors(ctx, vec_blob, vec_off, vec_ids, n_vec, dim, SDB_F32, n_elems, h->d_vec, d_present, &bad, st,
                              native);
  bad_total += bad;
  uint64_t n_dropped = 0;
  for (uint32_t l = 0; l < n_layers && rc == SDB_OK; l++) {
    DevBuf<uint64_t> drp;
    DevBuf<uint32_t> dci;
    uint64_t ne = 0;
    bad = 0;
    rc = stage_decode_nodes(ctx, node_blob[l], node_off[l], node_ids[l], n_nodes[l], n_elems, &drp, &dci, &ne, &bad, st);
    if (rc == SDB_OK) {
      bad_total += bad;
      // drop edges from / to elements that have no He value ("edge to an unknown element")
      DevBuf<uint64_t> rp2, d_tot;
      DevBuf<uint32_t> ci2;
      uint64_t kept = 0;
      const unsigned g1 = (unsigned)((n_elems + 1 + 255) / 256);
      if (rp2.reserve(n_elems + 1) != cudaSuccess || d_tot.reserve(1) != cudaSuccess) rc = SDB_ENOMEM;
      if (rc == SDB_OK) {
        csr_present_degree_kernel<<<g1, 256, 0, st>>>(drp, dci, d_present, n_elems, rp2);
        count_launch(ctx);
        rc = exclusive_scan(ctx, rp2, rp2, n_elems + 1, d_tot, st);
      }
      if (rc == SDB_OK && (cudaMemcpyAsync(&kept, d_tot, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                           cudaStreamSynchronize(st) != cudaSuccess))
        rc = SDB_ECUDA;
      if (rc == SDB_OK && ci2.reserve(kept ? kept : 1) != cudaSuccess) rc = SDB_ENOMEM;
      if (rc == SDB_OK && n_elems) {
        csr_present_fill_kernel<<<g1, 256, 0, st>>>(drp, dci, d_present, n_elems, rp2, ci2);
        count_launch(ctx);
        if (cudaStreamSynchronize(st) != cudaSuccess) rc = SDB_ECUDA;
      }
      if (rc == SDB_OK) {
        n_dropped += ne - kept;
        h->rp.push_back(rp2);
        h->ci.push_back(ci2);
        h->own_rp.push_back(std::move(rp2));
        h->own_ci.push_back(std::move(ci2));
      } else if (rc == SDB_ENOMEM) {
        set_error("hnsw load: CSR filter allocation failed");
      }
    }
  }
  bad_total += n_dropped;
  if (n_bad) *n_bad = bad_total;
  uint8_t ep_present = 1;
  if (rc == SDB_OK && entry_point >= 0 && n_elems &&
      cudaMemcpy(&ep_present, d_present + entry_point, 1, cudaMemcpyDeviceToHost) != cudaSuccess)
    rc = SDB_ECUDA;
  d_present.reset();
  if (rc == SDB_OK && !ep_present) {
    set_error("sdb_hnsw_load_staged: the entry point %lld has no He value", (long long)entry_point);
    rc = SDB_EINVAL;
  }
  if (rc != SDB_OK) {
    sdb_hnsw_destroy(h);
    return rc;
  }
  return hnsw_finish(h, out);
}

sdb_status sdb_hnsw_load_staged(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, uint64_t n_elems,
                                const uint8_t* vec_blob, const uint64_t* vec_off, const uint64_t* vec_ids, uint64_t n_vec,
                                uint32_t n_layers, const uint8_t* const* node_blob, const uint64_t* const* node_off,
                                const uint64_t* const* node_ids, const uint64_t* n_nodes, int64_t entry_point,
                                sdb_hnsw** out, uint64_t* n_bad) {
  return hnsw_load_staged_impl(ctx, dim, metric, SDB_VT_F32, -1, n_elems, vec_blob, vec_off, vec_ids, n_vec, n_layers,
                               node_blob, node_off, node_ids, n_nodes, entry_point, out, n_bad);
}

sdb_status sdb_hnsw_load_staged_typed(sdb_ctx* ctx, uint32_t dim, sdb_metric metric, sdb_vector_type vt, uint64_t n_elems,
                                      const uint8_t* vec_blob, const uint64_t* vec_off, const uint64_t* vec_ids,
                                      uint64_t n_vec, uint32_t n_layers, const uint8_t* const* node_blob,
                                      const uint64_t* const* node_off, const uint64_t* const* node_ids,
                                      const uint64_t* n_nodes, int64_t entry_point, sdb_hnsw** out, uint64_t* n_bad) {
  return hnsw_load_staged_impl(ctx, dim, metric, vt, (int)vt, n_elems, vec_blob, vec_off, vec_ids, n_vec, n_layers,
                               node_blob, node_off, node_ids, n_nodes, entry_point, out, n_bad);
}

// Heuristic::select for n elements: row0 + i, or d_elem_ids[i] when that is given
static sdb_status select_neighbors(sdb_ctx* ctx, const float* d_vectors, uint32_t dim, sdb_metric metric, uint64_t row0,
                                   const uint32_t* d_elem_ids, uint64_t n, const uint64_t* d_cand,
                                   const uint32_t* d_cand_cnt, uint32_t kc, uint32_t m_max, int presorted,
                                   uint32_t* d_out, uint32_t* d_out_cnt) {
  if (!ctx || !d_vectors || !d_cand || !d_cand_cnt || !d_out || !d_out_cnt || !dim || !kc || !m_max) return SDB_EINVAL;
  if (metric != SDB_COSINE && metric != SDB_EUCLIDEAN) return SDB_EUNSUPPORTED;
  if (n == 0) return SDB_OK;
  const size_t smem = sizeof(float) * (2 * (size_t)dim + 2 * kc) * 4;
  if (smem > 227 * 1024) {  // the opt-in limit of dynamic shared memory per block
    set_error("sdb_hnsw_select_neighbors: %zu bytes of shared memory per block needed (dimension + kc > 7264)", smem);
    return SDB_EUNSUPPORTED;
  }
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  auto kern = metric == SDB_COSINE ? hnsw_select_kernel<true> : hnsw_select_kernel<false>;
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)((n + 3) / 4), 128, smem, ctx->stream>>>(d_vectors, dim, row0, n, d_elem_ids, d_cand, d_cand_cnt, kc, m_max, presorted, d_out, d_out_cnt);
  count_launch(ctx);
  SDB_CUDA(cudaGetLastError());
  SDB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SDB_OK;
}

sdb_status sdb_hnsw_select_neighbors(sdb_ctx* ctx, const float* d_vectors, uint32_t dim, sdb_metric metric, uint64_t row0,
                                     uint64_t n, const uint64_t* d_cand, const uint32_t* d_cand_cnt, uint32_t kc,
                                     uint32_t m_max, int presorted, uint32_t* d_out, uint32_t* d_out_cnt) {
  return select_neighbors(ctx, d_vectors, dim, metric, row0, nullptr, n, d_cand, d_cand_cnt, kc, m_max, presorted, d_out,
                          d_out_cnt);
}

sdb_status sdb_hnsw_select_neighbors_ids(sdb_ctx* ctx, const float* d_vectors, uint32_t dim, sdb_metric metric,
                                         const uint32_t* d_elem_ids, uint64_t n, const uint64_t* d_cand,
                                         const uint32_t* d_cand_cnt, uint32_t kc, uint32_t m_max, int presorted,
                                         uint32_t* d_out, uint32_t* d_out_cnt) {
  if (!d_elem_ids) return SDB_EINVAL;
  return select_neighbors(ctx, d_vectors, dim, metric, 0, d_elem_ids, n, d_cand, d_cand_cnt, kc, m_max, presorted, d_out,
                          d_out_cnt);
}

sdb_status sdb_hnsw_knn_exact_device(sdb_hnsw* h, const void* d_queries, uint32_t nq, uint32_t k, const uint32_t* d_members,
                                     uint64_t n_members, uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count) {
  if (!h || k == 0 || k > 256) return SDB_EINVAL;
  if (nq && (!d_queries || !d_out_elems || !d_out_dist || !d_out_count)) return SDB_EINVAL;
  if (!d_members) n_members = h->n;
  if (n_members > h->n) return SDB_EINVAL;
  if (nq == 0) return SDB_OK;
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> guard(h->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  auto run = [&]() -> sdb_status {  // the temporaries are released on every path, before the synchronisation below
    AsyncBuf<uint32_t> sorted;
    AsyncBuf<unsigned int> d_max;
    AsyncBuf<char> d_tmp;
    VecState<Mem::Async> qs;
    if (d_members && n_members) {  // ascending ids: ties are then ranked by id; every id must name an element
      size_t tmp_bytes = 0;
      SDB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, d_members, sorted.get(), n_members, 0, 32, st));
      SDB_CUDA(sorted.reserve(n_members, st));
      SDB_CUDA(d_tmp.reserve(tmp_bytes ? tmp_bytes : 1, st));
      SDB_CUDA(d_max.reserve(1, st));
      SDB_CUDA(cub::DeviceRadixSort::SortKeys(d_tmp.get(), tmp_bytes, d_members, sorted.get(), n_members, 0, 32, st));
      count_launch(ctx);
      SDB_CUDA(cudaMemsetAsync(d_max, 0, sizeof(unsigned int), st));
      members_max_kernel<<<(unsigned)((n_members + 255) / 256), 256, 0, st>>>(sorted, n_members, d_max);
      count_launch(ctx);
      unsigned int mx = 0;
      SDB_CUDA(cudaMemcpyAsync(&mx, d_max, sizeof(mx), cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaStreamSynchronize(st));
      if (mx >= h->n) {
        set_error("sdb_hnsw_knn_exact_device: member id %u is not an element (%llu elements)", mx, (unsigned long long)h->n);
        return SDB_EINVAL;
      }
    }
    SDB_TRY(vec_state_make(ctx, h->metric, h->vt, d_queries, nq, h->dim, qs, st));
    HnswParams P = element_params(h);
    P.queries = d_queries;
    P.nq = nq;
    P.k = k;
    P.out_elems = d_out_elems;
    P.out_dist = d_out_dist;
    P.out_count = d_out_count;
    P.q_mean = qs.mean;
    P.q_sx2 = qs.sx2;
    P.q_bits = qs.bits;
    P.q_nbits = qs.nbits;
    P.q_norm = qs.norm;
    const size_t per_warp = hn_stage_bytes(h->dim, h->metric, h->vt) + 12 * ((size_t)k + 1) + 64;
    const uint32_t* mem = d_members ? sorted.get() : nullptr;
    return with_vt(h->vt, [&](auto tag) {
      using T = decltype(tag);
      return with_metric(h->metric, [&](auto met) {
        return launch_warps(ctx, hnsw_knn_exact_kernel<decltype(met)::value, T>, per_warp, nq, "sdb_hnsw_knn_exact_device",
                            P, mem, n_members);
      });
    });
  };
  sdb_status rc = run();
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == SDB_OK) {
    set_error("sdb_hnsw_knn_exact_device: %s", cudaGetErrorString(cudaGetLastError()));
    rc = SDB_ECUDA;
  }
  return rc;
}

sdb_status sdb_hnsw_select_device(sdb_hnsw* h, const uint32_t* d_elem_ids, uint64_t row0, uint64_t n, const uint64_t* d_cand,
                                  const uint32_t* d_cand_cnt, uint32_t kc, uint32_t m_max, int presorted, uint32_t* d_out,
                                  uint32_t* d_out_cnt) {
  if (!h || !kc || !m_max || (n && (!d_cand || !d_cand_cnt || !d_out || !d_out_cnt))) return SDB_EINVAL;
  if (!d_elem_ids && row0 + n > h->n) return SDB_EINVAL;
  if (n == 0) return SDB_OK;
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> guard(h->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  const HnswParams P = element_params(h);
  const size_t per_warp = hn_stage_bytes(h->dim, h->metric, h->vt) + 12 * (size_t)kc + 4 * (size_t)m_max + 64;
  const sdb_status rc = with_vt(h->vt, [&](auto tag) {
    using T = decltype(tag);
    return with_metric(h->metric, [&](auto met) {
      return launch_warps(ctx, hnsw_select_typed_kernel<decltype(met)::value, T>, per_warp, n, "sdb_hnsw_select_device", P,
                          d_elem_ids, row0, n, d_cand, d_cand_cnt, kc, m_max, presorted, d_out, d_out_cnt);
    });
  });
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess && rc == SDB_OK) {
    set_error("sdb_hnsw_select_device: %s", cudaGetErrorString(cudaGetLastError()));
    return SDB_ECUDA;
  }
  return rc;
}

using WalkKernel = void (*)(HnswParams);
static WalkKernel walk_kernel(sdb_metric metric, sdb_vector_type vt, int occ, bool bits) {
  if (vt == SDB_VT_F32 && metric == SDB_COSINE) {
    if (bits) return hnsw_search_kernel<SDB_COSINE, 4, float, true>;  // 123 registers: no spills (6 blocks spill)
    return occ >= 8 ? hnsw_search_kernel<SDB_COSINE, 8, float> : occ <= 4 ? hnsw_search_kernel<SDB_COSINE, 4, float> : hnsw_search_kernel<SDB_COSINE, 6, float>;
  }
  return with_vt(vt, [&](auto tag) {
    using T = decltype(tag);
    return with_metric(metric, [&](auto met) -> WalkKernel {
      constexpr int MET = decltype(met)::value;
      constexpr bool COS32 = MET == SDB_COSINE && is_f32_v<T>;  // (F32 cosine: returned above)
      return bits ? hnsw_search_kernel<MET, COS32 ? 4 : 1, T, true> : hnsw_search_kernel<MET, COS32 ? 6 : 1, T>;
    });
  });
}

// the bitmaps of sdb_hnsw_search_filtered_batch[_device] (see the header)
struct BatchFilter {
  const uint32_t* filters;
  uint32_t n_filters;
  const uint32_t* query_filter;  // host
  bool on_device;                // filters is device memory
};

// The spill tier of a batch-filtered call: n_sp queries of P.spill_list walked by hnsw_spill_kernel, in as many slots
// as free device memory holds (at most one per resident warp, at most one per query).  Queued on st, the walk's stream.
static sdb_status hnsw_spill(sdb_hnsw* h, const HnswParams& P, uint32_t n_sp, DevBuf<ulonglong2>& heap,
                             DevBuf<uint32_t>& stamp, AsyncBuf<uint32_t>& next, cudaStream_t st) {
  Ctx* ctx = h->ctx;
  const size_t per_warp = (hn_stage_bytes(h->dim, h->metric, h->vt) + 12 * ((size_t)P.ef + 2) + 64 + 15) & ~size_t(15);
  const size_t smem = per_warp * HN_WARPS;
  if (smem > 220 * 1024) {
    set_error("hnsw: dim %u / ef %u need %zu bytes of shared memory per block in the spill tier", h->dim, P.ef, smem);
    return SDB_EUNSUPPORTED;
  }
  return with_vt(h->vt, [&](auto tag) -> sdb_status {
    using T = decltype(tag);
    return with_metric(h->metric, [&](auto met) -> sdb_status {
      const auto kern = hnsw_spill_kernel<decltype(met)::value, T>;
      SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      int per_sm = 1;
      SDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, HN_WARPS * 32, smem));
      const uint64_t resident = (uint64_t)ctx->sm_count * std::max(per_sm, 1) * HN_WARPS;
      // a slot: the heap (16 bytes per element) and the visited stamps (4 bytes per element); the pool takes at most
      // half of the free memory, from cudaMalloc, so that it goes back to the device when the call returns (the stream
      // pool would keep it cached)
      const uint64_t slot_bytes = 20 * std::max<uint64_t>(h->n, 1);
      size_t free_b = 0, total_b = 0;
      SDB_CUDA(cudaMemGetInfo(&free_b, &total_b));
      uint64_t slots = std::min<uint64_t>({(uint64_t)n_sp, resident, free_b / 2 / slot_bytes});
      for (;; slots /= 2) {  // memory can be taken in between: halve until it fits
        if (slots == 0) {
          set_error("hnsw: not even one spill slot (%llu bytes) fits in device memory",
                    (unsigned long long)slot_bytes);
          return SDB_ENOMEM;
        }
        if (heap.reserve(slots * h->n) == cudaSuccess && stamp.reserve(slots * h->n) == cudaSuccess) break;
        heap.reset(), stamp.reset();
      }
      SDB_CUDA(next.reserve(1, st));
      SDB_CUDA(cudaMemsetAsync(stamp, 0, sizeof(uint32_t) * slots * h->n, st));
      SDB_CUDA(cudaMemsetAsync(next, 0, sizeof(uint32_t), st));
      SpillSlots S;
      S.heap = heap;
      S.stamp = stamp;
      S.n = h->n;
      S.n_slots = (uint32_t)slots;
      S.next = next;
      kern<<<(unsigned)((slots + HN_WARPS - 1) / HN_WARPS), HN_WARPS * 32, smem, st>>>(P, S, (uint32_t)per_warp);
      count_launch(ctx);
      SDB_CUDA(cudaGetLastError());
      return SDB_OK;
    });
  });
}

// ---- the walk driver, in two halves.  hnsw_enqueue sizes and stages everything, launches the walk and queues the
// copies of its results, of the spill count and of the overflow flag, then records the search's event; hnsw_complete
// waits for that event, runs the spill tier when queries spilled (and copies the results again), and maps the flags to a
// status.  A blocking call runs both back to back in the handle's blocking slot, holding h->mu throughout; a ticket runs
// the first in sdb_hnsw_submit* and the second in sdb_hnsw_wait, which releases h->mu whenever it waits for the device.

// the argument checks of every search, before anything is queued
static sdb_status hnsw_check(const sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                             const uint64_t* out_elems, const double* out_dist, const uint32_t* out_count,
                             const BatchFilter* bf) {
  if (!h || (nq && (!queries || !out_count)) || (nq && k && (!out_elems || !out_dist))) return SDB_EINVAL;
  if (bf && nq) {
    if (bf->n_filters == 0 || !bf->filters) {
      set_error("filtered hnsw: %s", bf->n_filters == 0 ? "no filter given (n_filters == 0)" : "filters is NULL");
      return SDB_EINVAL;
    }
    if (bf->query_filter)
      for (uint32_t q = 0; q < nq; q++)
        if (bf->query_filter[q] >= bf->n_filters) {
          set_error("filtered hnsw: query %u uses filter %u of %u", q, bf->query_filter[q], bf->n_filters);
          return SDB_EINVAL;
        }
  }
  if (nq && k && ef > 4096) {  // (k == 0 or ef == 0: an empty answer for any ef)
    set_error("hnsw: ef %u > 4096 unsupported", ef);
    return SDB_EUNSUPPORTED;
  }
  return SDB_OK;
}

// the result copies of a search: the outputs of a host variant, and the counters
static sdb_status copy_results(HnswTicket& t) {
  const size_t nk = (size_t)t.nq * t.k;
  if (!t.device_io) {
    SDB_CUDA(cudaMemcpyAsync(t.out_elems, t.P.out_elems, sizeof(uint64_t) * nk, cudaMemcpyDeviceToHost, t.st));
    SDB_CUDA(cudaMemcpyAsync(t.out_dist, t.P.out_dist, sizeof(double) * nk, cudaMemcpyDeviceToHost, t.st));
    SDB_CUDA(cudaMemcpyAsync(t.out_count, t.P.out_count, sizeof(uint32_t) * t.nq, cudaMemcpyDeviceToHost, t.st));
  }
  if (t.out_counters)
    SDB_CUDA(cudaMemcpyAsync(t.out_counters, t.P.out_counters, sizeof(uint64_t) * 2 * t.nq,
                             t.device_io ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, t.st));
  return SDB_OK;
}

// The first half: everything up to the walk and its result copies, queued on t.st (the caller has set t.st and t.vis,
// holds h->mu and has checked the arguments with hnsw_check).
static sdb_status hnsw_enqueue(sdb_hnsw* h, HnswTicket& t, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                               const uint8_t* truthy, const uint8_t* noexp, uint64_t* out_elems, double* out_dist,
                               uint32_t* out_count, uint64_t* out_counters, bool device_io, const BatchFilter* bf) {
  Ctx* ctx = h->ctx;
  cudaStream_t st = t.st;
  t.nq = nq, t.k = k;
  t.device_io = device_io;
  t.batch_filter = bf != nullptr;
  t.out_elems = out_elems, t.out_dist = out_dist, t.out_count = out_count, t.out_counters = out_counters;
  t.walked = false;
  if (!t.ev) SDB_CUDA(cudaEventCreateWithFlags(&t.ev, cudaEventDisableTiming));
  if (!h->h_words) SDB_CUDA(h->h_words.reserve(2 * (N_TICKETS + 1)));
  t.h_word = h->h_words.get() + 2 * (&t - h->slots);
  t.h_word[0] = t.h_word[1] = 0;
  if (nq == 0 || k == 0 || ef == 0) {  // to_vec_limit(0) underflows in the reference; we return nothing
    if (nq && device_io) SDB_CUDA(cudaMemsetAsync(out_count, 0, sizeof(uint32_t) * nq, st));
    else if (nq) memset(out_count, 0, sizeof(uint32_t) * nq);
    SDB_CUDA(cudaEventRecord(t.ev, st));
    return SDB_OK;
  }
  // unfiltered: live candidates are a subset of w plus ties, 2*ef+34 is ample.  Filtered: every admitted element is a
  // candidate but only truthy ones enter w, so the window is sized for a selectivity down to ~1/16 (more = EOVERFLOW,
  // or the spill tier for the batch-filtered calls)
  const bool filtered = truthy || bf;
  uint32_t ccap = 2 * ef + 34;
  const uint32_t wcap = ef + 2;
  // bytes of a staged query and of the distance scratch (the kernel's per-warp layout)
  const size_t q_tile = hn_q_bytes(h->dim, h->vt == SDB_VT_F32, h->metric == SDB_COSINE,
                                   h->metric == SDB_JACCARD ? jkey_size(h->vt) : vt_size(h->vt)) +
                        hn_tile_bytes(h->vt == SDB_VT_F32 && h->metric == SDB_COSINE);
  if (filtered) {
    ccap = 16 * ef + 34;
    if (ccap < 1024) ccap = 1024;
    const size_t fixed = q_tile + 12 * (size_t)wcap + 64 + 16;
    const size_t room = (220 * 1024) / HN_WARPS;
    if (fixed + 12 * (size_t)ccap > room) ccap = room > fixed + 12 * (2 * (size_t)ef + 34) ? (uint32_t)((room - fixed) / 12) : 2 * ef + 34;
  }
  size_t per_warp = q_tile + 12 * (size_t)(ccap + wcap) + 64;
  per_warp = (per_warp + 15) & ~size_t(15);
  const size_t smem = per_warp * HN_WARPS;
  if (smem > 220 * 1024) {
    set_error("hnsw: dim %u / ef %u need %zu bytes of shared memory per block", h->dim, ef, smem);
    return SDB_EUNSUPPORTED;
  }
  // cosine: 8 lanes per row keep ~16 loads in flight per lane; 80 registers (6 blocks per SM) holds that without spills
  const int occ = getenv("SDB_HNSW_OCC") ? atoi(getenv("SDB_HNSW_OCC")) : 6;  // measured r2 (1M x 768, ef 64): 6 -> 1.40M QPS, 4 -> 1.32M, 8 -> 1.02M (spills)
  const WalkKernel kern = walk_kernel(h->metric, h->vt, occ, bf != nullptr);
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // the walk gets nothing from L1 (0.7 % hit rate): give the whole array to shared memory, or the driver's default
  // carve-out (135 KB) caps the kernel at 5 blocks per SM
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  int per_sm = 1;
  SDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, HN_WARPS * 32, smem));
  if (per_sm < 1) per_sm = 1;
  uint32_t grid = (uint32_t)(ctx->sm_count * per_sm);
  if (grid > (nq + HN_WARPS - 1) / HN_WARPS) grid = (nq + HN_WARPS - 1) / HN_WARPS;
  // visited tables: one per resident warp; 16 x the worst-case expansion of a typical walk, >= 2^13 slots
  uint32_t tl = 13;
  while ((1u << tl) < ef * 64u * 4u && tl < 20) tl++;
  if (filtered) tl = tl + 3 > 18 ? (tl > 18 ? tl : 18) : tl + 3;  // filtered walks visit ~1/selectivity more elements
  const uint32_t n_tables = grid * HN_WARPS;
  VisitSet& vs = *t.vis;
  if (!vs.tab || vs.table_log2 != tl || vs.n_tables < n_tables) {
    vs.tab.reset();  // a free on st: after the walks already queued on this set
    SDB_CUDA(vs.tab.reserve((size_t)n_tables << tl, st));
    SDB_CUDA(cudaMemsetAsync(vs.tab, 0, sizeof(uint64_t) * ((size_t)n_tables << tl), st));
    vs.table_log2 = tl;
    vs.n_tables = n_tables;
    vs.gen = 1;
  }
  const uint32_t q_per_warp = (nq + n_tables - 1) / n_tables;
  const uint32_t gens_per_warp = q_per_warp * h->n_layers + 1;
  if ((uint64_t)vs.gen + (uint64_t)gens_per_warp * n_tables >= 0xFFFFFFF0ull) {  // generation counter wrap
    SDB_CUDA(cudaMemsetAsync(vs.tab, 0, sizeof(uint64_t) * ((size_t)vs.n_tables << tl), st));
    vs.gen = 1;
  }
  const size_t esz = vt_size(h->vt);
  // device_io: queries and outputs already live on the device (index construction), no staging
  void* d_q = const_cast<void*>(queries);
  uint64_t* d_elems = out_elems;
  double* d_dist = out_dist;
  uint32_t* d_cnt = out_count;
  if (!device_io) {
    SDB_CUDA(t.q_buf.reserve(esz * (size_t)nq * h->dim, st));
    SDB_CUDA(t.elems_buf.reserve((size_t)nq * k, st));
    SDB_CUDA(t.dist_buf.reserve((size_t)nq * k, st));
    SDB_CUDA(t.cnt_buf.reserve(nq, st));
    d_q = t.q_buf, d_elems = t.elems_buf, d_dist = t.dist_buf, d_cnt = t.cnt_buf;
    SDB_CUDA(cudaMemcpyAsync(d_q, queries, esz * (size_t)nq * h->dim, cudaMemcpyHostToDevice, st));
  }
  SDB_CUDA(t.d_ctr.reserve(2 * (size_t)nq, st));
  SDB_CUDA(t.d_ovf.reserve(1, st));
  SDB_CUDA(cudaMemsetAsync(t.d_ovf, 0, 4, st));
  if (noexp) {
    SDB_CUDA(t.d_noexp.reserve(h->n ? h->n : 1, st));
    SDB_CUDA(cudaMemcpyAsync(t.d_noexp, noexp, h->n, cudaMemcpyHostToDevice, st));
  }
  if (truthy) {
    SDB_CUDA(t.d_truthy.reserve(h->n ? h->n : 1, st));
    SDB_CUDA(cudaMemcpyAsync(t.d_truthy, truthy, h->n, cudaMemcpyHostToDevice, st));
  }
  const uint32_t fwords = (uint32_t)((h->n + 31) / 32);
  const uint32_t* filters = nullptr;
  if (bf) {
    filters = bf->filters;
    if (!bf->on_device) {
      const size_t words = (size_t)fwords * bf->n_filters;
      SDB_CUDA(t.d_filters.reserve(words ? words : 1, st));
      SDB_CUDA(cudaMemcpyAsync(t.d_filters, bf->filters, sizeof(uint32_t) * words, cudaMemcpyHostToDevice, st));
      filters = t.d_filters;
    }
    if (bf->query_filter) {  // copied first: the caller may reuse its array as soon as the call returns
      t.h_qf.assign(bf->query_filter, bf->query_filter + nq);
      SDB_CUDA(t.d_qf.reserve(nq, st));
      SDB_CUDA(cudaMemcpyAsync(t.d_qf, t.h_qf.data(), sizeof(uint32_t) * nq, cudaMemcpyHostToDevice, st));
    }
    h->last_spilled = 0;
    SDB_CUDA(t.d_spill.reserve((size_t)nq + 1, st));  // the spill list, then its length
    SDB_CUDA(cudaMemsetAsync(t.d_spill.get() + nq, 0, sizeof(uint32_t), st));
  }
  HnswParams& P = t.P;
  P = HnswParams{};
  P.filters = filters;
  P.query_filter = t.d_qf;
  P.fwords = fwords;
  P.spill_list = t.d_spill;
  P.n_spill = bf ? t.d_spill.get() + nq : nullptr;
  P.ccap = ccap;
  P.truthy = t.d_truthy;
  P.noexp = t.d_noexp;
  P.vec = h->d_vec;
  P.norm = h->elems.norm;
  P.rp = h->d_rp;
  P.ci = h->d_ci;
  P.dim = h->dim;
  P.n_layers = h->n_layers;
  P.entry = h->entry;
  P.queries = d_q;
  P.nq = nq;
  P.k = k;
  P.ef = ef;
  P.visited = vs.tab;
  P.table_log2 = tl;
  P.gen_base = vs.gen;
  P.gens_per_warp = gens_per_warp;
  P.cancel = ctx->d_cancel;
  P.out_elems = d_elems;
  P.out_dist = d_dist;
  P.out_count = d_cnt;
  P.out_counters = t.d_ctr;
  P.overflow = t.d_ovf;
  P.mink_p = h->minkowski_p;  // the spill tier at completion keeps the order of the submit
  P.e_mean = h->elems.mean;
  P.e_sx2 = h->elems.sx2;
  P.e_bits = h->elems.bits;
  P.e_nbits = h->elems.nbits;
  SDB_TRY(vec_state_make(ctx, h->metric, h->vt, d_q, nq, h->dim, t.qs, st));
  P.q_mean = t.qs.mean;
  P.q_sx2 = t.qs.sx2;
  P.q_bits = t.qs.bits;
  P.q_nbits = t.qs.nbits;
  P.q_norm = t.qs.norm;
  kern<<<grid, HN_WARPS * 32, smem, st>>>(P);
  count_launch(ctx);
  SDB_CUDA(cudaGetLastError());
  t.walked = true;
  vs.gen += gens_per_warp * n_tables;
  if (bf) SDB_CUDA(cudaMemcpyAsync(&t.h_word[0], P.n_spill, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  SDB_TRY(copy_results(t));
  SDB_CUDA(cudaMemcpyAsync(&t.h_word[1], t.d_ovf, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaEventRecord(t.ev, st));
  return SDB_OK;
}

// The second half: waits for the search's event, runs the spill tier for the queries the walk gave up on, maps the
// flags to a status.  lk: a ticket's hold of h->mu, released while this waits for the device (the spill tier can take
// seconds at 0 % selectivity and must not stall the handle's other submits); null for a blocking call.
static sdb_status hnsw_complete(sdb_hnsw* h, HnswTicket& t, std::unique_lock<std::mutex>* lk) {
  Ctx* ctx = h->ctx;
  auto wait_event = [&](bool drop_spill) {
    if (lk) lk->unlock();
    const cudaError_t e = cudaEventSynchronize(t.ev);
    if (drop_spill) t.spill_heap.reset(), t.spill_stamp.reset();  // cudaFree may wait for the device: not under h->mu
    if (lk) lk->lock();
    return e;
  };
  SDB_CUDA(wait_event(false));
  if (!t.walked) return SDB_OK;
  if (t.batch_filter) {  // the queries the on-chip walk gave up on go to the spill tier
    const uint32_t n_sp = t.h_word[0];
    h->last_spilled = n_sp;
    if (n_sp && !ctx_cancelled(ctx)) {
      SDB_TRY(hnsw_spill(h, t.P, n_sp, t.spill_heap, t.spill_stamp, t.spill_next, t.st));
      SDB_TRY(copy_results(t));  // the copies queued with the walk predate the spilled queries' results
      SDB_CUDA(cudaEventRecord(t.ev, t.st));
      SDB_CUDA(wait_event(true));
    }
  }
  SDB_CUDA(cudaGetLastError());
  if (ctx_cancelled(ctx)) {  // warps stop taking new queries once the flag is up: the outputs are incomplete
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  const uint32_t ovf = t.h_word[1];
  if (ovf == 1) {
    set_error("hnsw: visited table overflow (ef too large, or filter too selective, for the per-query table)");
    return SDB_EOVERFLOW;
  }
  if (ovf == 2) {
    set_error("hnsw: candidate window overflow (filter too selective for ef %u): use the CPU path for this query", t.P.ef);
    return SDB_EOVERFLOW;
  }
  return SDB_OK;
}

// a blocking search: both halves in the blocking slot, on the context's stream, under h->mu throughout
static sdb_status hnsw_search_impl(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                   const uint8_t* truthy, const uint8_t* noexp, uint64_t* out_elems, double* out_dist,
                                   uint32_t* out_count, uint64_t* out_counters, bool device_io = false,
                                   const BatchFilter* bf = nullptr) {
  SDB_TRY(hnsw_check(h, queries, nq, k, ef, out_elems, out_dist, out_count, bf));
  if (nq == 0) return SDB_OK;
  std::lock_guard<std::mutex> guard(h->mu);
  SDB_CUDA(cudaSetDevice(h->ctx->device));
  HnswTicket& t = h->slots[N_TICKETS];
  t.st = h->ctx->stream;
  t.vis = &h->vis[0];
  sdb_status rc = hnsw_enqueue(h, t, queries, nq, k, ef, truthy, noexp, out_elems, out_dist, out_count, out_counters,
                               device_io, bf);
  if (rc == SDB_OK) rc = hnsw_complete(h, t, nullptr);
  else cudaStreamSynchronize(t.st);  // what the failed call queued no longer reads the caller's buffers
  t.release();
  return rc;
}

// an asynchronous search: the first half in a free ticket slot (even slots on the context's stream, odd ones on stream2,
// each stream with its own visited tables), completed by sdb_hnsw_wait
static sdb_status hnsw_submit_impl(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                   const uint8_t* noexp, uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                                   uint64_t* out_counters, bool device_io, const BatchFilter* bf, uint32_t* ticket) {
  if (!ticket) return SDB_EINVAL;
  SDB_TRY(hnsw_check(h, queries, nq, k, ef, out_elems, out_dist, out_count, bf));
  Ctx* ctx = h->ctx;
  if (ctx_cancelled(ctx)) {
    set_error("query cancelled");
    return SDB_ECANCELLED;
  }
  std::lock_guard<std::mutex> guard(h->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  HnswTicket* t = nullptr;
  for (int i = 0; i < N_TICKETS && !t; i++)
    if (!h->slots[i].busy) t = &h->slots[i];
  if (!t) {
    set_error("too many batches in flight (%d): call the matching wait first", N_TICKETS);
    return SDB_EOVERFLOW;
  }
  const int slot = (int)(t - h->slots);
  t->st = slot & 1 ? ctx->stream2 : ctx->stream;
  t->vis = &h->vis[slot & 1];
  const sdb_status rc = hnsw_enqueue(h, *t, queries, nq, k, ef, nullptr, noexp, out_elems, out_dist, out_count,
                                     out_counters, device_io, bf);
  if (rc != SDB_OK) {
    cudaStreamSynchronize(t->st);  // what the failed submit queued no longer reads the caller's buffers
    t->release();
    return rc;
  }
  t->busy = true;
  t->id = h->next_ticket++;
  if (h->next_ticket == 0) h->next_ticket = 1;
  *ticket = t->id;
  return SDB_OK;
}

// Distance::calculate(&query, &vector) for n host vectors on the context's stream (the caller holds the lock that
// serialises it): typed_distance_kernel plus the PEARSON / JACCARD state of the query and of the vectors.
static sdb_status typed_distances(Ctx* ctx, sdb_metric metric, sdb_vector_type vt, double minkowski_p, uint32_t dim,
                                  const void* query, const void* vectors, uint64_t n, double* out, const char* what) {
  cudaStream_t st = ctx->stream;
  const size_t esz = vt_size(vt);
  auto run = [&]() -> sdb_status {  // the temporaries are released on every path, before the synchronisation below
    AsyncBuf<char> d_q, d_v;
    AsyncBuf<double> d_o;
    VecState<Mem::Async> qs, vs;
    SDB_CUDA(d_q.reserve(esz * dim, st));
    SDB_CUDA(d_v.reserve(esz * n * dim, st));
    SDB_CUDA(d_o.reserve(n, st));
    SDB_CUDA(cudaMemcpyAsync(d_q, query, esz * dim, cudaMemcpyHostToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(d_v, vectors, esz * n * dim, cudaMemcpyHostToDevice, st));
    SDB_TRY(vec_state_make(ctx, metric, vt, d_q, 1, dim, qs, st));
    SDB_TRY(vec_state_make(ctx, metric, vt, d_v, n, dim, vs, st));
    TypedArgs A;
    A.q = reinterpret_cast<const float*>(d_q.get());
    A.vecs = reinterpret_cast<const float*>(d_v.get());
    A.dim = dim;
    A.n = n;
    A.out = d_o;
    A.mq.p = minkowski_p;
    A.v_mean = vs.mean;
    A.v_sx2 = vs.sx2;
    A.q_bits = qs.bits;
    A.v_bits = vs.bits;
    A.v_nbits = vs.nbits;
    A.v_norm = vs.norm;
    A.q_norm = qs.norm;
    if (metric == SDB_PEARSON) {  // the query's scalars travel by value
      SDB_CUDA(cudaMemcpyAsync(&A.mq.mean, qs.mean, sizeof(double), cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaMemcpyAsync(&A.mq.sx2, qs.sx2, sizeof(double), cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaStreamSynchronize(st));
    }
    if (metric == SDB_JACCARD) {
      SDB_CUDA(cudaMemcpyAsync(&A.mq.u, qs.nbits, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaStreamSynchronize(st));
    }
    const unsigned grid = (unsigned)((n + 127) / 128);
    with_vt(vt, [&](auto tag) {
      using T = decltype(tag);
      with_metric(metric, [&](auto met) { typed_distance_kernel<decltype(met)::value, T><<<grid, 128, 0, st>>>(A); });
    });
    count_launch(ctx);
    SDB_CUDA(cudaGetLastError());
    SDB_CUDA(cudaMemcpyAsync(out, d_o, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    return SDB_OK;
  };
  const sdb_status rc = run();
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == SDB_OK) {
    set_error("%s: %s", what, cudaGetErrorString(cudaGetLastError()));
    return SDB_ECUDA;
  }
  return rc;
}

sdb_status sdb_vec_distance_f32(sdb_ctx* ctx, sdb_metric metric, uint32_t dim, const float* query, const float* vectors,
                                uint64_t n, double* out) {
  if (!ctx || !dim || (n && (!query || !vectors || !out))) return SDB_EINVAL;
  if (metric != SDB_COSINE && metric != SDB_EUCLIDEAN) {
    set_error("sdb_vec_distance_f32: metric %d not implemented on the GPU path", (int)metric);
    return SDB_EUNSUPPORTED;
  }
  if (n == 0) return SDB_OK;
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  return typed_distances(ctx, metric, SDB_VT_F32, 3.0, dim, query, vectors, n, out, "sdb_vec_distance_f32");
}

sdb_status sdb_hnsw_distance(sdb_hnsw* h, const void* query, const void* vectors, uint64_t n, double* out) {
  if (!h || (n && (!query || !vectors || !out))) return SDB_EINVAL;
  if (n == 0) return SDB_OK;
  std::lock_guard<std::mutex> guard(h->mu);
  SDB_CUDA(cudaSetDevice(h->ctx->device));
  return typed_distances(h->ctx, h->metric, h->vt, h->minkowski_p, h->dim, query, vectors, n, out, "sdb_hnsw_distance");
}

sdb_status sdb_hnsw_set_minkowski_order(sdb_hnsw* h, double order) {
  if (!h || !(order == order)) return SDB_EINVAL;
  std::lock_guard<std::mutex> guard(h->mu);  // blocking searches hold it for their whole run; tickets keep their order
  h->minkowski_p = order;
  return SDB_OK;
}

sdb_status sdb_hnsw_search(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef, uint64_t* out_elems,
                           double* out_dist, uint32_t* out_count, uint64_t* out_counters) {
  return hnsw_search_impl(h, queries, nq, k, ef, nullptr, nullptr, out_elems, out_dist, out_count, out_counters);
}

sdb_status sdb_hnsw_search_device(sdb_hnsw* h, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                  uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count) {
  return hnsw_search_impl(h, d_queries, nq, k, ef, nullptr, nullptr, d_out_elems, d_out_dist, d_out_count, nullptr, true);
}

sdb_status sdb_hnsw_search_pending(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                   const uint8_t* all_docs_pending, uint64_t* out_elems, double* out_dist,
                                   uint32_t* out_count, uint64_t* out_counters) {
  if (!all_docs_pending) {
    set_error("sdb_hnsw_search_pending: the pending mask is NULL (use sdb_hnsw_search)");
    return SDB_EINVAL;
  }
  return hnsw_search_impl(h, queries, nq, k, ef, nullptr, all_docs_pending, out_elems, out_dist, out_count, out_counters);
}

sdb_status sdb_hnsw_search_filtered(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                    const uint8_t* truthy, uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                                    uint64_t* out_counters) {
  if (!truthy) {
    set_error("sdb_hnsw_search_filtered: truthy mask is NULL (use sdb_hnsw_search)");
    return SDB_EINVAL;
  }
  return hnsw_search_impl(h, queries, nq, k, ef, truthy, nullptr, out_elems, out_dist, out_count, out_counters);
}

sdb_status sdb_hnsw_search_filtered_batch(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                          const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                          uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                                          uint64_t* out_counters) {
  const BatchFilter bf{filters, n_filters, query_filter, false};
  return hnsw_search_impl(h, queries, nq, k, ef, nullptr, nullptr, out_elems, out_dist, out_count, out_counters, false,
                          &bf);
}

sdb_status sdb_hnsw_search_filtered_batch_device(sdb_hnsw* h, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                                 const uint32_t* d_filters, uint32_t n_filters,
                                                 const uint32_t* query_filter, uint64_t* d_out_elems,
                                                 double* d_out_dist, uint32_t* d_out_count, uint64_t* d_out_counters) {
  const BatchFilter bf{d_filters, n_filters, query_filter, true};
  return hnsw_search_impl(h, d_queries, nq, k, ef, nullptr, nullptr, d_out_elems, d_out_dist, d_out_count, d_out_counters,
                          true, &bf);
}

sdb_status sdb_hnsw_submit(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                           const uint8_t* all_docs_pending, uint64_t* out_elems, double* out_dist, uint32_t* out_count,
                           uint64_t* out_counters, uint32_t* ticket) {
  return hnsw_submit_impl(h, queries, nq, k, ef, all_docs_pending, out_elems, out_dist, out_count, out_counters, false,
                          nullptr, ticket);
}

sdb_status sdb_hnsw_submit_device(sdb_hnsw* h, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                  uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count,
                                  uint64_t* d_out_counters, uint32_t* ticket) {
  return hnsw_submit_impl(h, d_queries, nq, k, ef, nullptr, d_out_elems, d_out_dist, d_out_count, d_out_counters, true,
                          nullptr, ticket);
}

sdb_status sdb_hnsw_submit_filtered(sdb_hnsw* h, const void* queries, uint32_t nq, uint32_t k, uint32_t ef,
                                    const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                    uint64_t* out_elems, double* out_dist, uint32_t* out_count, uint64_t* out_counters,
                                    uint32_t* ticket) {
  const BatchFilter bf{filters, n_filters, query_filter, false};
  return hnsw_submit_impl(h, queries, nq, k, ef, nullptr, out_elems, out_dist, out_count, out_counters, false, &bf,
                          ticket);
}

sdb_status sdb_hnsw_submit_filtered_device(sdb_hnsw* h, const void* d_queries, uint32_t nq, uint32_t k, uint32_t ef,
                                           const uint32_t* d_filters, uint32_t n_filters, const uint32_t* query_filter,
                                           uint64_t* d_out_elems, double* d_out_dist, uint32_t* d_out_count,
                                           uint64_t* d_out_counters, uint32_t* ticket) {
  const BatchFilter bf{d_filters, n_filters, query_filter, true};
  return hnsw_submit_impl(h, d_queries, nq, k, ef, nullptr, d_out_elems, d_out_dist, d_out_count, d_out_counters, true,
                          &bf, ticket);
}

sdb_status sdb_hnsw_wait(sdb_hnsw* h, uint32_t ticket) {
  if (!h) return SDB_EINVAL;
  std::unique_lock<std::mutex> lk(h->mu);
  SDB_CUDA(cudaSetDevice(h->ctx->device));
  HnswTicket* t = nullptr;
  for (int i = 0; i < N_TICKETS && !t; i++)
    if (h->slots[i].busy && !h->slots[i].waiting && h->slots[i].id == ticket) t = &h->slots[i];
  if (!t) {
    set_error("sdb_hnsw_wait: unknown or already completed ticket %u", ticket);
    return SDB_EINVAL;
  }
  t->waiting = true;  // a second wait on the same ticket, while this one has released the lock, is refused
  const sdb_status rc = hnsw_complete(h, *t, &lk);
  t->release();
  return rc;
}

uint32_t sdb_hnsw_last_spilled(const sdb_hnsw* h) { return h ? h->last_spilled : 0; }

}  // extern "C"
