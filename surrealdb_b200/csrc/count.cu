// count.cu -- the count path of Family::Count corpora (HAMMING / JACCARD): exact ranking, not a screen.  Exact
// distances of every row, batched over the queries on the Lp screen's tiling (LP_*), ranked per row range.
#include <algorithm>

#include "exactmath.cuh"
#include "internal.cuh"

namespace sdb {

// ---- HAMMING: exact mismatch counts, ranked per row range (DESIGN.md section 2, "HAMMING count path") ---------------
// The Lp screen's tiling with equality keys instead of floats (eq_key_f32 / eq_key_f64, exactmath.cuh): a (query, row,
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
// (dist_key(d), row) pairs.  Both order as (distance, row), which is unique per list.  A descending batch (desc) keeps
// the complement of the value's half instead -- ~count, order_key(d, true) -- so the same lists and the same merge keep
// the k largest values, earlier rows first: the union of every range's k best still holds the query's k best, ties
// included, in either direction.
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
    FiltArg filt, bool desc) {
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
            const uint64_t e = ((uint64_t)(desc ? ~acc[i][j] : acc[i][j]) << 32) | row;
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
          const uint32_t cv = (uint32_t)(v >> 32);
          const double d = (double)(desc ? ~cv : cv);
          const size_t o = (size_t)q * rr_stride + base + p;
          rr_key[o] = order_key(d, desc);
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
    FiltArg filt, bool desc) {
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
      if (ok)
        e.key = order_key(jaccard_counts(rows + row * dim, dim, jfirst + row * words, __ldg(jux + row), qk, n_look, uq),
                          desc);
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
      rr_dist[o] = __longlong_as_double((long long)((desc ? ~v.key : v.key) ^ 0x8000000000000000ull));
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
static sdb_status launch_count(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k,
                               uint32_t n_ranges, bool desc, cudaStream_t st) {
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
                                                 (const CountKey<T>*)s.d_qkey.get(), nq, k, n_ranges, s.d_cand_cnt,
                                                 s.d_rr_key, s.d_rr_dist, s.d_rr_row, s.rr_stride, filt, desc);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}
template <typename T, bool FILT>
static sdb_status launch_count_qb(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k,
                                  uint32_t n_ranges, bool desc, cudaStream_t st) {
  if (nq <= 8) return launch_count<T, FILT, 8, 1>(c, s, filt, nq, k, n_ranges, desc, st);
  if constexpr (sizeof(T) == 8) return launch_count<T, FILT, 32, 4>(c, s, filt, nq, k, n_ranges, desc, st);
  else return nq <= 32 ? launch_count<T, FILT, 32, 4>(c, s, filt, nq, k, n_ranges, desc, st)
                       : launch_count<T, FILT, 64, 4>(c, s, filt, nq, k, n_ranges, desc, st);
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

sdb_status count_prep_queries(const Corpus* c, Scratch& s, uint32_t nq, cudaStream_t st) {
  if (nq == 0) return SDB_OK;
  if (c->metric == SDB_JACCARD) {
    if (c->dtype == SDB_F32)
      count_jaccard_qprep_kernel<uint32_t><<<nq, 256, 0, st>>>(s.d_q64, nq, c->dim, s.d_qkey.get(), s.d_qjac,
                                                               s.d_qjac + 2 * (size_t)s.sc_nq);
    else
      count_jaccard_qprep_kernel<unsigned long long><<<nq, 256, 0, st>>>(
          s.d_q64, nq, c->dim, (unsigned long long*)s.d_qkey.get(), s.d_qjac, s.d_qjac + 2 * (size_t)s.sc_nq);
  } else if (c->dtype == SDB_F32) {
    count_qkeys_kernel<uint32_t><<<nq, 128, 0, st>>>(s.d_q64, nq, c->dim, s.d_qkey.get());
  } else {
    count_qkeys_kernel<unsigned long long><<<nq, 128, 0, st>>>(s.d_q64, nq, c->dim,
                                                               (unsigned long long*)s.d_qkey.get());
  }
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

template <typename T, bool FILT>
static sdb_status launch_count_jaccard(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k,
                                       uint32_t n_ranges, bool desc, cudaStream_t st) {
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
                                                 c->d_jux, (const EqKey<T>*)s.d_qkey.get(), s.d_qjac, nq, k,
                                                 n_ranges, s.d_cand_cnt, s.d_rr_key, s.d_rr_dist, s.d_rr_row,
                                                 s.rr_stride, filt, desc);
  count_launch(c->ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

sdb_status count_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k, cudaStream_t st,
                      bool desc) {
  if (nq == 0 || k == 0 || c->n == 0) return SDB_OK;
  const uint32_t n_ranges = count_ranges(c, nq, k);
  if (c->metric == SDB_JACCARD) {
    if (c->dtype == SDB_F32)
      return filt.bits ? launch_count_jaccard<float, true>(c, s, filt, nq, k, n_ranges, desc, st)
                       : launch_count_jaccard<float, false>(c, s, filt, nq, k, n_ranges, desc, st);
    return filt.bits ? launch_count_jaccard<double, true>(c, s, filt, nq, k, n_ranges, desc, st)
                     : launch_count_jaccard<double, false>(c, s, filt, nq, k, n_ranges, desc, st);
  }
  if (c->dtype == SDB_F32)
    return filt.bits ? launch_count_qb<float, true>(c, s, filt, nq, k, n_ranges, desc, st)
                     : launch_count_qb<float, false>(c, s, filt, nq, k, n_ranges, desc, st);
  return filt.bits ? launch_count_qb<double, true>(c, s, filt, nq, k, n_ranges, desc, st)
                   : launch_count_qb<double, false>(c, s, filt, nq, k, n_ranges, desc, st);
}

}  // namespace sdb
