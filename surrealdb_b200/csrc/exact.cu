// exact.cu -- KX: exact brute force for ONE query over the whole corpus, in the reference's own f64
// arithmetic (RefAcc, exactmath.cuh), followed by an exact radix selection of the k
// smallest (distance key, scan position) pairs.  Used for
//   * F64 corpora and SDB_SCREEN_NONE_EXACT,
//   * queries the screens cannot bound (zero / non-finite query norm),
//   * queries whose screened result failed the error-bound proof or overflowed its candidate buffer.
// It never approximates, so the library's answer does not depend on the screens being right.  It also ranks every
// vector function in either direction (sdb_corpus_order_*): the keys are order_key(value, desc).
#include "exactmath.cuh"
#include "internal.cuh"
#include "rowwalk.cuh"

namespace sdb {

constexpr uint32_t EX_QCHUNK = 1024;
constexpr uint64_t KEY_SKIPPED = ~0ull;  // never produced by dist_key(canonical value)

template <typename T, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) exact_keys_kernel(const T* __restrict__ rows, uint32_t dim, uint64_t n,
                                                                int metric, const double* __restrict__ mag,
                                                                const uint8_t* __restrict__ skip,
                                                                const double* __restrict__ q64 /* this query */,
                                                                const double* __restrict__ qmag_p,
                                                                const uint32_t* __restrict__ qflags_p,
                                                                uint64_t* __restrict__ keys,
                                                                double* __restrict__ vals /* non-null: every row's value */,
                                                                double mink_p, bool desc) {
  __shared__ T tile[WARPS][32][33];
  __shared__ double s_q[EX_QCHUNK];
  __shared__ double s_qstat[2];  // pearson: mean and (population) deviation of the query
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool q_nan = (*qflags_p & 2u) != 0;
  const double qm = *qmag_p;
  // `metric` also takes the projection-only ids SDB_FN_SIMILARITY_COSINE / SDB_FN_DOT / SDB_FN_MAGNITUDE
  if (metric == SDB_PEARSON && threadIdx.x == 0) {
    const double2 mom = pearson_moments(q64, dim);
    s_qstat[0] = mom.x;
    s_qstat[1] = RefAcc<SDB_PEARSON>::sd(mom.y, dim);
  }
  __syncthreads();
  const int n_phase = metric == SDB_PEARSON ? 2 : 1;
  const uint64_t rows_per_block = (uint64_t)WARPS * 32;
  for (uint64_t b0 = (uint64_t)blockIdx.x * rows_per_block; b0 < n; b0 += (uint64_t)gridDim.x * rows_per_block) {
    const uint64_t r = b0 + warp * 32 + lane;
    const uint32_t my_row = r < n ? (uint32_t)r : NO_ROW;
    RefSum acc;
    double m1 = 0.0;
    if (metric == SDB_CHEBYSHEV) acc.acc = RefAcc<SDB_CHEBYSHEV>::start;
    for (int phase = 0; phase < n_phase; phase++) {
      for (uint32_t cb = 0; cb < dim; cb += EX_QCHUNK) {
        const uint32_t cw = dim - cb < EX_QCHUNK ? dim - cb : EX_QCHUNK;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < cw; i += blockDim.x) s_q[i] = q64[cb + i];
        __syncthreads();
        const T* base = rows + cb;
        for (uint32_t c0 = 0; c0 < cw; c0 += 32) {
          const uint32_t c = c0 + lane;
#pragma unroll 8
          for (int rr = 0; rr < 32; rr++) {
            const uint32_t row = __shfl_sync(0xffffffffu, my_row, rr);
            T v = T(0);
            if (row != NO_ROW && c < cw) v = __ldg(base + (size_t)row * dim + c);
            tile[warp][rr][lane] = v;
          }
          __syncwarp();
          if (my_row != NO_ROW) {
            const uint32_t lim = cw - c0 < 32u ? cw - c0 : 32u;
            const T* t = tile[warp][lane];
            switch (metric) {  // uniform across the block
              case SDB_COSINE:
              case SDB_FN_SIMILARITY_COSINE:
              case SDB_FN_DOT:
                for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_COSINE>{}.step(acc, (double)t[j], s_q[c0 + j]);
                break;
              case SDB_FN_MAGNITUDE: break;  // precomputed at finalize
              case SDB_EUCLIDEAN:
                for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_EUCLIDEAN>{}.step(acc, (double)t[j], s_q[c0 + j]);
                break;
              case SDB_MANHATTAN:
                for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_MANHATTAN>{}.step(acc, (double)t[j], s_q[c0 + j]);
                break;
              case SDB_CHEBYSHEV:
                for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_CHEBYSHEV>{}.step(acc, (double)t[j], s_q[c0 + j]);
                break;
              case SDB_HAMMING:
                for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_HAMMING>{}.step(acc, (double)t[j], s_q[c0 + j]);
                break;
              case SDB_MINKOWSKI:
                for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_MINKOWSKI>{mink_p}.step(acc, (double)t[j], s_q[c0 + j]);
                break;
              default:  // SDB_PEARSON
                if (phase == 0) {
                  for (uint32_t j = 0; j < lim; j++) RefAcc<SDB_PEARSON>::mean_step(acc, (double)t[j]);
                } else {
                  const RefAcc<SDB_PEARSON> pe{m1, s_qstat[0]};
                  for (uint32_t j = 0; j < lim; j++) pe.step_dev(acc, (double)t[j], s_q[c0 + j]);
                }
                break;
            }
          }
          __syncwarp();
        }
      }
      if (metric == SDB_PEARSON && phase == 0) {
        m1 = __ddiv_rn(acc.acc, (double)dim);
        acc.acc = 0.0;
      }
    }
    if (my_row != NO_ROW) {
      uint64_t key;
      if (skip && skip[r]) {
        key = KEY_SKIPPED;
        if (vals) vals[r] = __longlong_as_double(0x7FF8000000000000ll);
      } else {
        double d;
        switch (metric) {
          case SDB_COSINE: d = RefAcc<SDB_COSINE>{}.finish(acc, mag[r], qm, q_nan); break;
          case SDB_FN_SIMILARITY_COSINE: d = RefAcc<SDB_FN_SIMILARITY_COSINE>{}.finish(acc, mag[r], qm, q_nan); break;
          case SDB_FN_DOT: d = RefAcc<SDB_FN_DOT>{}.finish(acc, q_nan); break;
          case SDB_FN_MAGNITUDE: d = RefAcc<SDB_FN_MAGNITUDE>{}.finish(mag[r]); break;
          case SDB_EUCLIDEAN: d = RefAcc<SDB_EUCLIDEAN>{}.finish(acc, q_nan); break;
          case SDB_MANHATTAN: d = RefAcc<SDB_MANHATTAN>{}.finish(acc, q_nan); break;
          case SDB_MINKOWSKI: d = RefAcc<SDB_MINKOWSKI>{mink_p}.finish(acc, q_nan); break;
          case SDB_CHEBYSHEV: d = RefAcc<SDB_CHEBYSHEV>{}.finish(acc, q_nan); break;
          case SDB_HAMMING: d = RefAcc<SDB_HAMMING>{}.finish(acc, q_nan); break;
          default:  // SDB_PEARSON
            d = RefAcc<SDB_PEARSON>::finish(acc, dim, RefAcc<SDB_PEARSON>::sd(acc.acc2, dim), s_qstat[1], q_nan);
        }
        key = order_key(d, desc);
        if (vals) vals[r] = d;
      }
      if (keys) keys[r] = key;
    }
  }
}

// ---- Jaccard (vector.rs:121-127): set semantics over the VALUES of the two vectors, so it needs a whole row and the
// whole query at once instead of a column stream.  union = set(row); every query element already present in the
// (growing) union counts towards the intersection; result = |intersection| / |union|.  Restated without a hash set:
//   in_row[j]  = q_j equals some row element            dup[j] = q_j equals an earlier query element (per query, once)
//   inter = #{j : in_row[j] or dup[j]}                  union = distinct(row) + #{j : not in_row[j] and not dup[j]}
// Number equality on floats: same bits, or both zero (val/number.rs PartialEq; NaN == NaN when the payloads agree).
// One warp per row, O(dim^2 / 32) comparisons per lane: a niche metric served for completeness, not for speed.
// (num_eq_f64: exactmath.cuh)
__global__ void jaccard_qdup_kernel(const double* __restrict__ q64, uint32_t dim, uint8_t* __restrict__ dup) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < dim; j += gridDim.x * blockDim.x) {
    bool d = false;
    for (uint32_t i = 0; i < j && !d; i++) d = num_eq_f64(q64[i], q64[j]);
    dup[j] = d ? 1 : 0;
  }
}
template <typename T>
__global__ void __launch_bounds__(128) jaccard_keys_kernel(const T* __restrict__ rows, uint32_t dim, uint64_t n,
                                                           const uint8_t* __restrict__ skip,
                                                           const double* __restrict__ q64, const uint8_t* __restrict__ qdup,
                                                           uint64_t* __restrict__ keys, double* __restrict__ vals,
                                                           bool desc) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t r = warp0; r < n; r += n_warps) {
    if (skip && skip[r]) {
      if (lane == 0) {
        if (keys) keys[r] = KEY_SKIPPED;
        if (vals) vals[r] = __longlong_as_double(0x7FF8000000000000ll);
      }
      continue;
    }
    const T* x = rows + r * dim;
    uint32_t distinct = 0, inter = 0, fresh = 0;
    for (uint32_t i = lane; i < dim; i += 32) {
      const double xi = (double)x[i];
      bool seen = false;
      for (uint32_t i2 = 0; i2 < i && !seen; i2++) seen = num_eq_f64((double)x[i2], xi);
      distinct += seen ? 0 : 1;
    }
    for (uint32_t j = lane; j < dim; j += 32) {
      const double qj = q64[j];
      bool in_row = false;
      for (uint32_t i = 0; i < dim && !in_row; i++) in_row = num_eq_f64((double)x[i], qj);
      if (in_row || qdup[j]) inter++;
      else fresh++;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      distinct += __shfl_xor_sync(0xffffffffu, distinct, o);
      inter += __shfl_xor_sync(0xffffffffu, inter, o);
      fresh += __shfl_xor_sync(0xffffffffu, fresh, o);
    }
    if (lane == 0) {
      const double d = __ddiv_rn((double)inter, (double)(distinct + fresh));  // (intersection_size / union.len() as f64)
      if (keys) keys[r] = order_key(d, desc);
      if (vals) vals[r] = d;
    }
  }
}
static sdb_status jaccard_launch(const Corpus* c, const double* d_q64, uint64_t* d_keys, double* d_vals,
                                 cudaStream_t st, bool desc = false) {
  Ctx* ctx = c->ctx;
  AsyncBuf<uint8_t> d_dup;
  SDB_CUDA(d_dup.reserve(c->dim, st));
  jaccard_qdup_kernel<<<(c->dim + 127) / 128, 128, 0, st>>>(d_q64, c->dim, d_dup);
  const int grid = ctx->sm_count * 16;
  if (c->dtype == SDB_F32)
    jaccard_keys_kernel<float><<<grid, 128, 0, st>>>((const float*)c->d_rows.get(), c->dim, c->n, c->d_skip, d_q64, d_dup, d_keys, d_vals, desc);
  else
    jaccard_keys_kernel<double><<<grid, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, c->n, c->d_skip, d_q64, d_dup, d_keys, d_vals, desc);
  count_launch(ctx, 2);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// ---- exact radix select over the 96-bit composite (key, row), MSB first, 12 passes of 8 bits --------
struct SelState {
  uint64_t prefix_key;
  uint32_t prefix_row;
  uint32_t remaining;  // rank (1-based) still to locate inside the current prefix bucket
  uint32_t k_eff;      // min(k, #valid rows)
  uint32_t out_count;  // gather cursor
  uint32_t hist[256];
};

__global__ void sel_init_kernel(SelState* st, uint32_t k) {
  if (threadIdx.x == 0) {
    st->prefix_key = 0;
    st->prefix_row = 0;
    st->remaining = k;
    st->k_eff = k;
    st->out_count = 0;
  }
  st->hist[threadIdx.x] = 0;
}

__global__ void __launch_bounds__(256) sel_hist_kernel(const uint64_t* __restrict__ keys, uint64_t n, uint32_t pass,
                                                       SelState* st) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  if (st->k_eff != 0) {
    const uint64_t pk = st->prefix_key;
    const uint32_t pr = st->prefix_row;
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
      const uint64_t key = keys[i];
      if (key == KEY_SKIPPED) continue;
      uint32_t digit;
      bool match;
      if (pass < 8) {
        const uint64_t hi_mask = pass == 0 ? 0ull : (~0ull << (64 - 8 * pass));
        match = ((key ^ pk) & hi_mask) == 0;
        digit = (uint32_t)(key >> (56 - 8 * pass)) & 255u;
      } else {
        const uint32_t p = pass - 8;
        const uint32_t rmask = p == 0 ? 0u : (~0u << (32 - 8 * p));
        const uint32_t row = (uint32_t)i;
        match = key == pk && ((row ^ pr) & rmask) == 0;
        digit = (row >> (24 - 8 * p)) & 255u;
      }
      if (match) atomicAdd(&h[digit], 1u);
    }
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&st->hist[threadIdx.x], h[threadIdx.x]);
}

__global__ void sel_scan_kernel(SelState* st, uint32_t pass) {  // one thread: 256 bins
  if (threadIdx.x != 0) return;
  if (pass == 0) {
    uint64_t total = 0;
    for (int d = 0; d < 256; d++) total += st->hist[d];
    if (st->remaining > total) {
      st->remaining = (uint32_t)total;
      st->k_eff = (uint32_t)total;
    }
  }
  if (st->k_eff != 0) {
    uint32_t cum = 0;
    int d = 0;
    for (; d < 256; d++) {
      if (cum + st->hist[d] >= st->remaining) break;
      cum += st->hist[d];
    }
    st->remaining -= cum;
    if (pass < 8) st->prefix_key |= (uint64_t)d << (56 - 8 * pass);
    else st->prefix_row |= (uint32_t)d << (24 - 8 * (pass - 8));
  }
  for (int d = 0; d < 256; d++) st->hist[d] = 0;
}

__global__ void __launch_bounds__(256) sel_gather_kernel(const uint64_t* __restrict__ keys, uint64_t n, SelState* st,
                                                         uint64_t* __restrict__ g_key, uint32_t* __restrict__ g_row) {
  if (st->k_eff == 0) return;
  const uint64_t pk = st->prefix_key;
  const uint32_t pr = st->prefix_row;
  const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
    const uint64_t key = keys[i];
    if (key == KEY_SKIPPED) continue;
    if (key < pk || (key == pk && (uint32_t)i <= pr)) {
      const uint32_t pos = atomicAdd(&st->out_count, 1u);
      g_key[pos] = key;
      g_row[pos] = (uint32_t)i;
    }
  }
}

// sort the k_eff gathered pairs and write the query's output row (single block).  The distance is the row's computed
// value, not the key inverted: dist_key maps -0.0 to 0.0 (they tie), and the reference returns the -0.0 it computed.
__global__ void __launch_bounds__(1024) sel_emit_kernel(const SelState* st, const uint64_t* __restrict__ g_key,
                                                        const uint32_t* __restrict__ g_row,
                                                        const double* __restrict__ vals, uint32_t k,
                                                        uint64_t row_base, uint64_t* __restrict__ out_rows,
                                                        double* __restrict__ out_dist, uint32_t* __restrict__ out_count) {
  extern __shared__ uint64_t s_mem[];
  const uint32_t n = st->k_eff;
  uint32_t p2 = 1;
  while (p2 < n) p2 <<= 1;
  uint64_t* s_key = s_mem;
  uint64_t* s_row = s_mem + p2;
  for (uint32_t i = threadIdx.x; i < p2; i += blockDim.x) {
    s_key[i] = i < n ? g_key[i] : ~0ull;
    s_row[i] = i < n ? (uint64_t)g_row[i] : ~0ull;
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
          }
        }
      }
      __syncthreads();
    }
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    out_rows[i] = row_base + s_row[i];
    out_dist[i] = vals[s_row[i]];
  }
  if (threadIdx.x == 0) *out_count = n;
}

// filtered queries: rows the query's bitmap rejects leave the selection like skipped rows
__global__ void __launch_bounds__(256) exact_filter_keys_kernel(uint64_t* __restrict__ keys, uint64_t n,
                                                                const uint32_t* __restrict__ bits) {
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x)
    if (!((__ldg(bits + (r >> 5)) >> (r & 31u)) & 1u)) keys[r] = KEY_SKIPPED;
}

sdb_status exact_init_device() {
  SDB_CUDA(cudaFuncSetAttribute(sel_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16 * 4096));
  return SDB_OK;
}

// d_out_rows / d_out_dist / d_out_count point at THIS query's output row
sdb_status exact_query(Corpus* c, const double* d_q64, const double* d_qmag, const uint32_t* d_qflags, uint32_t k,
                       uint64_t row_base, uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                       cudaStream_t st, const uint32_t* filter, uint32_t filter_words, const Ranking& rank) {
  Ctx* ctx = c->ctx;
  {
    const uint64_t cap = c->cap > c->n ? c->cap : c->n;
    SDB_CUDA(c->d_ex_key.reserve(cap ? cap : 1));
    SDB_CUDA(c->d_ex_val.reserve(cap ? cap : 1));
    // SelState + gather buffers (key u64[4096], row u32[4096])
    SDB_CUDA(c->d_sel.reserve((sizeof(SelState) + 4096 * 12 + 64) / sizeof(uint32_t)));
  }
  if (k > 4096) {
    set_error("exact path supports k <= 4096 (got %u)", k);
    return SDB_EUNSUPPORTED;
  }
  SelState* sel = reinterpret_cast<SelState*>(c->d_sel.get());
  uint64_t* g_key = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(c->d_sel.get()) + ((sizeof(SelState) + 63) / 64) * 64);
  uint32_t* g_row = reinterpret_cast<uint32_t*>(g_key + 4096);
  const uint64_t n = c->n;
  const int fn = rank.fn < 0 ? (int)c->metric : rank.fn;
  if (n && fn == SDB_JACCARD) {
    SDB_TRY(jaccard_launch(c, d_q64, c->d_ex_key, c->d_ex_val, st, rank.desc));
  } else if (n) {
    const int grid = ctx->sm_count * 8;
    if (c->dtype == SDB_F32)
      exact_keys_kernel<float, 4><<<grid, 128, 0, st>>>((const float*)c->d_rows.get(), c->dim, n, fn, c->d_mag,
                                                        c->d_skip, d_q64, d_qmag, d_qflags, c->d_ex_key, c->d_ex_val,
                                                        c->minkowski_p, rank.desc);
    else
      exact_keys_kernel<double, 4><<<grid, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, n, fn, c->d_mag,
                                                         c->d_skip, d_q64, d_qmag, d_qflags, c->d_ex_key, c->d_ex_val,
                                                         c->minkowski_p, rank.desc);
    count_launch(ctx);
  }
  if (n && filter) {
    if ((n + 31) / 32 > filter_words) {
      set_error("exact path: the row filter has %u words, the corpus needs %llu", filter_words,
                (unsigned long long)((n + 31) / 32));
      return SDB_EINVAL;
    }
    exact_filter_keys_kernel<<<ctx->sm_count * 4, 256, 0, st>>>(c->d_ex_key, n, filter);
    count_launch(ctx);
  }
  sel_init_kernel<<<1, 256, 0, st>>>(sel, k);
  count_launch(ctx);
  const int hgrid = ctx->sm_count * 4;
  for (uint32_t pass = 0; pass < 12; pass++) {
    sel_hist_kernel<<<hgrid, 256, 0, st>>>(c->d_ex_key, n, pass, sel);
    sel_scan_kernel<<<1, 32, 0, st>>>(sel, pass);
    count_launch(ctx, 2);
  }
  sel_gather_kernel<<<hgrid, 256, 0, st>>>(c->d_ex_key, n, sel, g_key, g_row);
  uint32_t p2 = 1;
  while (p2 < k) p2 <<= 1;
  sel_emit_kernel<<<1, 1024, sizeof(uint64_t) * 2 * p2, st>>>(sel, g_key, g_row, c->d_ex_val, k, row_base, d_out_rows,
                                                             d_out_dist, d_out_count);
  count_launch(ctx, 2);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}


// one reference-arithmetic value per row (SURVEY 8f-4: projected scalar vector functions)
sdb_status exact_project(const Corpus* c, int fn, const double* d_q64, const double* d_qmag, const uint32_t* d_qflags,
                         double* d_vals, cudaStream_t st) {
  Ctx* ctx = c->ctx;
  const uint64_t n = c->n;
  if (!n) return SDB_OK;
  if (fn == SDB_JACCARD) return jaccard_launch(c, d_q64, nullptr, d_vals, st);
  const int grid = ctx->sm_count * 8;
  if (c->dtype == SDB_F32)
    exact_keys_kernel<float, 4><<<grid, 128, 0, st>>>((const float*)c->d_rows.get(), c->dim, n, fn, c->d_mag, c->d_skip,
                                                      d_q64, d_qmag, d_qflags, nullptr, d_vals, c->minkowski_p, false);
  else
    exact_keys_kernel<double, 4><<<grid, 128, 0, st>>>((const double*)c->d_rows.get(), c->dim, n, fn, c->d_mag, c->d_skip,
                                                       d_q64, d_qmag, d_qflags, nullptr, d_vals, c->minkowski_p, false);
  count_launch(ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

}  // namespace sdb
