// screen_simt.cu -- K1: streaming f32 screen for small query batches (<= 8 queries per pass over the corpus).
//
// HBM-bound by construction: every corpus row (dim * 4 bytes) is read exactly once per launch.
//   producer warp : one elected thread issues cp.async.bulk (TMA 1-D bulk copy, SASS UBLKCP) of ROWS_PER_STAGE
//                   consecutive rows (they are contiguous in the row-major master copy) into a 2-stage
//                   shared-memory ring, completion on an mbarrier  -> ~100-190 KB of loads in flight per SM
//   8 consumer warps: each takes RPW rows of the stage, multiplies them with the <= 8 queries held in shared
//                   memory (16-byte conflict-free LDS, every query vector is read once per RPW rows), reduces
//                   with warp shuffles, scales by the row's screening norm and compares with the query's
//                   threshold tau; survivors are appended to the query's candidate list.
// Algorithmic bytes per row: dim*4 + 4 (snorm).  Replaces, as the *screen*, the scan loop of
// KnnTopK::execute (exec/operators/knn_topk.rs:185-228); exactness comes from candidates.cu.
#include "internal.cuh"

namespace sdb {

constexpr int SIMT_QB = 8;          // queries per launch
constexpr int SIMT_CWARPS = 8;      // consumer warps
constexpr int SIMT_THREADS = (SIMT_CWARPS + 1) * 32;
constexpr int SIMT_STAGES = 2;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sb_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void sb_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sb_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void sb_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// RPW = rows per consumer warp per stage (4, 2 or 1; chosen so that 2 stages + the queries fit shared memory)
// QB  = queries per launch (1, 4 or 8): fewer queries = less shared-memory read traffic per row
// FILT: filtered batch -- a row the query's filter rejects is never appended (filt.qf is indexed by q0 + query)
// DOT: Score::Dot -- the score is the dot itself, NaN for the rows whose screening norm is NaN; FAR: Score::EuclidFar,
// 2 acc + |x|^2; otherwise the score of `metric` (SDB_COSINE: cosine, else euclidean)
template <int RPW, int QB, bool FILT, bool DOT = false, bool FAR = false>
__global__ void __launch_bounds__(SIMT_THREADS, 1) screen_simt_kernel(
    const float* __restrict__ rows, const float* __restrict__ snorm, uint32_t dim, uint64_t n_rows,
    const float* __restrict__ q32, uint32_t q0, uint32_t nqb, int metric, PassDesc pass,
    const float* __restrict__ tau, Cand* __restrict__ cand, uint32_t* __restrict__ cand_cnt, uint32_t cap,
    FiltArg filt) {
  constexpr int RPS = RPW * SIMT_CWARPS;  // rows per stage
  extern __shared__ __align__(128) uint8_t smem_raw[];
  float* s_q = reinterpret_cast<float*>(smem_raw);                 // [QB][dim]
  float* s_rows = s_q + (size_t)QB * dim;                     // [STAGES][RPS][dim]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_rows + (size_t)SIMT_STAGES * RPS * dim);
  uint64_t* full_bar = bars;             // [STAGES]
  uint64_t* empty_bar = bars + SIMT_STAGES;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (uint32_t i = threadIdx.x; i < QB * dim; i += blockDim.x) {
    const uint32_t qi = i / dim;
    s_q[i] = qi < nqb ? q32[(size_t)(q0 + qi) * dim + (i - qi * dim)] : 0.f;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < SIMT_STAGES; s++) {
      sb_init(smem_addr(&full_bar[s]), 1);
      sb_init(smem_addr(&empty_bar[s]), SIMT_CWARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // work: tiles of TILE_ROWS rows, each cut into TILE_ROWS / RPS chunks; chunks are the pipeline unit
  constexpr uint32_t CHUNKS = TILE_ROWS / RPS;
  const uint32_t stage_bytes = (uint32_t)(RPS * dim * sizeof(float));

  if (warp == SIMT_CWARPS) {
    // ===================== producer =====================
    if (lane == 0) {
      uint32_t it = 0;
      for (uint32_t w = blockIdx.x; w < pass.count; w += gridDim.x) {
        const uint64_t tile_row0 = (uint64_t)pass_tile(pass, w) * TILE_ROWS;
        for (uint32_t ch = 0; ch < CHUNKS; ch++, it++) {
          const uint32_t s = it % SIMT_STAGES, ph = (it / SIMT_STAGES) & 1;
          const uint64_t r0 = tile_row0 + (uint64_t)ch * RPS;
          sb_wait(smem_addr(&empty_bar[s]), ph ^ 1);
          uint32_t bytes = 0;
          if (r0 < n_rows) {
            const uint64_t avail = n_rows - r0;
            bytes = avail >= (uint64_t)RPS ? stage_bytes : (uint32_t)(avail * dim * sizeof(float));
          }
          const uint32_t fb = smem_addr(&full_bar[s]);
          sb_expect_tx(fb, bytes);
          if (bytes) bulk_load(smem_addr(s_rows + (size_t)s * RPS * dim), rows + r0 * dim, bytes, fb);
        }
      }
    }
  } else {
    // ===================== consumers =====================
    float my_tau = __int_as_float(0x7f800000);  // +inf: lanes >= nqb never append
    if (lane < nqb) my_tau = tau[q0 + lane];
    const uint32_t nv = dim >> 2;
    uint32_t it = 0;
    for (uint32_t w = blockIdx.x; w < pass.count; w += gridDim.x) {
      const uint64_t tile_row0 = (uint64_t)pass_tile(pass, w) * TILE_ROWS;
      for (uint32_t ch = 0; ch < CHUNKS; ch++, it++) {
        const uint32_t s = it % SIMT_STAGES, ph = (it / SIMT_STAGES) & 1;
        sb_wait(smem_addr(&full_bar[s]), ph);
        const float* st = s_rows + (size_t)s * RPS * dim + (size_t)warp * RPW * dim;
        const uint64_t r_first = tile_row0 + (uint64_t)ch * RPS + (uint64_t)warp * RPW;
        float acc[RPW][QB];
#pragma unroll
        for (int rr = 0; rr < RPW; rr++)
#pragma unroll
          for (int qi = 0; qi < QB; qi++) acc[rr][qi] = 0.f;
        if (r_first < n_rows) {
          for (uint32_t v = lane; v < nv; v += 32) {
            float4 x[RPW];
#pragma unroll
            for (int rr = 0; rr < RPW; rr++) x[rr] = reinterpret_cast<const float4*>(st + (size_t)rr * dim)[v];
#pragma unroll
            for (int qi = 0; qi < QB; qi++) {
              const float4 qv = reinterpret_cast<const float4*>(s_q + (size_t)qi * dim)[v];
#pragma unroll
              for (int rr = 0; rr < RPW; rr++) {
                acc[rr][qi] = fmaf(x[rr].x, qv.x, acc[rr][qi]);
                acc[rr][qi] = fmaf(x[rr].y, qv.y, acc[rr][qi]);
                acc[rr][qi] = fmaf(x[rr].z, qv.z, acc[rr][qi]);
                acc[rr][qi] = fmaf(x[rr].w, qv.w, acc[rr][qi]);
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) sb_arrive(smem_addr(&empty_bar[s]));  // this warp is done reading the stage
        // warp reduction; afterwards lane qi keeps query qi's dot product
#pragma unroll
        for (int rr = 0; rr < RPW; rr++) {
          const uint64_t row = r_first + rr;
          float mine = 0.f;
#pragma unroll
          for (int qi = 0; qi < QB; qi++) {
            float vsum = acc[rr][qi];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) vsum += __shfl_xor_sync(0xffffffffu, vsum, o);
            if ((int)lane == qi) mine = vsum;
          }
          if (lane < nqb && row < n_rows) {
            const float sn = __ldg(snorm + row);
            const float sc = DOT   ? (sn == sn ? mine : sn)
                           : FAR ? fmaf(2.f, mine, sn)
                                 : metric == SDB_COSINE ? mine * sn : fmaf(2.f, mine, -sn);
            if (sc >= my_tau && (!FILT || filt_pass(filt, q0 + lane, (uint32_t)row))) {  // NaN (skipped / special rows) never passes
              const uint32_t pos = atomicAdd(cand_cnt + q0 + lane, 1u);
              if (pos < cap) {
                Cand cd;
                cd.score = sc;
                cd.row = (uint32_t)row;
                cand[(size_t)(q0 + lane) * cap + pos] = cd;
              }
            }
          }
        }
      }
    }
  }
}

// generic fallback for dimensions that are not a multiple of 4 (rows not 16-byte aligned): plain coalesced loads
template <bool FILT, bool DOT = false, bool FAR = false>
__global__ void __launch_bounds__(256) screen_simt_generic_kernel(
    const float* __restrict__ rows, const float* __restrict__ snorm, uint32_t dim, uint64_t n_rows,
    const float* __restrict__ q32, uint32_t q0, uint32_t nqb, int metric, PassDesc pass,
    const float* __restrict__ tau, Cand* __restrict__ cand, uint32_t* __restrict__ cand_cnt, uint32_t cap,
    FiltArg filt) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* s_q = reinterpret_cast<float*>(smem_raw);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (uint32_t i = threadIdx.x; i < SIMT_QB * dim; i += blockDim.x) {
    const uint32_t qi = i / dim;
    s_q[i] = qi < nqb ? q32[(size_t)(q0 + qi) * dim + (i - qi * dim)] : 0.f;
  }
  __syncthreads();
  float my_tau = __int_as_float(0x7f800000);
  if (lane < nqb) my_tau = tau[q0 + lane];
  for (uint32_t w = blockIdx.x; w < pass.count; w += gridDim.x) {
    const uint64_t tile_row0 = (uint64_t)pass_tile(pass, w) * TILE_ROWS;
    for (uint32_t j = warp; j < (uint32_t)TILE_ROWS; j += 8) {
      const uint64_t row = tile_row0 + j;
      if (row >= n_rows) break;
      float acc[SIMT_QB];
#pragma unroll
      for (int qi = 0; qi < SIMT_QB; qi++) acc[qi] = 0.f;
      for (uint32_t c = lane; c < dim; c += 32) {
        const float x = __ldg(rows + row * dim + c);
#pragma unroll
        for (int qi = 0; qi < SIMT_QB; qi++) acc[qi] = fmaf(x, s_q[(size_t)qi * dim + c], acc[qi]);
      }
      float mine = 0.f;
#pragma unroll
      for (int qi = 0; qi < SIMT_QB; qi++) {
        float v = acc[qi];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((int)lane == qi) mine = v;
      }
      if (lane < nqb) {
        const float sn = __ldg(snorm + row);
        const float sc = DOT   ? (sn == sn ? mine : sn)
                           : FAR ? fmaf(2.f, mine, sn)
                                 : metric == SDB_COSINE ? mine * sn : fmaf(2.f, mine, -sn);
        if (sc >= my_tau && (!FILT || filt_pass(filt, q0 + lane, (uint32_t)row))) {
          const uint32_t pos = atomicAdd(cand_cnt + q0 + lane, 1u);
          if (pos < cap) {
            Cand cd;
            cd.score = sc;
            cd.row = (uint32_t)row;
            cand[(size_t)(q0 + lane) * cap + pos] = cd;
          }
        }
      }
    }
  }
}

// the kernels' runtime `metric`: the form of the view's score (SDB_COSINE: acc / |x|), not the corpus metric
static int simt_metric(const View& v) { return v.sc == Score::Cosine ? (int)SDB_COSINE : (int)SDB_EUCLIDEAN; }

template <int RPW, int QB>
static sdb_status launch_ring_q(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                                cudaStream_t st, size_t smem, const View& v) {
  Ctx* ctx = c->ctx;
  auto kern = v.sc == Score::Dot ? (filt.bits ? screen_simt_kernel<RPW, QB, true, true> : screen_simt_kernel<RPW, QB, false, true>)
              : v.sc == Score::EuclidFar
                  ? (filt.bits ? screen_simt_kernel<RPW, QB, true, false, true> : screen_simt_kernel<RPW, QB, false, false, true>)
                  : (filt.bits ? screen_simt_kernel<RPW, QB, true> : screen_simt_kernel<RPW, QB, false>);
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  uint32_t grid = (uint32_t)ctx->sm_count;
  if (grid > p.count) grid = p.count;
  for (uint32_t q0 = 0; q0 < nq; q0 += QB) {
    const uint32_t nqb = nq - q0 < (uint32_t)QB ? nq - q0 : (uint32_t)QB;
    kern<<<grid, SIMT_THREADS, smem, st>>>((const float*)c->d_rows.get(), view_snorm(c, v), c->dim, c->n, s.d_q32, q0,
                                           nqb, simt_metric(v), p, s.d_tau, s.d_cand, s.d_cand_cnt, s.sc_cap, filt);
    count_launch(ctx);
  }
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

template <int RPW>
static sdb_status launch_ring(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                              cudaStream_t st, size_t q_bytes8, size_t ring, const View& v) {
  // the shared-memory query tile shrinks with QB; the row ring keeps its size
  if (nq == 1) return launch_ring_q<RPW, 1>(c, s, filt, nq, p, st, q_bytes8 / 8 + ring, v);
  if (nq <= 4) return launch_ring_q<RPW, 4>(c, s, filt, nq, p, st, q_bytes8 / 2 + ring, v);
  return launch_ring_q<RPW, 8>(c, s, filt, nq, p, st, q_bytes8 + ring, v);
}

sdb_status screen_simt_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, const PassDesc& p,
                            cudaStream_t st, const View& v) {
  if (p.count == 0) return SDB_OK;
  Ctx* ctx = c->ctx;
  const size_t q_bytes = sizeof(float) * SIMT_QB * c->dim;
  const size_t budget = 220 * 1024;
  auto ring_only = [&](int rpw) { return sizeof(float) * SIMT_STAGES * rpw * SIMT_CWARPS * (size_t)c->dim + 64; };
  auto ring_bytes = [&](int rpw) { return q_bytes + ring_only(rpw); };
  if (c->dim % 4 == 0 && ring_bytes(1) <= budget) {
    if (ring_bytes(4) <= budget) return launch_ring<4>(c, s, filt, nq, p, st, q_bytes, ring_only(4), v);
    if (ring_bytes(2) <= budget) return launch_ring<2>(c, s, filt, nq, p, st, q_bytes, ring_only(2), v);
    return launch_ring<1>(c, s, filt, nq, p, st, q_bytes, ring_only(1), v);
  }
  if (q_bytes > 200 * 1024) {
    set_error("screen_simt: dim %u too large for the shared-memory query tile", c->dim);
    return SDB_EUNSUPPORTED;
  }
  auto kern = v.sc == Score::Dot ? (filt.bits ? screen_simt_generic_kernel<true, true> : screen_simt_generic_kernel<false, true>)
              : v.sc == Score::EuclidFar
                  ? (filt.bits ? screen_simt_generic_kernel<true, false, true> : screen_simt_generic_kernel<false, false, true>)
                  : (filt.bits ? screen_simt_generic_kernel<true> : screen_simt_generic_kernel<false>);
  SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)q_bytes));
  int per_sm = 1;
  SDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, q_bytes));
  if (per_sm < 1) per_sm = 1;
  uint32_t grid = (uint32_t)(ctx->sm_count * per_sm);
  if (grid > p.count) grid = p.count;
  for (uint32_t q0 = 0; q0 < nq; q0 += SIMT_QB) {
    const uint32_t nqb = nq - q0 < (uint32_t)SIMT_QB ? nq - q0 : (uint32_t)SIMT_QB;
    kern<<<grid, 256, q_bytes, st>>>((const float*)c->d_rows.get(), view_snorm(c, v), c->dim, c->n, s.d_q32, q0, nqb,
                                     simt_metric(v), p, s.d_tau, s.d_cand, s.d_cand_cnt, s.sc_cap, filt);
    count_launch(ctx);
  }
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

}  // namespace sdb
