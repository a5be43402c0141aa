// graph.cu -- K4: `->edge->node` expansion over device-resident CSR adjacency.
//
// Replaces the per-source KV prefix scans of GraphEdgeScan::execute (exec/operators/scan/graph.rs:214-279)
// driven by LookupPart::evaluate_lookup (exec/parts/lookup.rs:139-170): for every frontier element, in
// frontier order, emit its targets in stored (KV key) order -- duplicates kept, per-source limit honoured
// (graph.rs:83,238,261).  Output position = exclusive prefix sum of the (limited) degrees, so the result is
// order-identical to the reference no matter how the work is split.  The expand kernel is OUTPUT-centric
// (each block owns a contiguous slice of the output and finds its sources by binary search), which balances
// power-law degree distributions at warp/block level without any per-vertex special casing.
// `+collect` (exec/operators/recursion/collect.rs:74-143) adds a first-seen de-duplication per BFS level.
//
// Algorithmic bytes per hop: 16|F| (two row_ptr reads per source) + 4|E_h| (col_idx) + 4|E_h| (output).
// A WHERE-filtered hop (filter_kernel, below) scans every candidate edge of its sources, even with a per-source limit.
#include "internal.cuh"

namespace sdb {

struct Graph {
  Ctx* ctx = nullptr;
  uint64_t n_rows = 0, n_edges = 0;
  DevBuf<uint64_t> d_row_ptr;
  DevBuf<uint32_t> d_col_idx;
  bool targets_in_rows = true;  // every col_idx < n_rows (required by +collect, which indexes per-row state by target)
  // row-sharded adjacency (SURVEY 8e): this rank holds rows [row_lo, row_hi) of the n_rows-row CSR; d_row_ptr is the
  // slice rebased to 0.  An unsharded graph is the shard [0, n_rows).
  uint64_t row_lo = 0, row_hi = 0;
  bool sharded = false;
  // +collect state, kept between calls (a 50M-node graph needs 450 MB of it: allocating it per call cost 145 ms)
  DevBuf<uint8_t> d_seen;
  DevBuf<uint32_t> d_first;
  DevBuf<uint32_t> d_res;
  std::mutex mu;
};

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// ---- exclusive prefix sum (u64), hierarchical ------------------------------------------------------
__global__ void __launch_bounds__(SCAN_THREADS) scan_tile_kernel(const uint64_t* __restrict__ in, uint64_t* __restrict__ out,
                                                                 uint64_t n, uint64_t* __restrict__ tile_sums) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
  uint64_t v[SCAN_ITEMS];
  uint64_t sum = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    v[i] = base + i < n ? in[base + i] : 0;
    sum += v[i];
  }
  // inclusive scan of per-thread sums inside the block
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= (uint32_t)o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint64_t w = lane < SCAN_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) {
      const uint64_t t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= (uint32_t)o) w += t;
    }
    if (lane < SCAN_THREADS / 32) s_warp[lane] = w;
  }
  __syncthreads();
  uint64_t excl = inc - sum + (warp ? s_warp[warp - 1] : 0);
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    if (base + i < n) out[base + i] = excl;
    excl += v[i];
  }
  if (threadIdx.x == SCAN_THREADS - 1 && tile_sums) tile_sums[blockIdx.x] = excl;
}
__global__ void scan_add_kernel(uint64_t* __restrict__ out, uint64_t n, const uint64_t* __restrict__ tile_off) {
  const uint64_t i = (uint64_t)blockIdx.x * SCAN_TILE + threadIdx.x;
  const uint64_t add = tile_off[blockIdx.x];
  for (int k = 0; k < SCAN_ITEMS; k++) {
    const uint64_t j = i + (uint64_t)k * SCAN_THREADS;
    if (j < n) out[j] += add;
  }
}
// out[0..n) = exclusive scan of in[0..n); *d_total = sum.  in/out may alias.
sdb_status exclusive_scan(Ctx* ctx, const uint64_t* d_in, uint64_t* d_out, uint64_t n, uint64_t* d_total,
                                 cudaStream_t st) {
  if (n == 0) {
    SDB_CUDA(cudaMemsetAsync(d_total, 0, 8, st));
    return SDB_OK;
  }
  const uint64_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  AsyncBuf<uint64_t> d_sums;
  SDB_CUDA(d_sums.reserve(tiles + 1, st));
  scan_tile_kernel<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(d_in, d_out, n, d_sums);
  count_launch(ctx);
  if (tiles > 1) {
    SDB_TRY(exclusive_scan(ctx, d_sums, d_sums, tiles, d_total, st));
    scan_add_kernel<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(d_out, n, d_sums);
    count_launch(ctx);
  } else {
    SDB_CUDA(cudaMemcpyAsync(d_total, d_sums, 8, cudaMemcpyDeviceToDevice, st));
  }
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// ---- one hop -----------------------------------------------------------------------------------------
// row_ptr is this rank's slice [row_lo, row_hi) rebased to 0; sources owned by another rank contribute 0 here and
// their degree arrives through the all-reduce
__global__ void degree_kernel(const uint64_t* __restrict__ row_ptr, uint64_t n_rows, uint64_t row_lo, uint64_t row_hi,
                              const uint32_t* __restrict__ frontier, uint64_t n_f, uint32_t limit,
                              uint64_t* __restrict__ deg, uint32_t* __restrict__ err) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_f) return;
  const uint32_t v = frontier[i];
  if (v >= n_rows) {
    *err = 1;
    deg[i] = 0;
    return;
  }
  uint64_t d = 0;
  if (v >= row_lo && v < row_hi) {
    d = row_ptr[v - row_lo + 1] - row_ptr[v - row_lo];
    if (limit && d > limit) d = limit;
  }
  deg[i] = d;
}

constexpr int EXP_THREADS = 256;
constexpr int EXP_PER_THREAD = 8;
constexpr int EXP_TILE = EXP_THREADS * EXP_PER_THREAD;  // outputs per block
constexpr int EXP_SRC_MAX = EXP_TILE + 2;

__device__ __forceinline__ uint64_t upper_bound_minus1(const uint64_t* a, uint64_t lo, uint64_t hi, uint64_t x) {
  // largest i in [lo, hi) with a[i] <= x   (a is non-decreasing, a[lo] <= x)
  while (hi - lo > 1) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (a[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(EXP_THREADS) expand_kernel(const uint64_t* __restrict__ row_ptr,
                                                             const uint32_t* __restrict__ col_idx,
                                                             const uint32_t* __restrict__ frontier, uint64_t n_f,
                                                             const uint64_t* __restrict__ off /* n_f + 1 */,
                                                             uint64_t total, uint32_t* __restrict__ out,
                                                             uint64_t row_lo, uint64_t row_hi) {
  __shared__ uint64_t s_off[EXP_SRC_MAX];
  __shared__ uint64_t s_row[EXP_SRC_MAX];
  __shared__ uint64_t s_i0, s_i1;
  const uint64_t o0 = (uint64_t)blockIdx.x * EXP_TILE;
  const uint64_t o1 = o0 + EXP_TILE < total ? o0 + EXP_TILE : total;
  if (threadIdx.x == 0) {
    s_i0 = upper_bound_minus1(off, 0, n_f + 1, o0);
    s_i1 = upper_bound_minus1(off, 0, n_f + 1, o1 - 1);
  }
  __syncthreads();
  const uint64_t i0 = s_i0, i1 = s_i1;
  const bool in_smem = (i1 - i0 + 2) <= (uint64_t)EXP_SRC_MAX;
  if (in_smem) {
    for (uint64_t t = threadIdx.x; t < i1 - i0 + 2; t += EXP_THREADS) {
      const uint64_t i = i0 + t;
      s_off[t] = off[i];  // i <= i1 + 1 <= n_f
      uint64_t rb = ~0ull;  // ~0: the source belongs to another rank's rows -- its output slots stay zero here
      if (i < n_f) {
        const uint64_t v = frontier[i];
        if (v >= row_lo && v < row_hi) rb = row_ptr[v - row_lo];
      }
      s_row[t] = rb;
    }
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < EXP_PER_THREAD; u++) {
    const uint64_t o = o0 + (uint64_t)u * EXP_THREADS + threadIdx.x;  // coalesced output
    if (o >= o1) break;
    uint64_t src, start, rbeg;
    if (in_smem) {
      const uint64_t t = upper_bound_minus1(s_off, 0, i1 - i0 + 2, o);
      src = i0 + t;
      start = s_off[t];
      rbeg = s_row[t];
    } else {  // pathological: thousands of zero-degree sources inside this slice
      src = upper_bound_minus1(off, i0, i1 + 2, o);
      start = off[src];
      const uint64_t v = frontier[src];
      rbeg = (v >= row_lo && v < row_hi) ? row_ptr[v - row_lo] : ~0ull;
    }
    if (rbeg != ~0ull) out[o] = __ldg(col_idx + rbeg + (o - start));
    (void)src;
  }
}

// *d_out: an empty buffer, which receives the next frontier (stays empty when it has no elements)
static sdb_status hop_device(Graph* g, const uint32_t* d_frontier, uint64_t n_f, uint32_t limit, AsyncBuf<uint32_t>* d_out,
                             uint64_t* n_out, cudaStream_t st) {
  Ctx* ctx = g->ctx;
  *n_out = 0;
  if (n_f == 0) return SDB_OK;
  AsyncBuf<uint64_t> d_off;
  AsyncBuf<uint32_t> d_err;
  SDB_CUDA(d_off.reserve(n_f + 2, st));
  uint64_t* d_total = d_off + n_f;  // off[n_f] = total: exactly the sentinel the expand kernel wants
  SDB_CUDA(d_err.reserve(1, st));
  SDB_CUDA(cudaMemsetAsync(d_err, 0, 4, st));
  degree_kernel<<<(unsigned)((n_f + 255) / 256), 256, 0, st>>>(g->d_row_ptr, g->n_rows, g->row_lo, g->row_hi, d_frontier, n_f,
                                                               limit, d_off, d_err);
  count_launch(ctx);
  // sharded adjacency: every source is owned by exactly one rank, so the SUM over ranks is the full degree array
  const bool multi = g->sharded && comm_size(ctx) > 1;
  if (multi) SDB_TRY(comm_allreduce_sum(ctx, d_off, n_f, 8, st));
  SDB_TRY(exclusive_scan(ctx, d_off, d_off, n_f, d_total, st));
  uint64_t total = 0;
  uint32_t err = 0;
  SDB_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (err) {
    set_error("graph expand: frontier id out of range (graph has %llu rows)", (unsigned long long)g->n_rows);
    return SDB_EINVAL;
  }
  if (total > 0xFFFFFFF0ull) {
    set_error("graph expand: %llu results exceed the 2^32 frontier limit", (unsigned long long)total);
    return SDB_EOVERFLOW;
  }
  if (total) {
    SDB_CUDA(d_out->reserve(total, st));
    if (multi) SDB_CUDA(cudaMemsetAsync(*d_out, 0, sizeof(uint32_t) * total, st));
    expand_kernel<<<(unsigned)((total + EXP_TILE - 1) / EXP_TILE), EXP_THREADS, 0, st>>>(
        g->d_row_ptr, g->d_col_idx, d_frontier, n_f, d_off, total, *d_out, g->row_lo, g->row_hi);
    count_launch(ctx);
    // every output slot was written by exactly one rank (the owner of its source), the others hold 0: the sum over
    // ranks IS the next frontier, in the reference's order, on every rank -- ONE exchange per hop
    if (multi) SDB_TRY(comm_allreduce_sum(ctx, *d_out, total, 4, st));
  }
  SDB_CUDA(cudaGetLastError());
  *n_out = total;
  return SDB_OK;
}

// ---- +collect: first-seen de-duplication of one BFS level ----------------------------------------------
__global__ void collect_mark_kernel(const uint32_t* __restrict__ lvl, uint64_t n, const uint8_t* __restrict__ seen,
                                    uint32_t* __restrict__ first_pos) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t v = lvl[p];
  // hubs occur millions of times per level: only positions that could still lower the minimum issue the atomic
  // (a plain load first -- positions are handed out in increasing order, so later duplicates almost always skip it)
  if (!seen[v] && __ldcg(first_pos + v) > (uint32_t)p) atomicMin(first_pos + v, (uint32_t)p);
}
__global__ void collect_flag_kernel(const uint32_t* __restrict__ lvl, uint64_t n, const uint8_t* __restrict__ seen,
                                    const uint32_t* __restrict__ first_pos, uint64_t* __restrict__ keep) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t v = lvl[p];
  keep[p] = (!seen[v] && first_pos[v] == (uint32_t)p) ? 1 : 0;
}
__global__ void collect_compact_kernel(const uint32_t* __restrict__ lvl, uint64_t n, const uint64_t* __restrict__ pos /* n+1 */,
                                       uint8_t* __restrict__ seen, uint32_t* __restrict__ first_pos,
                                       uint32_t* __restrict__ next) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  if (pos[p + 1] != pos[p]) {  // kept
    const uint32_t v = lvl[p];
    next[pos[p]] = v;
    seen[v] = 1;
    first_pos[v] = 0xFFFFFFFFu;
  }
}

// ---- filtered hop: a WHERE condition on the edge records and/or the target records, evaluated by the caller ----------
// into bitmaps (bit i = bit i % 32 of word i / 32).  CSR position p with target t passes iff
// (edge_bits == nullptr || bit p of edge_bits) && (target_bits == nullptr || bit t of target_bits); the result is the
// unfiltered hop's with the failing positions removed, and a per-source limit keeps each source's first n PASSING ones.
//
// The candidate space is the unfiltered hop's output [0, T) (degree_kernel without a limit + exclusive_scan).  It is
// split into equal runs of EXP_TILE-candidate tiles, one run per block of a fixed grid, and filter_kernel walks each run
// twice: the COUNT pass counts the passing candidates per block (and per source when a limit is set), the WRITE pass
// recomputes the flags and writes the passing targets compacted, in order.  T stays on the device, so a hop synchronises
// with the host once, for its output size, and the unfiltered level is never written.
using HopFilter = sdb_hop_filter;  // with device bitmaps; nullptr = no condition on that side

__device__ __forceinline__ bool bit_set(const uint32_t* bits, uint64_t i) { return (__ldg(bits + (i >> 5)) >> (i & 31)) & 1u; }
// the pass flag of CSR position p whose target is t: the one definition every filtered hop and +collect level uses
__device__ __forceinline__ bool hop_pass(const HopFilter& f, uint64_t p, uint32_t t) {
  return (!f.edge_bits || bit_set(f.edge_bits, p)) && (!f.target_bits || bit_set(f.target_bits, t));
}

// COUNT: blk[b] = passing candidates of block b's run; with a limit also src_cnt[i] += passing candidates of source i.
// WRITE: blk = exclusive scan of the COUNT blk (so blk[b] + the passing candidates before a candidate in b's run = its
//        rank among all passing ones); with a limit, src_cnt = exclusive scan of the per-source passing counts and
//        src_out = exclusive scan of min(count, limit): the r-th passing candidate of source i goes to src_out[i] + r
//        when r < limit.
template <bool WRITE>
__global__ void __launch_bounds__(EXP_THREADS) filter_kernel(const uint64_t* __restrict__ row_ptr,
                                                             const uint32_t* __restrict__ col_idx, uint64_t n_rows,
                                                             const uint32_t* __restrict__ frontier, uint64_t n_f,
                                                             const uint64_t* __restrict__ off /* n_f + 1, off[n_f] = T */,
                                                             HopFilter f, uint32_t limit, uint64_t* __restrict__ blk,
                                                             uint64_t* __restrict__ src_cnt,
                                                             const uint64_t* __restrict__ src_out, uint32_t* __restrict__ out) {
  __shared__ uint64_t s_off[EXP_SRC_MAX];
  __shared__ uint64_t s_row[EXP_SRC_MAX];
  __shared__ uint32_t s_cnt[WRITE ? 1 : EXP_SRC_MAX];  // COUNT with a limit: passing candidates per source of the tile
  __shared__ uint64_t s_warp[EXP_THREADS / 32];
  __shared__ uint64_t s_i0, s_i1;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t T = off[n_f];
  const uint64_t n_tiles = (T + EXP_TILE - 1) / EXP_TILE;
  const uint64_t t_end = n_tiles * (blockIdx.x + 1) / gridDim.x;
  uint64_t base = WRITE ? blk[blockIdx.x] : 0;  // WRITE: passing candidates before the current round (block-uniform)
  uint64_t mine = 0;                            // COUNT: passing candidates this thread saw
  for (uint64_t tile = n_tiles * blockIdx.x / gridDim.x; tile < t_end; tile++) {
    const uint64_t o0 = tile * EXP_TILE;
    const uint64_t o1 = o0 + EXP_TILE < T ? o0 + EXP_TILE : T;
    if (threadIdx.x == 0) {
      s_i0 = upper_bound_minus1(off, 0, n_f + 1, o0);
      s_i1 = upper_bound_minus1(off, 0, n_f + 1, o1 - 1);
    }
    __syncthreads();
    const uint64_t i0 = s_i0, i1 = s_i1;
    const bool in_smem = (i1 - i0 + 2) <= (uint64_t)EXP_SRC_MAX;
    if (in_smem) {
      for (uint64_t t = threadIdx.x; t < i1 - i0 + 2; t += EXP_THREADS) {
        const uint64_t i = i0 + t;
        s_off[t] = off[i];
        // a frontier id out of range has degree 0 (degree_kernel flagged it; the hop fails after this pass): never read
        s_row[t] = i < n_f && frontier[i] < n_rows ? row_ptr[frontier[i]] : 0;
        if (!WRITE) s_cnt[t] = 0;
      }
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < EXP_PER_THREAD; u++) {  // every thread runs every round: the warp votes below need all lanes
      const uint64_t o = o0 + (uint64_t)u * EXP_THREADS + threadIdx.x;
      uint64_t src = 0, p = 0;
      uint32_t t = 0;
      bool pass = false;
      if (o < o1) {
        uint64_t start, rbeg;
        if (in_smem) {
          const uint64_t k = upper_bound_minus1(s_off, 0, i1 - i0 + 2, o);
          src = i0 + k;
          start = s_off[k];
          rbeg = s_row[k];
        } else {  // pathological: thousands of zero-degree sources inside this tile
          src = upper_bound_minus1(off, i0, i1 + 2, o);
          start = off[src];
          rbeg = row_ptr[frontier[src]];  // src owns candidate o, so its id is in range
        }
        p = rbeg + (o - start);
        if (f.target_bits) t = __ldg(col_idx + p);
        pass = hop_pass(f, p, t);
      }
      if (!WRITE) {
        mine += pass;
        if (limit) {  // one atomic per (warp, source): a hub's candidates fill whole warps
          const uint32_t peers = __match_any_sync(0xFFFFFFFFu, pass ? src : ~0ull);
          if (pass && lane == (uint32_t)(__ffs(peers) - 1)) {
            if (in_smem) atomicAdd(&s_cnt[src - i0], (uint32_t)__popc(peers));
            else atomicAdd((unsigned long long*)&src_cnt[src], (unsigned long long)__popc(peers));
          }
        }
      } else {
        const uint32_t vote = __ballot_sync(0xFFFFFFFFu, pass);
        if (lane == 0) s_warp[warp] = __popc(vote);
        __syncthreads();
        uint64_t rank = base + __popc(vote & ((1u << lane) - 1u)), round = 0;
        for (uint32_t w = 0; w < EXP_THREADS / 32; w++) {
          if (w < warp) rank += s_warp[w];
          round += s_warp[w];
        }
        if (pass) {
          const uint64_t r = limit ? rank - src_cnt[src] : 0;
          if (r < limit || !limit) {
            // an edge condition alone reads only the targets it writes (a limit drops most passing ones)
            if (!f.target_bits) t = __ldg(col_idx + p);
            out[limit ? src_out[src] + r : rank] = t;
          }
        }
        base += round;
        __syncthreads();  // s_warp is rewritten by the next round
      }
    }
    if (!WRITE && limit && in_smem) {
      __syncthreads();
      for (uint64_t t = threadIdx.x; t < i1 - i0 + 1; t += EXP_THREADS)
        if (s_cnt[t]) atomicAdd((unsigned long long*)&src_cnt[i0 + t], (unsigned long long)s_cnt[t]);
    }
    __syncthreads();  // the next tile rewrites the shared tables
  }
  if (!WRITE) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xFFFFFFFFu, mine, o);
    if (lane == 0) s_warp[warp] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint64_t s = 0;
      for (int w = 0; w < EXP_THREADS / 32; w++) s += s_warp[w];
      blk[blockIdx.x] = s;
    }
  }
}

__global__ void clamp_kernel(const uint64_t* __restrict__ cnt, uint64_t n, uint32_t limit, uint64_t* __restrict__ out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = cnt[i] < limit ? cnt[i] : limit;
}

// the filtered counterpart of hop_device (same contract); the graph is unsharded and f's bitmaps are device memory
static sdb_status hop_filtered(Graph* g, const HopFilter& f, const uint32_t* d_frontier, uint64_t n_f, uint32_t limit,
                               AsyncBuf<uint32_t>* d_out, uint64_t* n_out, cudaStream_t st) {
  Ctx* ctx = g->ctx;
  *n_out = 0;
  if (n_f == 0) return SDB_OK;
  // one run of tiles per resident block; both passes must use the same grid
  int occ_count = 0, occ_write = 0;
  SDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_count, filter_kernel<false>, EXP_THREADS, 0));
  SDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_write, filter_kernel<true>, EXP_THREADS, 0));
  const uint64_t grid = (uint64_t)ctx->sm_count * std::max(1, std::min(occ_count, occ_write));
  AsyncBuf<uint64_t> d_off, d_blk, d_src, d_src_out;
  AsyncBuf<uint32_t> d_err;
  SDB_CUDA(d_off.reserve(n_f + 2, st));
  SDB_CUDA(d_blk.reserve(grid + 1, st));
  SDB_CUDA(d_err.reserve(1, st));
  SDB_CUDA(cudaMemsetAsync(d_err, 0, 4, st));
  if (limit) {
    SDB_CUDA(d_src.reserve(n_f + 1, st));
    SDB_CUDA(d_src_out.reserve(n_f + 1, st));
    SDB_CUDA(cudaMemsetAsync(d_src, 0, sizeof(uint64_t) * n_f, st));
  }
  degree_kernel<<<(unsigned)((n_f + 255) / 256), 256, 0, st>>>(g->d_row_ptr, g->n_rows, 0, g->n_rows, d_frontier, n_f, 0,
                                                               d_off, d_err);
  count_launch(ctx);
  SDB_TRY(exclusive_scan(ctx, d_off, d_off, n_f, d_off + n_f, st));
  filter_kernel<false><<<(unsigned)grid, EXP_THREADS, 0, st>>>(g->d_row_ptr, g->d_col_idx, g->n_rows, d_frontier, n_f, d_off,
                                                                f, limit, d_blk, d_src, nullptr, nullptr);
  count_launch(ctx);
  SDB_TRY(exclusive_scan(ctx, d_blk, d_blk, grid, d_blk + grid, st));
  const uint64_t* d_total = d_blk + grid;
  if (limit) {
    clamp_kernel<<<(unsigned)((n_f + 255) / 256), 256, 0, st>>>(d_src, n_f, limit, d_src_out);
    count_launch(ctx);
    SDB_TRY(exclusive_scan(ctx, d_src, d_src, n_f, d_src + n_f, st));
    SDB_TRY(exclusive_scan(ctx, d_src_out, d_src_out, n_f, d_src_out + n_f, st));
    d_total = d_src_out + n_f;
  }
  uint64_t total = 0;
  uint32_t err = 0;
  SDB_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (err) {
    set_error("graph expand: frontier id out of range (graph has %llu rows)", (unsigned long long)g->n_rows);
    return SDB_EINVAL;
  }
  if (total > 0xFFFFFFF0ull) {
    set_error("graph expand: %llu results exceed the 2^32 frontier limit", (unsigned long long)total);
    return SDB_EOVERFLOW;
  }
  if (total) {
    SDB_CUDA(d_out->reserve(total, st));
    filter_kernel<true><<<(unsigned)grid, EXP_THREADS, 0, st>>>(g->d_row_ptr, g->d_col_idx, g->n_rows, d_frontier, n_f,
                                                                 d_off, f, limit, d_blk, d_src, d_src_out, *d_out);
    count_launch(ctx);
  }
  SDB_CUDA(cudaGetLastError());
  *n_out = total;
  return SDB_OK;
}

}  // namespace sdb

struct sdb_graph : sdb::Graph {};
using namespace sdb;

// the context's pinned staging buffer, grown to `bytes` (nullptr if that fails: the caller copies without it)
static uint8_t* stage_buffer(Ctx* ctx, size_t bytes) {
  return ctx->h_stage.reserve(bytes) == cudaSuccess ? ctx->h_stage.get() : nullptr;
}

extern "C" {

void sdb_graph_destroy(sdb_graph* g);

static sdb_status graph_load(sdb_ctx* ctx, uint64_t n_rows, uint64_t row_lo, uint64_t row_hi, const uint64_t* row_ptr,
                             const uint32_t* col_idx, bool sharded, sdb_graph** out) {
  if (!ctx || !out || !row_ptr || n_rows >= 0xFFFFFFF0ull || row_lo > row_hi || row_hi > n_rows) return SDB_EINVAL;
  *out = nullptr;
  const uint64_t n_local = row_hi - row_lo;
  if (row_ptr[0] != 0) {
    set_error("graph load: row_ptr[0] must be 0 (a shard's slice is rebased to its first row)");
    return SDB_EINVAL;
  }
  const uint64_t n_edges = row_ptr[n_local];
  if (n_edges && !col_idx) return SDB_EINVAL;
  for (uint64_t i = 0; i < n_local; i++)
    if (row_ptr[i + 1] < row_ptr[i]) {
      set_error("row_ptr is not non-decreasing at %llu", (unsigned long long)i);
      return SDB_EINVAL;
    }
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  sdb_graph* g = new sdb_graph();
  g->ctx = ctx;
  g->n_rows = n_rows;
  g->n_edges = n_edges;
  g->row_lo = row_lo;
  g->row_hi = row_hi;
  g->sharded = sharded;
  cudaError_t e = g->d_row_ptr.reserve(n_local + 1);
  if (e == cudaSuccess) e = g->d_col_idx.reserve(n_edges ? n_edges : 1);
  if (e != cudaSuccess) {
    set_error("graph allocation failed: %s", cudaGetErrorString(e));
    sdb_graph_destroy(g);
    return SDB_ENOMEM;
  }
  SDB_CUDA(cudaMemcpyAsync(g->d_row_ptr, row_ptr, sizeof(uint64_t) * (n_local + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (n_edges)
    SDB_CUDA(cudaMemcpyAsync(g->d_col_idx, col_idx, sizeof(uint32_t) * n_edges, cudaMemcpyHostToDevice, ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(ctx->stream));
  {  // range check on the device copy (ADVICE r1): row_ptr consistent with the edge count; do targets stay inside the rows?
    unsigned long long bad[2] = {0, 0};
    const sdb_status rc = csr_check(ctx, g->d_row_ptr, g->d_col_idx, n_local, n_edges, n_rows, bad, "sdb_graph_load_csr", ctx->stream);
    if (rc != SDB_OK || bad[0]) {
      if (rc == SDB_OK) set_error("sdb_graph_load_csr: malformed row_ptr (%llu violations)", bad[0]);
      sdb_graph_destroy(g);
      return rc != SDB_OK ? rc : SDB_EINVAL;
    }
    g->targets_in_rows = bad[1] == 0;  // targets of another table may exceed this table's rows: fine for plain hops
  }
  *out = g;
  return SDB_OK;
}

sdb_status sdb_graph_load_csr(sdb_ctx* ctx, uint64_t n_rows, const uint64_t* row_ptr, const uint32_t* col_idx,
                              sdb_graph** out) {
  return graph_load(ctx, n_rows, 0, n_rows, row_ptr, col_idx, false, out);
}

sdb_status sdb_graph_load_csr_shard(sdb_ctx* ctx, uint64_t n_rows_total, uint64_t row_lo, uint64_t row_hi,
                                    const uint64_t* row_ptr, const uint32_t* col_idx, sdb_graph** out) {
  return graph_load(ctx, n_rows_total, row_lo, row_hi, row_ptr, col_idx, true, out);
}

void sdb_graph_destroy(sdb_graph* g) {
  if (!g) return;
  cudaSetDevice(g->ctx->device);
  delete g;
}

static bool has_filter(const HopFilter* f) { return f && (f->edge_bits || f->target_bits); }

// device-resident core: frontier and result stay in HBM (sdb_graph_expand_device hands the result to the caller).
// filters: nullptr, or one per hop (device bitmaps); a hop without bitmaps runs the unfiltered hop
static sdb_status graph_expand_dev(sdb_graph* const* hops, uint32_t n_hops, const uint32_t* d_frontier, uint64_t n_frontier,
                                   uint32_t per_source_limit, AsyncBuf<uint32_t>* d_out, uint64_t* out_n, cudaStream_t st,
                                   const HopFilter* filters = nullptr) {
  AsyncBuf<uint32_t> d_f;
  uint64_t n_f = n_frontier;
  bool owned = false;  // the caller's frontier is never freed
  for (uint32_t h = 0; h < n_hops && n_f; h++) {
    AsyncBuf<uint32_t> d_next;
    uint64_t n_next = 0;
    if (ctx_cancelled(hops[h]->ctx)) {  // polled once per hop
      set_error("query cancelled");
      return SDB_ECANCELLED;
    }
    const uint32_t* d_in = owned ? d_f.get() : d_frontier;
    if (filters && has_filter(&filters[h]))
      SDB_TRY(hop_filtered(hops[h], filters[h], d_in, n_f, per_source_limit, &d_next, &n_next, st));
    else
      SDB_TRY(hop_device(hops[h], d_in, n_f, per_source_limit, &d_next, &n_next, st));
    d_f = std::move(d_next);
    owned = true;
    n_f = n_next;
  }
  if (!owned && n_f) {  // zero hops: hand back a copy
    SDB_CUDA(d_f.reserve(n_f, st));
    SDB_CUDA(cudaMemcpyAsync(d_f, d_frontier, sizeof(uint32_t) * n_f, cudaMemcpyDeviceToDevice, st));
  }
  *d_out = std::move(d_f);
  *out_n = n_f;
  return SDB_OK;
}

// what the filtered entry points refuse: shard handles, and a target condition on a CSR whose targets leave its rows
// (target_bits has one bit per row)
static sdb_status check_filtered(const sdb_graph* g, const sdb_hop_filter* f, const char* fn) {
  if (g->sharded) {
    set_error("%s: filtered hops are not served on shard handles (sdb_graph_load_csr_shard)", fn);
    return SDB_EUNSUPPORTED;
  }
  if (f && f->target_bits && !g->targets_in_rows) {
    set_error("%s: a target condition needs every target id below the graph's row count", fn);
    return SDB_EINVAL;
  }
  return SDB_OK;
}

// copies host bitmaps to the device: ceil(n_edges / 32) words of edge bits and ceil(n_rows / 32) of target bits per
// graph.  dev[i] holds the device copies of host[i]; bufs owns them.
static sdb_status upload_filters(sdb_graph* const* graphs, const sdb_hop_filter* host, uint32_t n,
                                 std::vector<AsyncBuf<uint32_t>>* bufs, std::vector<HopFilter>* dev, cudaStream_t st) {
  bufs->resize(2 * (size_t)n);
  dev->assign(n, HopFilter{nullptr, nullptr});
  for (uint32_t h = 0; h < n; h++) {
    const uint32_t* src[2] = {host[h].edge_bits, host[h].target_bits};
    const uint64_t words[2] = {(graphs[h]->n_edges + 31) / 32, (graphs[h]->n_rows + 31) / 32};
    const uint32_t* dst[2] = {nullptr, nullptr};
    for (int k = 0; k < 2; k++) {
      if (!src[k] || !words[k]) continue;  // no positions (or no rows) to test: no bitmap needed
      AsyncBuf<uint32_t>& b = (*bufs)[2 * (size_t)h + k];
      SDB_CUDA(b.reserve(words[k], st));
      SDB_CUDA(cudaMemcpyAsync(b, src[k], sizeof(uint32_t) * words[k], cudaMemcpyHostToDevice, st));
      dst[k] = b;
    }
    (*dev)[h] = HopFilter{dst[0], dst[1]};
  }
  return SDB_OK;
}

static sdb_status expand_device_call(sdb_graph* const* hops, const sdb_hop_filter* d_filters, uint32_t n_hops,
                                     const uint32_t* d_frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                     uint32_t** d_out_ids, uint64_t* out_n) {
  Ctx* ctx = hops[0]->ctx;
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  AsyncBuf<uint32_t> d_out;
  SDB_TRY(graph_expand_dev(hops, n_hops, d_frontier, n_frontier, per_source_limit, &d_out, out_n, ctx->stream, d_filters));
  *d_out_ids = d_out.release();
  SDB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SDB_OK;
}

sdb_status sdb_graph_expand_device(sdb_graph* const* hops, uint32_t n_hops, const uint32_t* d_frontier, uint64_t n_frontier,
                                   uint32_t per_source_limit, uint32_t** d_out_ids, uint64_t* out_n) {
  if (!hops || !n_hops || !d_out_ids || !out_n || (n_frontier && !d_frontier)) return SDB_EINVAL;
  *d_out_ids = nullptr;
  *out_n = 0;
  for (uint32_t h = 0; h < n_hops; h++)
    if (!hops[h]) return SDB_EINVAL;
  return expand_device_call(hops, nullptr, n_hops, d_frontier, n_frontier, per_source_limit, d_out_ids, out_n);
}

sdb_status sdb_graph_expand_filtered_device(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                            const uint32_t* d_frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                            uint32_t** d_out_ids, uint64_t* out_n) {
  if (!hops || !n_hops || !d_out_ids || !out_n || (n_frontier && !d_frontier)) return SDB_EINVAL;
  *d_out_ids = nullptr;
  *out_n = 0;
  for (uint32_t h = 0; h < n_hops; h++) {
    if (!hops[h]) return SDB_EINVAL;
    SDB_TRY(check_filtered(hops[h], filters ? &filters[h] : nullptr, "sdb_graph_expand_filtered_device"));
  }
  return expand_device_call(hops, filters, n_hops, d_frontier, n_frontier, per_source_limit, d_out_ids, out_n);
}

void sdb_device_free(sdb_ctx* ctx, void* d_ptr) {
  if (!ctx || !d_ptr) return;
  cudaSetDevice(ctx->device);
  AsyncBuf<uint32_t>::free_released(d_ptr, ctx->stream);
}

// host frontier and result; filters: nullptr or one per hop, host bitmaps (copied for this call)
static sdb_status expand_host_call(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                   const uint32_t* frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                   uint32_t** out_ids, uint64_t* out_n) {
  Ctx* ctx = hops[0]->ctx;
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  std::vector<AsyncBuf<uint32_t>> bits;
  std::vector<HopFilter> d_filters;
  if (filters) SDB_TRY(upload_filters(hops, filters, n_hops, &bits, &d_filters, st));
  AsyncBuf<uint32_t> d_in;
  if (n_frontier) {
    SDB_CUDA(d_in.reserve(n_frontier, st));
    SDB_CUDA(cudaMemcpyAsync(d_in, frontier, sizeof(uint32_t) * n_frontier, cudaMemcpyHostToDevice, st));
  }
  AsyncBuf<uint32_t> d_f;
  uint64_t n_f = 0;
  SDB_TRY(graph_expand_dev(hops, n_hops, d_in, n_frontier, per_source_limit, &d_f, &n_f, st,
                           filters ? d_filters.data() : nullptr));
  d_in.reset();
  if (n_f) {
    uint32_t* h_out = (uint32_t*)malloc(sizeof(uint32_t) * n_f);
    if (!h_out) return SDB_ENOMEM;
    // device -> pinned staging (full PCIe rate) -> caller-owned pageable buffer
    const size_t bytes = sizeof(uint32_t) * n_f;
    void* dst = stage_buffer(ctx, bytes);
    if (!dst) dst = h_out;
    SDB_CUDA(cudaMemcpyAsync(dst, d_f, bytes, cudaMemcpyDeviceToHost, st));
    d_f.reset();
    SDB_CUDA(cudaStreamSynchronize(st));
    if (dst != (void*)h_out) memcpy(h_out, dst, bytes);
    *out_ids = h_out;
    *out_n = n_f;
  } else {
    SDB_CUDA(cudaStreamSynchronize(st));
  }
  return SDB_OK;
}

sdb_status sdb_graph_expand(sdb_graph* const* hops, uint32_t n_hops, const uint32_t* frontier, uint64_t n_frontier,
                            uint32_t per_source_limit, uint32_t** out_ids, uint64_t* out_n) {
  if (!hops || !n_hops || !out_ids || !out_n || (n_frontier && !frontier)) return SDB_EINVAL;
  *out_ids = nullptr;
  *out_n = 0;
  for (uint32_t h = 0; h < n_hops; h++)
    if (!hops[h]) return SDB_EINVAL;
  return expand_host_call(hops, nullptr, n_hops, frontier, n_frontier, per_source_limit, out_ids, out_n);
}

sdb_status sdb_graph_expand_filtered(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                     const uint32_t* frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                     uint32_t** out_ids, uint64_t* out_n) {
  if (!hops || !n_hops || !out_ids || !out_n || (n_frontier && !frontier)) return SDB_EINVAL;
  *out_ids = nullptr;
  *out_n = 0;
  for (uint32_t h = 0; h < n_hops; h++) {
    if (!hops[h]) return SDB_EINVAL;
    SDB_TRY(check_filtered(hops[h], filters ? &filters[h] : nullptr, "sdb_graph_expand_filtered"));
  }
  return expand_host_call(hops, filters, n_hops, frontier, n_frontier, per_source_limit, out_ids, out_n);
}

// +collect; filter: nullptr, or host bitmaps applied at every BFS level (the start set is not filtered)
static sdb_status collect_call(sdb_graph* g, const sdb_hop_filter* filter, const uint32_t* start, uint64_t n_start,
                               uint32_t min_depth, uint32_t max_depth, int inclusive, uint32_t** out_ids, uint64_t* out_n) {
  Ctx* ctx = g->ctx;
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  if (!g->targets_in_rows) {
    set_error("graph collect: this CSR has targets outside its own rows (an edge table into another node table); "
              "+collect needs source and target ids in one id space");
    return SDB_EINVAL;
  }
  for (uint64_t i = 0; i < n_start; i++)
    if (start[i] >= g->n_rows) {
      set_error("graph collect: start id out of range");
      return SDB_EINVAL;
    }
  std::vector<AsyncBuf<uint32_t>> bits;
  std::vector<HopFilter> d_filter;
  sdb_graph* graphs[1] = {g};
  if (filter) SDB_TRY(upload_filters(graphs, filter, 1, &bits, &d_filter, st));
  const bool filtered = filter && has_filter(&d_filter[0]);
  // the stream-ordered temporaries below are released on every return path, then the stream is drained
  struct Drain {
    cudaStream_t st;
    ~Drain() { cudaStreamSynchronize(st); }
  } drain{st};
  const uint64_t nr = g->n_rows ? g->n_rows : 1;
  // every node is emitted at most once (+ the start values): the result is accumulated on the device
  const uint64_t res_cap = g->n_rows + n_start;
  SDB_CUDA(g->d_seen.reserve(nr));
  SDB_CUDA(g->d_first.reserve(nr));
  SDB_CUDA(g->d_res.reserve(res_cap));
  uint8_t* d_seen = g->d_seen;
  uint32_t *d_first = g->d_first, *d_res = g->d_res;
  AsyncBuf<uint32_t> d_f;
  uint64_t n_res = 0;
  SDB_CUDA(cudaMemsetAsync(d_seen, 0, nr, st));
  SDB_CUDA(cudaMemsetAsync(d_first, 0xFF, sizeof(uint32_t) * nr, st));
  uint64_t n_f = n_start;
  if (n_f) {
    SDB_CUDA(d_f.reserve(n_f, st));
    SDB_CUDA(cudaMemcpyAsync(d_f, start, sizeof(uint32_t) * n_f, cudaMemcpyHostToDevice, st));
  }
  if (inclusive && n_start) {  // collect.rs:83-86: the start value is emitted and marked seen only when inclusive
    const uint8_t one = 1;
    for (uint64_t i = 0; i < n_start; i++)
      SDB_CUDA(cudaMemcpyAsync(d_seen + start[i], &one, 1, cudaMemcpyHostToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(d_res, d_f, sizeof(uint32_t) * n_start, cudaMemcpyDeviceToDevice, st));
    n_res = n_start;
    SDB_CUDA(cudaStreamSynchronize(st));  // `one` lives on this stack frame
  }
  uint32_t depth = 0;
  while (n_f && (max_depth == 0 || depth < max_depth)) {
    if (ctx_cancelled(ctx)) {  // polled once per BFS level
      set_error("query cancelled");
      return SDB_ECANCELLED;
    }
    AsyncBuf<uint32_t> d_lvl;
    uint64_t n_lvl = 0;
    if (filtered)
      SDB_TRY(hop_filtered(g, d_filter[0], d_f, n_f, 0, &d_lvl, &n_lvl, st));
    else
      SDB_TRY(hop_device(g, d_f, n_f, 0, &d_lvl, &n_lvl, st));
    d_f.reset();
    n_f = 0;
    if (n_lvl) {
      AsyncBuf<uint64_t> d_pos;
      SDB_CUDA(d_pos.reserve(n_lvl + 2, st));
      const unsigned grid = (unsigned)((n_lvl + 255) / 256);
      collect_mark_kernel<<<grid, 256, 0, st>>>(d_lvl, n_lvl, d_seen, d_first);
      collect_flag_kernel<<<grid, 256, 0, st>>>(d_lvl, n_lvl, d_seen, d_first, d_pos);
      count_launch(ctx, 2);
      SDB_TRY(exclusive_scan(ctx, d_pos, d_pos, n_lvl, d_pos + n_lvl, st));
      uint64_t n_next = 0;
      SDB_CUDA(cudaMemcpyAsync(&n_next, d_pos + n_lvl, 8, cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaStreamSynchronize(st));
      if (n_next) {
        SDB_CUDA(d_f.reserve(n_next, st));
        collect_compact_kernel<<<grid, 256, 0, st>>>(d_lvl, n_lvl, d_pos, d_seen, d_first, d_f);
        count_launch(ctx);
        n_f = n_next;
        if (depth + 1 >= min_depth) {  // nodes below min_depth are traversed but not emitted
          if (n_res + n_next > res_cap) {
            set_error("graph collect: internal result overflow");
            return SDB_EOVERFLOW;
          }
          SDB_CUDA(cudaMemcpyAsync(d_res + n_res, d_f, sizeof(uint32_t) * n_next, cudaMemcpyDeviceToDevice, st));
          n_res += n_next;
        }
      }
    }
    depth++;
  }
  SDB_CUDA(cudaGetLastError());
  if (n_res) {
    uint32_t* h_out = (uint32_t*)malloc(sizeof(uint32_t) * n_res);
    if (!h_out) return SDB_ENOMEM;
    // large results go through the context's pinned staging buffer (pageable D2H is several times slower)
    const size_t bytes = sizeof(uint32_t) * n_res;
    cudaError_t e = cudaSuccess;
    uint8_t* stage = bytes >= (1u << 20) ? stage_buffer(ctx, bytes) : nullptr;
    if (stage) {
      e = cudaMemcpyAsync(stage, d_res, bytes, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (e == cudaSuccess) memcpy(h_out, stage, bytes);
    } else {
      e = cudaMemcpyAsync(h_out, d_res, bytes, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e != cudaSuccess) {
      free(h_out);
      set_error("graph collect: result copy failed: %s", cudaGetErrorString(e));
      return SDB_ECUDA;
    }
    *out_ids = h_out;
    *out_n = n_res;
  }
  return SDB_OK;
}

sdb_status sdb_graph_collect(sdb_graph* g, const uint32_t* start, uint64_t n_start, uint32_t min_depth,
                             uint32_t max_depth, int inclusive, uint32_t** out_ids, uint64_t* out_n) {
  if (!g || !out_ids || !out_n || (n_start && !start)) return SDB_EINVAL;
  *out_ids = nullptr;
  *out_n = 0;
  return collect_call(g, nullptr, start, n_start, min_depth, max_depth, inclusive, out_ids, out_n);
}

sdb_status sdb_graph_collect_filtered(sdb_graph* g, const sdb_hop_filter* filter, const uint32_t* start, uint64_t n_start,
                                      uint32_t min_depth, uint32_t max_depth, int inclusive, uint32_t** out_ids,
                                      uint64_t* out_n) {
  if (!g || !out_ids || !out_n || (n_start && !start)) return SDB_EINVAL;
  *out_ids = nullptr;
  *out_n = 0;
  SDB_TRY(check_filtered(g, filter, "sdb_graph_collect_filtered"));
  return collect_call(g, filter, start, n_start, min_depth, max_depth, inclusive, out_ids, out_n);
}

}  // extern "C"
