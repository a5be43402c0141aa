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
  // diagnostics of the last sdb_graph_collect_batch (sdb_graph_last_collect_table): the pair table's peak bytes, its
  // growths, the level passes an overflow repeated, and the runs of documents split in two
  uint64_t table_peak_bytes = 0;
  uint32_t table_grows = 0, table_repeats = 0, collect_splits = 0;
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

// ---- document boundaries of a batch (sdb_graph_expand_batch / sdb_graph_collect_batch) ------------------------------
// seg[0..n_seg) are positions into a level whose output positions are given by the exclusive scan off (off[n] = total):
// the boundaries move to the next level by one gather.  Each thread reads and writes its own entry, so in place is safe.
__global__ void seg_gather_kernel(const uint64_t* __restrict__ off, uint64_t* seg, uint64_t n_seg) {
  const uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d < n_seg) seg[d] = off[seg[d]];
}
static sdb_status seg_gather(Ctx* ctx, const uint64_t* d_off, uint64_t* d_seg, uint64_t n_seg, cudaStream_t st) {
  seg_gather_kernel<<<(unsigned)((n_seg + 255) / 256), 256, 0, st>>>(d_off, d_seg, n_seg);
  count_launch(ctx);
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

// *d_out: an empty buffer, which receives the next frontier (stays empty when it has no elements).
// d_seg: nullptr, or n_seg document boundaries into the frontier, moved to the output's boundaries
static sdb_status hop_device(Graph* g, const uint32_t* d_frontier, uint64_t n_f, uint32_t limit, AsyncBuf<uint32_t>* d_out,
                             uint64_t* n_out, cudaStream_t st, uint64_t* d_seg = nullptr, uint64_t n_seg = 0) {
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
  if (d_seg) SDB_TRY(seg_gather(ctx, d_off, d_seg, n_seg, st));
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

// the filtered counterpart of hop_device (same contract); the graph is unsharded and f's bitmaps are device memory.
// Document boundaries need the output offset of every source, which only the per-source path has (src_out): with
// d_seg and no limit the hop takes that path with an unbounded limit, i.e. one per-source count per passing candidate
// group and two more scans over the frontier.
static sdb_status hop_filtered(Graph* g, const HopFilter& f, const uint32_t* d_frontier, uint64_t n_f, uint32_t limit,
                               AsyncBuf<uint32_t>* d_out, uint64_t* n_out, cudaStream_t st, uint64_t* d_seg = nullptr,
                               uint64_t n_seg = 0) {
  Ctx* ctx = g->ctx;
  *n_out = 0;
  if (n_f == 0) return SDB_OK;
  if (d_seg && !limit) limit = 0xFFFFFFFFu;
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
    if (d_seg) SDB_TRY(seg_gather(ctx, d_src_out, d_seg, n_seg, st));
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

// ---- batch +collect: first-seen de-duplication per (document, node) pair ----------------------------------------------
// An open-addressing table keyed on (doc << 32) | node holds every pair the call has visited, so its size follows the
// visited pairs, never n_docs x n_rows.  A slot's value is the first level position of its pair while the level is
// marked (PAIR_NONE before any), then PAIR_SEEN once the pair has been kept; level positions stay below 0xFFFFFFF0.
// Insertions reserve a unit of `fill` first and fail (setting the overflow flag) past max_fill < capacity, so probing
// always finds a free slot; the host then grows the table and repeats the pass, which is idempotent.
constexpr unsigned long long PAIR_EMPTY = ~0ull;  // node ids are < 2^32 - 16: no pair has this key
constexpr uint32_t PAIR_NONE = 0xFFFFFFFFu, PAIR_SEEN = 0xFFFFFFFEu;

struct PairTable {
  unsigned long long* keys;
  uint32_t* vals;
  uint64_t mask;                 // capacity - 1 (a power of two)
  unsigned long long* fill;      // [0] reserved slots, [1] overflow flag
  unsigned long long max_fill;
};

__device__ __forceinline__ uint64_t pair_hash(uint64_t k) {  // splitmix64 finaliser
  k ^= k >> 30;
  k *= 0xbf58476d1ce4e5b9ull;
  k ^= k >> 27;
  k *= 0x94d049bb133111ebull;
  return k ^ (k >> 31);
}
// slot of `key`, inserted if absent; ~0 when the table is too full (the overflow flag is set)
__device__ uint64_t pair_insert(const PairTable& t, unsigned long long key) {
  uint64_t s = pair_hash(key) & t.mask;
  for (uint64_t i = 0; i <= t.mask; i++, s = (s + 1) & t.mask) {
    unsigned long long k = __ldcg(t.keys + s);
    if (k == PAIR_EMPTY) {
      if (*(volatile unsigned long long*)(t.fill + 1)) return ~0ull;  // the pass repeats anyway: no more fill atomics
      if (atomicAdd(t.fill, 1ull) >= t.max_fill) {
        atomicAdd(t.fill, ~0ull);  // give the unit back
        t.fill[1] = 1;
        return ~0ull;
      }
      k = atomicCAS(t.keys + s, PAIR_EMPTY, key);
      if (k == PAIR_EMPTY) return s;
      atomicAdd(t.fill, ~0ull);  // another thread took the slot
    }
    if (k == key) return s;
  }
  t.fill[1] = 1;
  return ~0ull;
}
// slot of a pair that was inserted, ~0 if absent
__device__ uint64_t pair_find(const PairTable& t, unsigned long long key) {
  uint64_t s = pair_hash(key) & t.mask;
  for (uint64_t i = 0; i <= t.mask; i++, s = (s + 1) & t.mask) {
    const unsigned long long k = t.keys[s];
    if (k == key) return s;
    if (k == PAIR_EMPTY) return ~0ull;
  }
  return ~0ull;
}
// the document of level position p: seg holds n_docs + 1 boundaries and p < seg[n_docs]
__device__ __forceinline__ unsigned long long pair_key(const uint64_t* seg, uint64_t n_docs, uint64_t p, uint32_t v) {
  return (upper_bound_minus1(seg, 0, n_docs + 1, p) << 32) | v;
}

// +inclusive: the start ids are emitted and marked seen in their own document
__global__ void pair_seed_kernel(const uint32_t* __restrict__ ids, uint64_t n, const uint64_t* __restrict__ seg,
                                 uint64_t n_docs, PairTable t) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint64_t s = pair_insert(t, pair_key(seg, n_docs, p, ids[p]));
  if (s != ~0ull) t.vals[s] = PAIR_SEEN;
}
__global__ void pair_mark_kernel(const uint32_t* __restrict__ lvl, uint64_t n, const uint64_t* __restrict__ seg,
                                 uint64_t n_docs, PairTable t) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint64_t s = pair_insert(t, pair_key(seg, n_docs, p, lvl[p]));
  if (s == ~0ull) return;
  const uint32_t v = __ldcg(t.vals + s);  // PAIR_SEEN is only written between levels
  if (v != PAIR_SEEN && v > (uint32_t)p) atomicMin(t.vals + s, (uint32_t)p);
}
__global__ void pair_flag_kernel(const uint32_t* __restrict__ lvl, uint64_t n, const uint64_t* __restrict__ seg,
                                 uint64_t n_docs, PairTable t, uint64_t* __restrict__ keep) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint64_t s = pair_find(t, pair_key(seg, n_docs, p, lvl[p]));
  keep[p] = s != ~0ull && t.vals[s] == (uint32_t)p;
}
__global__ void pair_compact_kernel(const uint32_t* __restrict__ lvl, uint64_t n, const uint64_t* __restrict__ seg,
                                    uint64_t n_docs, PairTable t, const uint64_t* __restrict__ pos /* n+1 */,
                                    uint32_t* __restrict__ next) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || pos[p + 1] == pos[p]) return;
  const uint32_t v = lvl[p];
  next[pos[p]] = v;
  t.vals[pair_find(t, pair_key(seg, n_docs, p, v))] = PAIR_SEEN;  // kept, so present
}
// re-inserts the pairs of a smaller table (with their values) into a grown one
__global__ void pair_rehash_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                   uint64_t cap, PairTable t) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap || keys[i] == PAIR_EMPTY) return;
  const uint64_t s = pair_insert(t, keys[i]);
  if (s != ~0ull) t.vals[s] = vals[i];
}

// ---- per-document assembly of a batch result ------------------------------------------------------------------------
// cnt[d] += seg[d + 1] - seg[d]
__global__ void seg_count_kernel(const uint64_t* __restrict__ seg, uint64_t n_docs, uint64_t* __restrict__ cnt) {
  const uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d < n_docs) cnt[d] += seg[d + 1] - seg[d];
}
// writes a level's segment d after what earlier levels wrote for document d: out[out_off[d] + done[d] + (p - seg[d])]
__global__ void seg_scatter_kernel(const uint32_t* __restrict__ ids, uint64_t n, const uint64_t* __restrict__ seg,
                                   uint64_t n_docs, const uint64_t* __restrict__ out_off,
                                   const uint64_t* __restrict__ done, uint32_t* __restrict__ out) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint64_t d = upper_bound_minus1(seg, 0, n_docs + 1, p);
  out[out_off[d] + done[d] + (p - seg[d])] = ids[p];
}
// device doc_off check: seg = doc_off clamped to [0, n], *bad = 1 unless doc_off[0] == 0, non-decreasing, doc_off[n_docs] == n
__global__ void seg_check_kernel(const uint64_t* __restrict__ doc_off, uint64_t n_docs, uint64_t n,
                                 uint64_t* __restrict__ seg, uint32_t* __restrict__ bad) {
  const uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d > n_docs) return;
  const uint64_t v = doc_off[d];
  if ((d == 0 && v != 0) || (d == n_docs && v != n) || (d > 0 && v < doc_off[d - 1]) || v > n) *bad = 1;
  seg[d] = v < n ? v : n;
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
// filters: nullptr, or one per hop (device bitmaps); a hop without bitmaps runs the unfiltered hop.
// d_seg: nullptr, or n_seg document boundaries into the frontier, moved hop by hop to the result's boundaries
static sdb_status graph_expand_dev(sdb_graph* const* hops, uint32_t n_hops, const uint32_t* d_frontier, uint64_t n_frontier,
                                   uint32_t per_source_limit, AsyncBuf<uint32_t>* d_out, uint64_t* out_n, cudaStream_t st,
                                   const HopFilter* filters = nullptr, uint64_t* d_seg = nullptr, uint64_t n_seg = 0) {
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
      SDB_TRY(hop_filtered(hops[h], filters[h], d_in, n_f, per_source_limit, &d_next, &n_next, st, d_seg, n_seg));
    else
      SDB_TRY(hop_device(hops[h], d_in, n_f, per_source_limit, &d_next, &n_next, st, d_seg, n_seg));
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

// d_doc_off: nullptr, or n_docs + 1 document boundaries into d_frontier (device), checked on the device; the result's
// boundaries go to d_out_doc_off (device)
static sdb_status expand_device_call(sdb_graph* const* hops, const sdb_hop_filter* d_filters, uint32_t n_hops,
                                     const uint32_t* d_frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                     uint32_t** d_out_ids, uint64_t* out_n, const uint64_t* d_doc_off = nullptr,
                                     uint64_t n_docs = 0, uint64_t* d_out_doc_off = nullptr) {
  Ctx* ctx = hops[0]->ctx;
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  AsyncBuf<uint64_t> d_seg;
  AsyncBuf<uint32_t> d_bad;
  if (d_doc_off) {
    SDB_CUDA(d_seg.reserve(n_docs + 1, st));
    SDB_CUDA(d_bad.reserve(1, st));
    SDB_CUDA(cudaMemsetAsync(d_bad, 0, 4, st));
    seg_check_kernel<<<(unsigned)((n_docs + 256) / 256), 256, 0, st>>>(d_doc_off, n_docs, n_frontier, d_seg, d_bad);
    count_launch(ctx);
    SDB_CUDA(cudaGetLastError());
    // the verdict comes first: a malformed d_doc_off runs no hop, and no hop's status can hide it
    uint32_t bad = 0;
    SDB_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    if (bad) {
      set_error("graph expand batch: doc_off must start at 0, not decrease and end at n_frontier");
      return SDB_EINVAL;
    }
  }
  AsyncBuf<uint32_t> d_out;
  SDB_TRY(graph_expand_dev(hops, n_hops, d_frontier, n_frontier, per_source_limit, &d_out, out_n, st, d_filters, d_seg,
                           n_docs + 1));
  if (d_doc_off)
    SDB_CUDA(cudaMemcpyAsync(d_out_doc_off, d_seg, sizeof(uint64_t) * (n_docs + 1), cudaMemcpyDeviceToDevice, st));
  *d_out_ids = d_out.release();
  SDB_CUDA(cudaStreamSynchronize(st));
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

// host frontier and result; filters: nullptr or one per hop, host bitmaps (copied for this call).  doc_off: nullptr, or
// n_docs + 1 checked document boundaries into frontier (host); the result's boundaries go to out_doc_off (host)
static sdb_status expand_host_call(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                   const uint32_t* frontier, uint64_t n_frontier, uint32_t per_source_limit,
                                   uint32_t** out_ids, uint64_t* out_n, const uint64_t* doc_off = nullptr,
                                   uint64_t n_docs = 0, uint64_t* out_doc_off = nullptr) {
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
  AsyncBuf<uint64_t> d_seg;
  if (doc_off) {
    SDB_CUDA(d_seg.reserve(n_docs + 1, st));
    SDB_CUDA(cudaMemcpyAsync(d_seg, doc_off, sizeof(uint64_t) * (n_docs + 1), cudaMemcpyHostToDevice, st));
  }
  AsyncBuf<uint32_t> d_f;
  uint64_t n_f = 0;
  SDB_TRY(graph_expand_dev(hops, n_hops, d_in, n_frontier, per_source_limit, &d_f, &n_f, st,
                           filters ? d_filters.data() : nullptr, d_seg, n_docs + 1));
  d_in.reset();
  if (doc_off)  // pageable: complete when the synchronisation below returns
    SDB_CUDA(cudaMemcpyAsync(out_doc_off, d_seg, sizeof(uint64_t) * (n_docs + 1), cudaMemcpyDeviceToHost, st));
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

// ---- batches of documents: document d is frontier[doc_off[d] .. doc_off[d + 1]) -----------------------------------------
static sdb_status check_doc_off(const uint64_t* doc_off, uint64_t n_docs, uint64_t n, const char* fn) {
  if (n_docs >= (1ull << 32)) {
    set_error("%s: %llu documents exceed the 2^32 limit", fn, (unsigned long long)n_docs);
    return SDB_EINVAL;
  }
  bool ok = doc_off[0] == 0 && doc_off[n_docs] == n;
  for (uint64_t d = 0; ok && d < n_docs; d++) ok = doc_off[d + 1] >= doc_off[d];
  if (!ok) {
    set_error("%s: doc_off must start at 0, not decrease and end at %llu", fn, (unsigned long long)n);
    return SDB_EINVAL;
  }
  return SDB_OK;
}

// the checks every batch expand shares; filters on shard handles are refused as by the filtered calls
static sdb_status check_expand_batch(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops, const char* fn) {
  for (uint32_t h = 0; h < n_hops; h++) {
    if (!hops[h]) return SDB_EINVAL;
    if (filters) SDB_TRY(check_filtered(hops[h], &filters[h], fn));
  }
  return SDB_OK;
}

sdb_status sdb_graph_expand_batch(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                  const uint32_t* frontier, uint64_t n_frontier, const uint64_t* doc_off, uint64_t n_docs,
                                  uint32_t per_source_limit, uint32_t** out_ids, uint64_t* out_doc_off, uint64_t* out_n) {
  if (!hops || !n_hops || !out_ids || !out_n || !doc_off || !out_doc_off || (n_frontier && !frontier)) return SDB_EINVAL;
  *out_ids = nullptr;
  *out_n = 0;
  SDB_TRY(check_expand_batch(hops, filters, n_hops, "sdb_graph_expand_batch"));
  SDB_TRY(check_doc_off(doc_off, n_docs, n_frontier, "sdb_graph_expand_batch"));
  return expand_host_call(hops, filters, n_hops, frontier, n_frontier, per_source_limit, out_ids, out_n, doc_off, n_docs,
                          out_doc_off);
}

sdb_status sdb_graph_expand_batch_device(sdb_graph* const* hops, const sdb_hop_filter* filters, uint32_t n_hops,
                                         const uint32_t* d_frontier, uint64_t n_frontier, const uint64_t* d_doc_off,
                                         uint64_t n_docs, uint32_t per_source_limit, uint32_t** d_out_ids,
                                         uint64_t* d_out_doc_off, uint64_t* out_n) {
  if (!hops || !n_hops || !d_out_ids || !out_n || !d_doc_off || !d_out_doc_off || (n_frontier && !d_frontier))
    return SDB_EINVAL;
  *d_out_ids = nullptr;
  *out_n = 0;
  SDB_TRY(check_expand_batch(hops, filters, n_hops, "sdb_graph_expand_batch_device"));
  if (n_docs >= (1ull << 32)) {
    set_error("sdb_graph_expand_batch_device: %llu documents exceed the 2^32 limit", (unsigned long long)n_docs);
    return SDB_EINVAL;
  }
  return expand_device_call(hops, filters, n_hops, d_frontier, n_frontier, per_source_limit, d_out_ids, out_n, d_doc_off,
                            n_docs, d_out_doc_off);
}

}  // extern "C"

// the pair table of a batch +collect (PairTable), with the buffers behind it
struct PairTableBufs {
  AsyncBuf<unsigned long long> keys, fill;
  AsyncBuf<uint32_t> vals;
  uint64_t cap = 0;
  PairTable view() { return PairTable{keys, vals, cap - 1, fill, cap / 2}; }
  uint64_t bytes() const { return cap * (sizeof(unsigned long long) + sizeof(uint32_t)); }
};
// a failed device allocation of a batch +collect: SDB_ENOMEM when the device has no room, SDB_ECUDA otherwise
static sdb_status room(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return SDB_OK;
  set_error("graph collect batch: no room for %s: %s", what, cudaGetErrorString(e));
  return e == cudaErrorMemoryAllocation ? SDB_ENOMEM : SDB_ECUDA;
}
static sdb_status table_alloc(PairTableBufs* t, uint64_t cap, cudaStream_t st) {
  SDB_TRY(room(t->keys.reserve(cap, st), "the pair table"));
  SDB_TRY(room(t->vals.reserve(cap, st), "the pair table"));
  SDB_TRY(room(t->fill.reserve(2, st), "the pair table"));
  t->cap = cap;
  SDB_CUDA(cudaMemsetAsync(t->keys, 0xFF, sizeof(unsigned long long) * cap, st));                  // PAIR_EMPTY
  SDB_CUDA(cudaMemsetAsync(t->vals, (int)(PAIR_NONE & 0xFF), sizeof(uint32_t) * cap, st));  // every byte of PAIR_NONE
  SDB_CUDA(cudaMemsetAsync(t->fill, 0, 2 * sizeof(unsigned long long), st));
  return SDB_OK;
}
// a table of cap slots (a larger power of two) holding the same pairs and values
static sdb_status table_grow(Graph* g, PairTableBufs* t, uint64_t cap, cudaStream_t st) {
  PairTableBufs n;
  SDB_TRY(table_alloc(&n, cap, st));
  g->table_peak_bytes = std::max(g->table_peak_bytes, t->bytes() + n.bytes());
  pair_rehash_kernel<<<(unsigned)((t->cap + 255) / 256), 256, 0, st>>>(t->keys, t->vals, t->cap, n.view());
  count_launch(g->ctx);
  SDB_CUDA(cudaGetLastError());
  *t = std::move(n);
  g->table_grows++;
  return SDB_OK;
}
// runs `pass` (idempotent insertions into t) until it fits: a pass that overflows doubles the table and runs again.
// read: extra 8-byte device words copied back with the overflow flag (the level's size), in the same synchronisation
template <class Pass>
static sdb_status table_pass(Graph* g, PairTableBufs* t, cudaStream_t st, Pass pass, const uint64_t* d_read = nullptr,
                             uint64_t* h_read = nullptr) {
  for (;;) {
    SDB_CUDA(cudaMemsetAsync(t->fill.get() + 1, 0, sizeof(unsigned long long), st));
    SDB_TRY(pass(t->view()));
    unsigned long long overflow = 0;
    SDB_CUDA(cudaMemcpyAsync(&overflow, t->fill.get() + 1, 8, cudaMemcpyDeviceToHost, st));
    if (d_read) SDB_CUDA(cudaMemcpyAsync(h_read, d_read, 8, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    if (!overflow) return SDB_OK;
    g->table_repeats++;
    SDB_TRY(table_grow(g, t, 2 * t->cap, st));
  }
}
// SDB_DEBUG_PAIR_TABLE_SLOTS=n caps the table's size before a level (diagnostics: it makes the levels overflow and
// exercises the doubling above); unset, the size before a level is bounded by the device's free memory only
static uint64_t table_size_cap() {
  const char* s = getenv("SDB_DEBUG_PAIR_TABLE_SLOTS");
  const unsigned long long v = s ? strtoull(s, nullptr, 10) : 0;
  return v >= 64 ? (uint64_t)v : ~0ull;
}

struct CollectArgs {
  Graph* g;
  const HopFilter* f;  // device bitmaps, nullptr = unfiltered
  uint32_t min_depth, max_depth;
  int inclusive;
  cudaStream_t st;
};

// +collect of one run of documents: the levels of its documents run together, each document with its own first-seen
// set.  Appends the run's ids to *ids and writes its n_docs + 1 offsets (from 0) to run_off.  The 2^32-id limit holds
// for the whole batch: res_before ids precede this run; *total_overflow says the batch's result exceeded it.
static sdb_status collect_run(const CollectArgs& a, const uint32_t* start, const uint64_t* doc_off, uint64_t n_docs,
                              std::vector<uint32_t>* ids, uint64_t* run_off, uint64_t res_before, bool* total_overflow) {
  Graph* g = a.g;
  Ctx* ctx = g->ctx;
  cudaStream_t st = a.st;
  struct Drain {  // the stream-ordered temporaries below are released on every return path, then the stream is drained
    cudaStream_t st;
    ~Drain() { cudaStreamSynchronize(st); }
  } drain{st};
  const uint64_t n_start = doc_off[n_docs], n_seg = n_docs + 1;
  AsyncBuf<uint64_t> d_seg;  // the current frontier's document boundaries
  SDB_TRY(room(d_seg.reserve(n_seg, st), "the document offsets"));
  SDB_CUDA(cudaMemcpyAsync(d_seg, doc_off, sizeof(uint64_t) * n_seg, cudaMemcpyHostToDevice, st));
  AsyncBuf<uint32_t> d_f;
  uint64_t n_f = n_start;
  if (n_f) {
    SDB_TRY(room(d_f.reserve(n_f, st), "the start ids"));
    SDB_CUDA(cudaMemcpyAsync(d_f, start, sizeof(uint32_t) * n_f, cudaMemcpyHostToDevice, st));
  }
  const uint64_t size_cap = table_size_cap();
  PairTableBufs tab;
  uint64_t cap = 4096;
  while (cap < 4 * n_start && cap < size_cap) cap *= 2;
  SDB_TRY(table_alloc(&tab, cap, st));
  g->table_peak_bytes = std::max(g->table_peak_bytes, tab.bytes());
  // the emitted levels with their document boundaries, assembled per document at the end
  struct Level {
    AsyncBuf<uint32_t> ids;
    AsyncBuf<uint64_t> seg;
    uint64_t n;
  };
  std::vector<Level> levels;
  uint64_t n_res = 0;
  uint64_t n_pairs = a.inclusive ? n_start : 0;  // an upper bound of the pairs in the table
  auto emit = [&](const uint32_t* d_ids, uint64_t n) -> sdb_status {
    if (res_before + n_res + n > 0xFFFFFFF0ull) {
      set_error("graph collect batch: %llu results exceed the 2^32 limit", (unsigned long long)(res_before + n_res + n));
      *total_overflow = true;
      return SDB_EOVERFLOW;
    }
    Level l;
    l.n = n;
    SDB_TRY(room(l.ids.reserve(n, st), "a level's result"));
    SDB_TRY(room(l.seg.reserve(n_seg, st), "a level's result"));
    SDB_CUDA(cudaMemcpyAsync(l.ids, d_ids, sizeof(uint32_t) * n, cudaMemcpyDeviceToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(l.seg, d_seg, sizeof(uint64_t) * n_seg, cudaMemcpyDeviceToDevice, st));
    levels.push_back(std::move(l));
    n_res += n;
    return SDB_OK;
  };
  if (a.inclusive && n_start) {  // collect.rs:83-86: the start values are emitted and marked seen only when inclusive
    SDB_TRY(table_pass(g, &tab, st, [&](PairTable t) -> sdb_status {
      pair_seed_kernel<<<(unsigned)((n_start + 255) / 256), 256, 0, st>>>(d_f, n_start, d_seg, n_docs, t);
      count_launch(ctx);
      SDB_CUDA(cudaGetLastError());
      return SDB_OK;
    }));
    SDB_TRY(emit(d_f, n_start));
  }
  uint32_t depth = 0;
  while (n_f && (a.max_depth == 0 || depth < a.max_depth)) {
    if (ctx_cancelled(ctx)) {  // polled once per BFS level
      set_error("query cancelled");
      return SDB_ECANCELLED;
    }
    AsyncBuf<uint32_t> d_lvl;
    uint64_t n_lvl = 0;
    if (a.f)
      SDB_TRY(hop_filtered(g, *a.f, d_f, n_f, 0, &d_lvl, &n_lvl, st, d_seg, n_seg));
    else
      SDB_TRY(hop_device(g, d_f, n_f, 0, &d_lvl, &n_lvl, st, d_seg, n_seg));
    d_f.reset();
    n_f = 0;
    if (n_lvl) {
      // within the level the first position of each (document, node) pair not seen before is kept
      AsyncBuf<uint64_t> d_pos;
      SDB_TRY(room(d_pos.reserve(n_lvl + 2, st), "a level's positions"));
      const unsigned grid = (unsigned)((n_lvl + 255) / 256);
      // between levels the table grows to hold every pair the level could add at half load, as far as half of the
      // device's free memory allows (the rest is for the next frontier and the emitted levels) -- the largest power of
      // two that fits; a level whose distinct pairs still overflow it doubles it in table_pass
      uint64_t want = tab.cap;
      while (want / 2 < n_pairs + n_lvl && want < size_cap) want *= 2;
      size_t free_b = 0, total_b = 0;
      SDB_CUDA(cudaMemGetInfo(&free_b, &total_b));
      while (want > tab.cap && (want + tab.cap) * (sizeof(unsigned long long) + sizeof(uint32_t)) > free_b / 2) want /= 2;
      while (want > tab.cap) {
        const sdb_status rc = table_grow(g, &tab, want, st);
        if (rc != SDB_ENOMEM) {
          SDB_TRY(rc);
          break;
        }
        want /= 2;
      }
      uint64_t n_next = 0;
      SDB_TRY(table_pass(g, &tab, st, [&](PairTable t) -> sdb_status {
        pair_mark_kernel<<<grid, 256, 0, st>>>(d_lvl, n_lvl, d_seg, n_docs, t);
        pair_flag_kernel<<<grid, 256, 0, st>>>(d_lvl, n_lvl, d_seg, n_docs, t, d_pos);
        count_launch(ctx, 2);
        SDB_CUDA(cudaGetLastError());
        return exclusive_scan(ctx, d_pos, d_pos, n_lvl, d_pos + n_lvl, st);
      }, d_pos + n_lvl, &n_next));
      if (n_next) {
        SDB_TRY(room(d_f.reserve(n_next, st), "the next frontier"));
        pair_compact_kernel<<<grid, 256, 0, st>>>(d_lvl, n_lvl, d_seg, n_docs, tab.view(), d_pos, d_f);
        count_launch(ctx);
        SDB_CUDA(cudaGetLastError());
      }
      SDB_TRY(seg_gather(ctx, d_pos, d_seg, n_seg, st));  // the kept positions' boundaries: the next frontier's
      n_f = n_next;
      n_pairs += n_next;
      if (n_next && depth + 1 >= a.min_depth) SDB_TRY(emit(d_f, n_next));  // below min_depth: traversed, not emitted
    }
    depth++;
  }
  tab = PairTableBufs();
  // per document in level order: out_off = exclusive scan of the per-document totals, then each level's segment d
  // after what the levels before it wrote for d
  AsyncBuf<uint64_t> d_off, d_done;
  AsyncBuf<uint32_t> d_res;
  SDB_TRY(room(d_off.reserve(n_seg, st), "the result offsets"));
  SDB_TRY(room(d_done.reserve(n_seg, st), "the result offsets"));
  SDB_CUDA(cudaMemsetAsync(d_off, 0, sizeof(uint64_t) * n_seg, st));
  SDB_CUDA(cudaMemsetAsync(d_done, 0, sizeof(uint64_t) * n_seg, st));
  const unsigned dgrid = (unsigned)((n_docs + 255) / 256);
  if (n_docs)
    for (const Level& l : levels) seg_count_kernel<<<dgrid, 256, 0, st>>>(l.seg, n_docs, d_off);
  count_launch(ctx, levels.size());
  SDB_TRY(exclusive_scan(ctx, d_off, d_off, n_docs, d_off + n_docs, st));
  if (n_res) {
    SDB_TRY(room(d_res.reserve(n_res, st), "the result"));
    for (Level& l : levels) {
      seg_scatter_kernel<<<(unsigned)((l.n + 255) / 256), 256, 0, st>>>(l.ids, l.n, l.seg, n_docs, d_off, d_done, d_res);
      seg_count_kernel<<<dgrid, 256, 0, st>>>(l.seg, n_docs, d_done);
      count_launch(ctx, 2);
      l.ids.reset();
      l.seg.reset();
    }
  }
  SDB_CUDA(cudaGetLastError());
  const uint64_t base = ids->size();
  ids->resize(base + n_res);
  const size_t bytes = sizeof(uint32_t) * n_res;
  uint8_t* stage = bytes >= (1u << 20) ? stage_buffer(ctx, bytes) : nullptr;
  SDB_CUDA(cudaMemcpyAsync(run_off, d_off, sizeof(uint64_t) * n_seg, cudaMemcpyDeviceToHost, st));
  if (n_res) SDB_CUDA(cudaMemcpyAsync(stage ? (void*)stage : (void*)(ids->data() + base), d_res, bytes, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (stage) memcpy(ids->data() + base, stage, bytes);
  return SDB_OK;
}

// documents [d0, d1) of the batch (doc_off: the batch's offsets); their offsets go to out_off[d0 .. d1] (the batch's).
// Documents are independent: a run that a hop refuses because its level exceeds 2^32 ids, or (unsharded) that finds no
// room on the device, is served as two halves.  On shard handles the level's size is the same on every rank, so every
// rank splits alike; a per-rank allocation failure is not split.
static sdb_status collect_split(const CollectArgs& a, const uint32_t* start, const uint64_t* doc_off, uint64_t d0,
                                uint64_t d1, std::vector<uint32_t>* ids, uint64_t* out_off) {
  std::vector<uint64_t> off(d1 - d0 + 1), run_off(d1 - d0 + 1);
  for (uint64_t i = 0; i <= d1 - d0; i++) off[i] = doc_off[d0 + i] - doc_off[d0];
  const uint64_t base = ids->size();
  bool total_overflow = false;
  const sdb_status rc = collect_run(a, start + doc_off[d0], off.data(), d1 - d0, ids, run_off.data(), base, &total_overflow);
  if (rc == SDB_OK) {
    for (uint64_t i = 0; i <= d1 - d0; i++) out_off[d0 + i] = base + run_off[i];
    return SDB_OK;
  }
  if (d1 - d0 < 2 || total_overflow || !(rc == SDB_EOVERFLOW || (rc == SDB_ENOMEM && !a.g->sharded))) return rc;
  a.g->collect_splits++;
  const uint64_t dm = d0 + (d1 - d0) / 2;
  SDB_TRY(collect_split(a, start, doc_off, d0, dm, ids, out_off));
  return collect_split(a, start, doc_off, dm, d1, ids, out_off);
}

extern "C" {

static sdb_status collect_batch_call(sdb_graph* g, const sdb_hop_filter* filter, const uint32_t* start, uint64_t n_start,
                                     const uint64_t* doc_off, uint64_t n_docs, uint32_t min_depth, uint32_t max_depth,
                                     int inclusive, uint32_t** out_ids, uint64_t* out_doc_off, uint64_t* out_n) {
  Ctx* ctx = g->ctx;
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  if (!g->targets_in_rows) {
    set_error("graph collect batch: this CSR has targets outside its own rows (an edge table into another node table); "
              "+collect needs source and target ids in one id space");
    return SDB_EINVAL;
  }
  for (uint64_t i = 0; i < n_start; i++)
    if (start[i] >= g->n_rows) {
      set_error("graph collect batch: start id out of range");
      return SDB_EINVAL;
    }
  std::vector<AsyncBuf<uint32_t>> bits;
  std::vector<HopFilter> d_filter;
  sdb_graph* graphs[1] = {g};
  if (filter) SDB_TRY(upload_filters(graphs, filter, 1, &bits, &d_filter, st));
  g->table_peak_bytes = 0;
  g->table_grows = g->table_repeats = g->collect_splits = 0;
  const CollectArgs args{g, filter && has_filter(&d_filter[0]) ? &d_filter[0] : nullptr, min_depth, max_depth, inclusive, st};
  std::vector<uint32_t> ids;
  SDB_TRY(collect_split(args, start, doc_off, 0, n_docs, &ids, out_doc_off));
  if (!ids.empty()) {
    uint32_t* h_out = (uint32_t*)malloc(sizeof(uint32_t) * ids.size());
    if (!h_out) return SDB_ENOMEM;
    memcpy(h_out, ids.data(), sizeof(uint32_t) * ids.size());
    *out_ids = h_out;
    *out_n = ids.size();
  }
  return SDB_OK;
}

sdb_status sdb_graph_collect_batch(sdb_graph* g, const sdb_hop_filter* filter, const uint32_t* start, uint64_t n_start,
                                   const uint64_t* doc_off, uint64_t n_docs, uint32_t min_depth, uint32_t max_depth,
                                   int inclusive, uint32_t** out_ids, uint64_t* out_doc_off, uint64_t* out_n) {
  if (!g || !out_ids || !out_n || !doc_off || !out_doc_off || (n_start && !start)) return SDB_EINVAL;
  *out_ids = nullptr;
  *out_n = 0;
  if (filter) SDB_TRY(check_filtered(g, filter, "sdb_graph_collect_batch"));
  SDB_TRY(check_doc_off(doc_off, n_docs, n_start, "sdb_graph_collect_batch"));
  return collect_batch_call(g, filter, start, n_start, doc_off, n_docs, min_depth, max_depth, inclusive, out_ids,
                            out_doc_off, out_n);
}

void sdb_graph_last_collect_table(const sdb_graph* g, uint64_t* peak_bytes, uint32_t* grows, uint32_t* repeated_passes,
                                  uint32_t* splits) {
  uint64_t b = 0;
  uint32_t n[3] = {0, 0, 0};
  if (g) {
    std::lock_guard<std::mutex> guard(g->ctx->mu);  // sdb_graph_collect_batch writes them under the same lock
    b = g->table_peak_bytes;
    n[0] = g->table_grows, n[1] = g->table_repeats, n[2] = g->collect_splits;
  }
  if (peak_bytes) *peak_bytes = b;
  if (grows) *grows = n[0];
  if (repeated_passes) *repeated_passes = n[1];
  if (splits) *splits = n[2];
}

}  // extern "C"
