// screen_tc.cu -- K2: wgmma bf16 / int8 GEMM screen with a fused threshold-filter epilogue (sm_90a).
//
//   scores[q][x] = <q~, x~>  (bf16 or int8 operands, fp32 / s32 accumulation in registers), q = queries (M),
//   x = corpus rows (N)
//
// One CTA = one SM, persistent over work items (corpus tile of 256 rows) x (block of 128 queries):
//   warp 8          TMA producer : cp.async.bulk.tensor 2-D tiles (SWIZZLE_128B) of A (128 x 64) and B (256 x 64)
//                                  into a 4-stage shared-memory ring, completion on mbarriers
//   warpgroups 0, 1 consumers    : each issues wgmma.mma_async m64n256 (K = 16 bf16 / 32 int8 per instruction) for
//                                  its 64 queries of the item, then filters its 64 x 256 accumulator straight from the
//                                  registers: scale by the row's screening norm, compare with the query's threshold
//                                  tau and append the rare survivors to the query's candidate lists -- the 128 x 256
//                                  score tile is never written to memory (at 1024 x 10M it would be 41 GB).
//   warp 9          refiner      : (streaming mode) raises the thresholds WHILE the kernel runs.  Every survivor is also
//                                  counted (fire-and-forget RED) in its query's 256-bin score histogram in L2; the
//                                  refiner of CTA b owns the queries q = b (mod grid), reads their histograms, finds the
//                                  bin in which the count from the top reaches k -- a proof that the k-th best score
//                                  seen so far is at least that bin's lower edge -- and publishes tau = edge - margin.
//                                  The consumers re-read tau (ld.cg, L2) at every work item.  One launch therefore covers
//                                  the whole corpus: no per-pass launches, compactions or host round trips.
//   warp 10         drain        : (int8 threshold passes) the consumers write their survivors into a shared-memory
//                                  ring; this warp appends them to the candidate lists and histograms, so the
//                                  consumers go on to the next item's MMAs instead of waiting on the appends.
// The producer runs up to STAGES k-blocks ahead, so the loads of item i+1 overlap the epilogue of item i.
// The int8 streaming launch with an even number of query blocks runs as 2-CTA clusters that share each corpus tile:
// each CTA's producer multicasts one half of the B tile into both CTAs, and a stage is free once the consumer warps
// of both CTAs have released it.
//
// Replaces, as the *screen*, the distance loop of KnnTopK::execute (exec/operators/knn_topk.rs:185-228);
// exactness is restored by candidates.cu (f64 re-rank + error-bound proof) and exact.cu.
#include <cuda.h>

#include <type_traits>

#include "internal.cuh"

namespace sdb {

namespace tc {
constexpr uint32_t BLOCK_M = 128;   // queries per work item (two warpgroups of 64)
constexpr uint32_t BLOCK_N = 256;   // corpus rows per work item (= TILE_ROWS)
constexpr uint32_t BLOCK_K = 64;    // bf16 elements per smem stage row = 128 bytes = one swizzle atom
constexpr uint32_t WG_M = 64;       // queries per consumer warpgroup (wgmma M)
constexpr uint32_t STAGES = 4;
constexpr uint32_t A_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr uint32_t B_BYTES = BLOCK_N * BLOCK_K * 2;  // 32 KB
constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
constexpr uint32_t CONS_WARPS = 8;                 // two consumer warpgroups
constexpr uint32_t PROD_WARP = CONS_WARPS;         // warp 8
constexpr uint32_t DRAIN_WARP = CONS_WARPS + 2;    // warp 10 (int8 threshold passes only); warp 9 is the refiner
constexpr uint32_t MAX_MBLOCKS = 16;           // queries per launch <= 2048 (the driver splits larger batches)
constexpr uint32_t SUBCAP = 16;                // private candidate slots per (query, CTA, column half) and pass
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 2 * BLOCK_N * 4 + 256 + MAX_MBLOCKS * 256 * 4 + 1024;
static_assert(BLOCK_N == TILE_ROWS, "screen tile must match the pass schedule tile");
static_assert(SMEM_BYTES <= 227 * 1024, "screen CTA must fit the shared memory of one SM");
// The int8 threshold passes (MODE 1, 2) hand their survivors to a drain warp through a ring in shared memory: the
// consumers only find the survivors, the drain warp appends them (sub-list counter, store or spill, histogram RED),
// 32 at a time, while the consumers run the next item's MMAs.  The ring lives in the two screening-norm buffers,
// which these kernels never stage; so the CTA's shared memory, and what it leaves to the tail kernels, is unchanged.
constexpr uint32_t RING = 128;                     // entries: value, corpus row, (sequence << 16 | query)
static_assert(3 * RING * 4 <= 2 * BLOCK_N * 4, "the survivor ring must fit the screening-norm buffers");
static_assert(MAX_MBLOCKS * BLOCK_M <= 0x10000 && RING <= 32 * 1024, "ring tags: 16-bit query and sequence fields");
template <bool INT8, int MODE>
constexpr bool has_drain() { return INT8 && (MODE == 1 || MODE == 2); }
// the other kernels keep 10 warps: an idle 11th warp would take the registers a tail kernel needs beside the screen
template <bool INT8, int MODE>
constexpr uint32_t threads() { return (CONS_WARPS + (has_drain<INT8, MODE>() ? 3 : 2)) * 32; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// work item w -> (corpus tile w / n_mb, query block): the query block is skewed by the tile index so that every CTA
// serves every query block equally often (keeps the per-(query, CTA) private candidate sub-lists evenly filled)
__device__ __forceinline__ uint32_t item_mb(uint32_t w, uint32_t n_mb) { return (w % n_mb + w / n_mb) % n_mb; }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
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
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t c0, uint32_t c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
// the same box written to the same shared-memory offset of both CTAs of a 2-CTA cluster, completing on the mbarrier
// at the same offset in each
__device__ __forceinline__ void tma_load_2d_pair(uint32_t dst, const CUtensorMap* map, uint32_t c0, uint32_t c1,
                                                 uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%2, %3}], [%4], %5;"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar), "h"((uint16_t)0x3)
      : "memory");
}
// arrive on the mbarrier at the same offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cta(uint32_t bar, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(rank));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- wgmma (one warpgroup, M=64 N=256, both operands K-major in shared memory) ---------------------------------------
// Accumulator layout (PTX "wgmma register fragment", m64nNk16): register d[4j + 2i + c] of lane l in warp w of the
// warpgroup holds row 16w + l/4 + 8i, column 8j + 2(l%4) + c.
#define SDB_WG_REGS                                                                                   \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                           \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                  \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                  \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "                  \
  "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "                  \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "                  \
  "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "      \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define SDB_WG8(C, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])
#define SDB_WG128(C)                                                                                     \
  SDB_WG8(C, 0), SDB_WG8(C, 8), SDB_WG8(C, 16), SDB_WG8(C, 24), SDB_WG8(C, 32), SDB_WG8(C, 40), SDB_WG8(C, 48), \
      SDB_WG8(C, 56), SDB_WG8(C, 64), SDB_WG8(C, 72), SDB_WG8(C, 80), SDB_WG8(C, 88), SDB_WG8(C, 96),             \
      SDB_WG8(C, 104), SDB_WG8(C, 112), SDB_WG8(C, 120)

__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " SDB_WG_REGS ", %128, %129, p, 1, 1, 0, 0;\n\t}"
      : SDB_WG128("+f")
      : "l"(a_desc), "l"(b_desc), "r"(acc));
}
__device__ __forceinline__ void wgmma_i8(uint32_t (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 " SDB_WG_REGS ", %128, %129, p;\n\t}"
      : SDB_WG128("+r")
      : "l"(a_desc), "l"(b_desc), "r"(acc));
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; i++) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void acc_fence(uint32_t (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; i++) asm volatile("" : "+r"(d[i])::"memory");
}
#undef SDB_WG128
#undef SDB_WG8
#undef SDB_WG_REGS
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// shared-memory matrix descriptor (Hopper GMMA): K-major, SWIZZLE_128B, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);  // start address
  d |= (uint64_t)1 << 16;                  // leading byte offset (unused for swizzled K-major; canonical 1)
  d |= (uint64_t)(1024 >> 4) << 32;        // stride byte offset: next 8-row core-matrix group
  d |= (uint64_t)1 << 62;                  // SWIZZLE_128B
  return d;
}

// value t (0..63) of row i (0, 1) of this lane's accumulator fragment, and its column in the tile
template <typename Acc>
__device__ __forceinline__ Acc acc_at(const Acc (&acc)[128], int i, int t) {
  return acc[4 * (t >> 1) + 2 * i + (t & 1)];
}
__device__ __forceinline__ uint32_t fragment_col(int t, uint32_t col_l) { return 8 * (t >> 1) + col_l + (t & 1); }
// the same with a run-time t, as a chain of selects: the accumulator stays in registers
template <typename Acc>
__device__ __forceinline__ Acc acc_at_dyn(const Acc (&acc)[128], int i, int t) {
  Acc v = acc[2 * i];
#pragma unroll
  for (int u = 1; u < 64; u++) v = u == t ? acc_at(acc, i, u) : v;
  return v;
}
__device__ __forceinline__ uint32_t ld_volatile(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
__device__ __forceinline__ void st_volatile(uint32_t* p, uint32_t v) { *reinterpret_cast<volatile uint32_t*>(p) = v; }

// The int8 survivor scan of the epilogue is one pass of compares that sets a bit per passing value, then a rolled loop
// over the set bits that writes each survivor into the drain warp's ring (push_survivors); the drain warp runs the
// single copy of append_survivor.  Unrolled over all 64 values of both rows, the append is inlined 128 times (~150 KB
// of code that every scanning warp walks through); rolled, the streaming kernel is ~8x smaller and twice as fast
// (DESIGN.md §5).  The bf16 kernels keep the unrolled scan with the append inlined: at their 168 registers the rolled
// loop spills, and an 11th warp at 168 registers would leave no room for a tail kernel's block beside the screen.

// one survivor (query q = mb * BLOCK_M + row, corpus column col of the tile): appended to the (query, CTA, column
// half) private sub-list, spilling to the query's shared list when that is full; streaming mode also counts it in the
// query's histogram (a fire-and-forget RED)
template <int MODE>
__device__ __forceinline__ void append_survivor(float score, uint32_t q, uint32_t row, uint32_t col, uint32_t row0,
                                                float2 hpv, uint32_t* s_cnt_mb, Cand* __restrict__ cand,
                                                uint32_t* __restrict__ cand_cnt, uint32_t cap, Cand* __restrict__ sub,
                                                uint32_t* hist) {
  const uint32_t half = col >> 7;
  const uint32_t pos = atomicAdd(s_cnt_mb + half * BLOCK_M + row, 1u);
  const uint2 cd = make_uint2(__float_as_uint(score), row0 + col);
  const uint32_t n_slots = gridDim.x * 2;
  if (pos < SUBCAP) {
    *reinterpret_cast<uint2*>(sub + ((size_t)q * n_slots + blockIdx.x * 2 + half) * SUBCAP + pos) = cd;
  } else {  // private slots full: spill to the query's shared list
    const uint32_t p2 = atomicAdd(cand_cnt + q, 1u);
    if (p2 < cap) *reinterpret_cast<uint2*>(cand + (size_t)q * cap + p2) = cd;
  }
  if (MODE == 2) {
    HistParam hp;
    hp.lo = hpv.x;
    hp.inv_w0 = hpv.y;
    hp.w0 = 0.f;
    hp.margin = 0.f;
    atomicAdd(hist + (size_t)q * HIST_BINS + hist_bin(hp, score), 1u);
  }
}

// Warp-collective (every lane of a consumer warp calls it): writes the values of row i that `hits` marks into the
// drain warp's ring.  One shared atomic reserves the warp's entries; they are written in rounds of at most one entry
// per lane, round-major, so a round's entries are consecutive.  Entry e reuses the slot of entry e - RING, so a round
// first waits until the drain has consumed that far.  Every such wait ends.  Take the lowest entry not yet written:
// its round has either passed its wait already, or begins with that entry.  In the second case every entry below it
// is written, the drain consumes written entries in order without waiting on anything else, and a round of at most
// 32 <= RING entries starting there only needs the drain to reach its first entry.  So that entry gets written, and
// by induction so does every reserved entry.
__device__ __forceinline__ void push_survivors(const uint32_t (&acc)[128], int i, uint64_t hits, uint32_t q,
                                               uint32_t row0, uint32_t col_l, uint32_t lane, uint32_t* r_val,
                                               uint32_t* r_row, uint32_t* r_tag, uint32_t* s_ring_tail,
                                               const uint32_t* s_ring_head) {
  const uint32_t total = __reduce_add_sync(0xffffffffu, (uint32_t)__popcll(hits));
  if (total == 0) return;
  uint32_t base = 0;
  if (lane == 0) base = atomicAdd(s_ring_tail, total);
  base = __shfl_sync(0xffffffffu, base, 0);
  const uint32_t lt = (1u << lane) - 1;
  for (uint32_t off = 0; off < total;) {
    const uint32_t act = __ballot_sync(0xffffffffu, hits != 0);
    const uint32_t e = base + off + __popc(act & lt);
    off += __popc(act);
    while ((int)(base + off - RING - ld_volatile(s_ring_head)) > 0) {
    }
    if (hits) {
      const int t = __ffsll((long long)hits) - 1;
      hits &= hits - 1;
      const uint32_t slot = e % RING;
      r_val[slot] = acc_at_dyn(acc, i, t);
      r_row[slot] = row0 + fragment_col(t, col_l);
      __threadfence_block();  // the entry before its tag
      st_volatile(r_tag + slot, e << 16 | q);
    }
  }
}

// MODE 0: pass 0 -- every score of the pass's tiles goes to a fixed slot of the query's main list (tau = -inf)
// MODE 1: threshold pass -- survivors of a fixed tau (legacy multi-pass schedule)
// MODE 2: streaming pass -- tau is re-read at every work item and raised by the refiner warps while the kernel runs
// MODE 3: probe -- nothing is appended; the maximum of every 32-column chunk of every query is written
//         (probe[q][tile * 8 + chunk]).  The chunk maxima belong to DISJOINT row sets, so the k-th largest of them is a
//         lower bound of the k-th best score of the corpus: the seed of the streaming pass's thresholds, at the cost
//         of one round of MMAs and no candidate traffic.
// FILT: filtered batch -- rows a query's filter rejects never reach its lists, its histogram or its chunk maxima.  The
// test sits where a survivor is appended (bf16: the consumer's append; int8: the drain warp, next to the screening-norm
// look-up) and, in the probe, on the one bitmap word of every 32-row chunk.  Pass 0 writes every row; cand_filter_list
// drops the rejected ones there.
// S: the score of the bf16 epilogue (View::sc); the int8 screen scores Score::Cosine alone.
template <Score S, bool INT8, int MODE, bool FILT>
__global__ void __launch_bounds__(threads<INT8, MODE>(), 1)
screen_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const float* __restrict__ snorm, uint32_t k_blocks, uint32_t n_mblocks, uint32_t nq,
                 PassDesc pass, float* tau, Cand* __restrict__ cand,
                 uint32_t* __restrict__ cand_cnt, uint32_t cap, Cand* __restrict__ sub, uint32_t* __restrict__ sub_cnt,
                 uint32_t k, const HistParam* __restrict__ hparam, uint32_t* hist, float* __restrict__ probe,
                 uint32_t probe_stride, uint32_t sleep_min_ns, uint32_t sleep_max_ns, uint32_t pair, FiltArg filt) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B operand tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;                                  // [STAGES][128][64] bf16
  uint8_t* smem_b = smem + STAGES * A_BYTES;               // [STAGES][256][64] bf16
  float* s_snorm = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);  // [2][256]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_snorm + 2 * BLOCK_N);
  uint64_t* full_bar = bars;                      // [STAGES]
  uint64_t* empty_bar = bars + STAGES;            // [STAGES]
  uint32_t* s_done = reinterpret_cast<uint32_t*>(bars + 2 * STAGES);  // consumer warps that have finished
  uint32_t* s_ring_tail = s_done + 1;  // ring entries reserved by the consumers
  uint32_t* s_ring_head = s_done + 2;  // ring entries the drain warp has consumed (its slots may be written again)
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(bars) + 256);  // [n_mblocks][2][128]
  // survivor ring (has_drain only; in the screening-norm buffers): int8 score, corpus row, (sequence << 16 | query)
  uint32_t* r_val = reinterpret_cast<uint32_t*>(s_snorm);
  uint32_t* r_row = r_val + RING;
  uint32_t* r_tag = r_row + RING;
  constexpr bool DRAIN = has_drain<INT8, MODE>();

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // CTA pairs (int8 streaming launch as 2-CTA clusters, even n_mblocks): both CTAs of pair p take the same corpus
  // tiles, CTA `rank` with query block 2 m + rank, and each loads one 128-row half of the B tile into both CTAs, so a
  // work item pulls 192 KB instead of 288 KB from L2.  Work item w then numbers (tile, m) of the pair.
  const bool PAIR = INT8 && MODE == 2 && pair != 0;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0;
  const uint32_t n_mb = PAIR ? n_mblocks / 2 : n_mblocks;  // query blocks (pairs of them) per corpus tile
  const uint32_t w_first = PAIR ? blockIdx.x / 2 : blockIdx.x, w_step = PAIR ? gridDim.x / 2 : gridDim.x;
  const uint32_t n_items = pass.count * n_mb;

  if (DRAIN) {
    // no sequence number matches 0xFFFF before the slot is first written (sequence s lands in slot s % RING)
    for (uint32_t i = threadIdx.x; i < RING; i += blockDim.x) r_tag[i] = 0xFFFF0000u;
  }
  if (threadIdx.x == 0) {
    *s_ring_tail = 0;
    *s_ring_head = 0;
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    for (uint32_t s = 0; s < STAGES; s++) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), PAIR ? 2 * CONS_WARPS : CONS_WARPS);  // one arrive per consumer warp (of both CTAs)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    *s_done = 0;
  }
  for (uint32_t i = threadIdx.x; i < n_mblocks * 256; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  if (PAIR) cluster_sync();  // the peer's barriers are initialised before anything arrives on them or fills them

  if (warp == PROD_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t it = 0;
      for (uint32_t w = w_first; w < n_items; w += w_step) {
        const uint32_t tile = pass_tile(pass, w / n_mb);
        const uint32_t mb = PAIR ? 2 * item_mb(w, n_mb) + rank : item_mb(w, n_mb);
        for (uint32_t kb = 0; kb < k_blocks; kb++, it++) {
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
          // (pair: the stage is free in both CTAs -- the barrier counts the consumer warps of both)
          mbar_wait(smem_u32(&empty_bar[s]), ph ^ 1);
          const uint32_t fb = smem_u32(&full_bar[s]);
          const uint32_t kc = kb * (INT8 ? 2 * BLOCK_K : BLOCK_K);
          mbar_expect_tx(fb, STAGE_BYTES);  // (pair: own A, own B half, the peer's B half)
          tma_load_2d(smem_u32(smem_a + s * A_BYTES), &map_a, kc, mb * BLOCK_M, fb);
          if (PAIR)
            tma_load_2d_pair(smem_u32(smem_b + s * B_BYTES + rank * (B_BYTES / 2)), &map_b, kc,
                             tile * BLOCK_N + rank * (BLOCK_N / 2), fb);
          else
            tma_load_2d(smem_u32(smem_b + s * B_BYTES), &map_b, kc, tile * BLOCK_N, fb);
        }
      }
    }
    __syncwarp();
  } else if (warp < CONS_WARPS) {
    // ===================== consumers (2 warpgroups; warpgroup g = queries 64g..64g+63 of the item) ==========
    const uint32_t ct = threadIdx.x;              // 0..255
    const uint32_t g = warp >> 2;
    const uint32_t row_base = g * WG_M + (warp & 3) * 16 + (lane >> 2);  // rows row_base and row_base + 8
    const uint32_t col_l = 2 * (lane & 3);        // this lane's first column in every group of 8
    constexpr bool pass0 = MODE == 0;             // pass 0: tau = -inf everywhere, positions are deterministic
    using Acc = typename std::conditional<INT8, uint32_t, float>::type;
    Acc acc[128];
    uint32_t it = 0, j = 0;
    // a stage is released to the producer of this CTA and, in a pair, to the peer's, which fills half of it
    auto release = [&](uint32_t s) {
      if (lane == 0) {
        mbar_arrive(smem_u32(&empty_bar[s]));
        if (PAIR) mbar_arrive_cta(smem_u32(&empty_bar[s]), rank ^ 1);
      }
    };
    for (uint32_t w = w_first; w < n_items; w += w_step, j++) {
      const uint32_t tidx = w / n_mb;
      const uint32_t tile = pass_tile(pass, tidx);
      const uint32_t mb = PAIR ? 2 * item_mb(w, n_mb) + rank : item_mb(w, n_mb);
      const uint32_t row0 = tile * BLOCK_N;
      // thresholds of this thread's two queries (L2: sees the refiners' updates); the loads complete under the MMAs
      float my_tau[2];
      float2 my_hp[2];
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const uint32_t q = mb * BLOCK_M + row_base + 8 * i;
        my_tau[i] = __int_as_float(0x7f800000);
        my_hp[i] = make_float2(0.f, 0.f);
        if (q < nq) {
          my_tau[i] = __ldcg(tau + q);
          if (MODE == 2) my_hp[i] = __ldg(reinterpret_cast<const float2*>(hparam + q));
        }
      }
      float* sn = s_snorm + (j & 1) * BLOCK_N;
      if (!INT8 || MODE == 3) {
        // stage this tile's screening norms (safe: every consumer thread passed the named barrier of item j-1 only
        // after finishing item j-2, the previous user of this buffer)
        sn[ct] = __ldg(snorm + row0 + ct);
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }

      // ---- MMAs: one k-block in flight behind the one being issued ----
      const uint32_t a_off = g * (WG_M * 128);  // this warpgroup's 64 rows of the A stage
      for (uint32_t kb = 0; kb < k_blocks; kb++, it++) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        mbar_wait(smem_u32(&full_bar[s]), ph);
        const uint64_t da = make_desc(smem_u32(smem_a + s * A_BYTES + a_off));
        const uint64_t db = make_desc(smem_u32(smem_b + s * B_BYTES));
        wgmma_fence();
        acc_fence(acc);
#pragma unroll
        for (uint32_t kk = 0; kk < 4; kk++) {
          // advance 32 bytes (16 bf16 / 32 int8) inside the 128-byte swizzle atom: +2 in the (>>4) address field
          if constexpr (INT8) wgmma_i8(acc, da + 2 * kk, db + 2 * kk, (kb | kk) != 0);
          else wgmma_bf16(acc, da + 2 * kk, db + 2 * kk, (kb | kk) != 0);
        }
        wgmma_commit();
        acc_fence(acc);
        if (kb > 0) {
          wgmma_wait<1>();  // the previous k-block's MMAs have read their stage
          release((it - 1) % STAGES);
        }
      }
      wgmma_wait<0>();
      acc_fence(acc);
      release((it - 1) % STAGES);

      // ---- epilogue straight from the registers ----
      if constexpr (!INT8) {
#pragma unroll
        for (int jj = 0; jj < 32; jj++) {
          const float2 n2 = *reinterpret_cast<const float2*>(sn + 8 * jj + col_l);
#pragma unroll
          for (int i = 0; i < 2; i++) {
            float& a0 = acc[4 * jj + 2 * i];
            float& a1 = acc[4 * jj + 2 * i + 1];
            if constexpr (S == Score::Dot) {
              // the dot itself; the staged norm still marks invalid rows (NaN: skipped, special, padding), whose score
              // becomes that NaN.  (A select, not acc + (n - n): a valid COSINE row's 1/|x| may be +inf in f32.)
              a0 = n2.x == n2.x ? a0 : n2.x;
              a1 = n2.y == n2.y ? a1 : n2.y;
            } else if constexpr (S == Score::EuclidFar) {
              a0 = fmaf(2.f, a0, n2.x);  // |x|^2 - 2 x.q against the copy of -q (NaN norm: NaN score)
              a1 = fmaf(2.f, a1, n2.y);
            } else {
              a0 = S == Score::Cosine ? a0 * n2.x : fmaf(2.f, a0, -n2.x);
              a1 = S == Score::Cosine ? a1 * n2.y : fmaf(2.f, a1, -n2.y);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const uint32_t row = row_base + 8 * i;
        const uint32_t q = mb * BLOCK_M + row;
        if (MODE == 3) {
          // maximum of every 32-column chunk: 8 values per lane, the quad of lanes sharing the row covers the chunk
          // FILT: chunk h's 32 rows are word h of the tile's 8 words of the query's bitmap (row0 is a multiple of 256);
          // lane j of the quad holds words j and j + 4, and the quad exchanges them per chunk
          uint32_t fw_lo = 0u, fw_hi = 0u;
          if constexpr (FILT) {
            const uint32_t w = (row0 >> 5) + (lane & 3u);
            if (q < nq) {
              const uint32_t* fb = filt.bits + (size_t)__ldg(filt.qf + q) * filt.words;
              if (w < filt.words) fw_lo = __ldg(fb + w);
              if (w + 4 < filt.words) fw_hi = __ldg(fb + w + 4);
            }
          }
#pragma unroll
          for (int h = 0; h < 8; h++) {
            float m = __int_as_float(0xff800000);  // -inf: no valid row in the chunk
            uint32_t fw = 0xffffffffu;
            if constexpr (FILT) fw = __shfl_sync(0xffffffffu, h < 4 ? fw_lo : fw_hi, (lane & ~3u) | (uint32_t)(h & 3));
#pragma unroll
            for (int jj = 4 * h; jj < 4 * h + 4; jj++) {
#pragma unroll
              for (int c = 0; c < 2; c++) {
                if (FILT && !((fw >> (8 * (jj - 4 * h) + col_l + c)) & 1u)) continue;
                if constexpr (INT8) {
                  // invalid rows (NaN screening norm) score 0 in the integer screen: they must not pose as a score
                  const float snv = sn[8 * jj + col_l + c];
                  if (snv == snv) m = fmaxf(m, __int2float_rd((int)acc[4 * jj + 2 * i + c]));
                } else {
                  m = fmaxf(m, acc[4 * jj + 2 * i + c]);  // fmaxf drops NaNs
                }
              }
            }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            if ((lane & 3) == 0 && q < nq) probe[(size_t)q * probe_stride + tidx * 8 + h] = m;
          }
        } else if (pass0) {
          if (q < nq) {  // every (finite or NaN) score goes to its fixed slot; compaction drops the NaNs
            Cand* my_cand = cand + (size_t)q * cap + (size_t)tidx * BLOCK_N;
#pragma unroll
            for (int jj = 0; jj < 32; jj++) {
              const uint32_t col = 8 * jj + col_l;
              float s0, s1;
              if constexpr (INT8) {
                s0 = __int2float_rn((int)acc[4 * jj + 2 * i]);
                s1 = __int2float_rn((int)acc[4 * jj + 2 * i + 1]);
              } else {
                s0 = acc[4 * jj + 2 * i];
                s1 = acc[4 * jj + 2 * i + 1];
              }
              *reinterpret_cast<uint2*>(my_cand + col) = make_uint2(__float_as_uint(s0), row0 + col);
              *reinterpret_cast<uint2*>(my_cand + col + 1) = make_uint2(__float_as_uint(s1), row0 + col + 1);
            }
          }
        } else {
          // survivors are rare: one max over the lane's 64 values decides whether the lane scans them
          uint32_t* s_cnt_mb = s_cnt + mb * 256;
          if constexpr (INT8) {
            // integer threshold: acc >= tau  <=>  acc >= ceil(tau)
            const float ct_ = ceilf(my_tau[i]);
            const int tau_i = ct_ >= 2147483520.f ? 0x7fffffff : (ct_ <= -2147483520.f ? (int)0x80000000 : (int)ct_);
            int m = (int)0x80000000;
#pragma unroll
            for (int jj = 0; jj < 32; jj++) m = max(m, max((int)acc[4 * jj + 2 * i], (int)acc[4 * jj + 2 * i + 1]));
            if (__any_sync(0xffffffffu, m >= tau_i)) {
              uint64_t hits = 0;
              if (m >= tau_i) {
#pragma unroll
                for (int t = 0; t < 64; t++)
                  if ((int)acc_at(acc, i, t) >= tau_i) hits |= 1ull << t;
                if constexpr (FILT) {
                  // rejected rows never reach the ring: while a selective filter keeps tau low, they would flood it.
                  // Values 8h .. 8h+7 lie in the tile's 32-row chunk h (word h of the query's 8 bitmap words), at bits
                  // col_l + {0, 1, 8, 9, 16, 17, 24, 25} of it.
                  // Only for batches with selective filters (filt.mask_hits): with dense ones the drain warp's test is
                  // cheaper.
                  if (filt.mask_hits && hits && q < nq) {
                    const uint32_t* fb = filt.bits + (size_t)__ldg(filt.qf + q) * filt.words + (row0 >> 5);
                    const uint32_t nw = filt.words > (row0 >> 5) ? filt.words - (row0 >> 5) : 0u;
                    uint64_t keep = 0;
#pragma unroll 1
                    for (uint32_t h = 0; h < 8; h++) {
                      if (h >= nw || !((hits >> (8 * h)) & 0xFFull)) continue;
                      const uint32_t g = __ldg(fb + h) >> col_l;
                      const uint32_t m8 = (g & 3u) | ((g >> 6) & 0xCu) | ((g >> 12) & 0x30u) | ((g >> 18) & 0xC0u);
                      keep |= (uint64_t)m8 << (8 * h);
                    }
                    hits &= keep;
                  }
                }
              }
              push_survivors(acc, i, hits, q, row0, col_l, lane, r_val, r_row, r_tag, s_ring_tail, s_ring_head);
            }
          } else {
            float m = __int_as_float(0xff800000);
#pragma unroll
            for (int jj = 0; jj < 32; jj++) m = fmaxf(m, fmaxf(acc[4 * jj + 2 * i], acc[4 * jj + 2 * i + 1]));
            if (m >= my_tau[i]) {
#pragma unroll
              for (int jj = 0; jj < 32; jj++) {
#pragma unroll
                for (int c = 0; c < 2; c++) {
                  const float v = acc[4 * jj + 2 * i + c];
                  if (v >= my_tau[i] && (!FILT || filt_pass(filt, q, row0 + 8 * jj + col_l + c)))  // NaN never passes
                    append_survivor<MODE>(v, q, row, 8 * jj + col_l + c, row0, my_hp[i], s_cnt_mb, cand, cand_cnt,
                                          cap, sub, hist);
                }
              }
            }
          }
        }
      }
    }
    if (DRAIN) {
      // this warp's ring entries are written; once all consumer warps are done the drain warp empties the ring
      __syncwarp();
      __threadfence_block();
      if (lane == 0) atomicAdd(s_done, 1u);
    }
    // publish the private append counters: slot (CTA, column half) of every query
    if (MODE == 1 || MODE == 2) {
      if (DRAIN) asm volatile("bar.sync 2, 288;" ::: "memory");  // with the drain warp: every survivor is appended
      else asm volatile("bar.sync 1, 256;" ::: "memory");
      const uint32_t n_slots = gridDim.x * 2;
      const uint32_t half = ct / BLOCK_M, row = ct % BLOCK_M;
      for (uint32_t mb = 0; mb < n_mblocks; mb++) {
        const uint32_t qq = mb * BLOCK_M + row;
        if (qq < nq) sub_cnt[(size_t)qq * n_slots + blockIdx.x * 2 + half] = s_cnt[mb * 256 + half * BLOCK_M + row];
      }
    }
    __syncwarp();
    if (!DRAIN && lane == 0) atomicAdd(s_done, 1u);
  } else if (warp == DRAIN_WARP) {
    // ===================== drain (int8 threshold passes): append the survivors of the ring, 32 at a time ==========
    if (DRAIN) {
      uint32_t head = 0;  // entries consumed
      for (;;) {
        const uint32_t e = head + lane, slot = e % RING;
        const uint32_t tag = ld_volatile(r_tag + slot);
        const uint32_t ready = __ballot_sync(0xffffffffu, (tag >> 16) == (e & 0xFFFFu));
        const uint32_t n = ready == 0xffffffffu ? 32 : __ffs(~ready) - 1;  // consecutive written entries
        if (n == 0) {
          // finished: every consumer warp is done (its entries are reserved and written) and all are consumed
          uint32_t fin = 0;
          if (lane == 0 && ld_volatile(s_done) == CONS_WARPS) {
            __threadfence_block();
            fin = ld_volatile(s_ring_tail) == head;
          }
          if (__shfl_sync(0xffffffffu, fin, 0)) break;
          __nanosleep(32);  // leave the issue slots to the consumers of this SM sub-partition
          continue;
        }
        __threadfence_block();  // the entries after their tags
        if (lane < n) {
          const int v = (int)r_val[slot];
          const uint32_t grow = r_row[slot], q = tag & 0xFFFFu;
          const uint32_t col = grow % BLOCK_N, row = q % BLOCK_M;
          // invalid rows (skipped / special / padding) are all-zero in the int8 copy and score exactly 0: only a
          // zero score needs the look-up of the row's screening norm
          if ((v != 0 || __ldg(snorm + grow) == __ldg(snorm + grow)) && (!FILT || filt_pass(filt, q, grow))) {
            const float2 hpv = MODE == 2 ? __ldg(reinterpret_cast<const float2*>(hparam + q)) : make_float2(0.f, 0.f);
            append_survivor<MODE>(__int2float_rn(v), q, row, col, grow - col, hpv, s_cnt + q / BLOCK_M * 256, cand,
                                  cand_cnt, cap, sub, hist);
          }
        }
        __syncwarp();
        __threadfence_block();  // the entries are read before their slots are handed back
        head += n;
        if (lane == 0) st_volatile(s_ring_head, head);
      }
      asm volatile("bar.sync 2, 288;" ::: "memory");
    }
  } else {
    // ===================== refiner (streaming mode): raise the thresholds of the queries this CTA owns ==========
    if (MODE == 2) {
      volatile uint32_t* done = s_done;
      const uint32_t stride = gridDim.x;
      uint32_t n_own = nq > blockIdx.x ? (nq - blockIdx.x + stride - 1) / stride : 0;
      if (n_own > 32) n_own = 32;  // (tiny grids only; the rest keeps its seed threshold)
      float my_tau = __int_as_float(0xff800000);  // lane j: the threshold last published for owned query j
      if (lane < n_own) my_tau = __ldcg(tau + blockIdx.x + lane * stride);
      uint32_t sleep_ns = sleep_min_ns;
      while (*done < CONS_WARPS) {
        bool any = false;
        for (uint32_t j = 0; j < n_own; j++) {
          const uint32_t q = blockIdx.x + j * stride;
          const uint4* hq = reinterpret_cast<const uint4*>(hist + (size_t)q * HIST_BINS) + lane * 2;
          const uint4 ha = __ldcg(hq), hb = __ldcg(hq + 1);  // bins lane*8 .. lane*8+7
          const uint32_t c[8] = {ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w};
          uint32_t sum = 0;
#pragma unroll
          for (int i = 0; i < 8; i++) sum += c[i];
          uint32_t incl = sum;  // suffix sum over lanes: higher lanes hold higher bins
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
            if (lane + o < 32) incl += t;
          }
          const uint32_t above = incl - sum;
          const bool mine = above < k && k <= incl;  // the count from the top reaches k inside this lane's bins
          const uint32_t who = __ballot_sync(0xffffffffu, mine);
          if (who == 0) continue;  // fewer than k survivors counted so far
          uint32_t bstar = 0;
          if (mine) {
            uint32_t acc = above;
#pragma unroll
            for (int i = 7; i >= 0; i--) {
              acc += c[i];
              if (acc >= k) {
                bstar = lane * 8 + i;
                break;
              }
            }
          }
          bstar = __shfl_sync(0xffffffffu, bstar, __ffs(who) - 1);
          const float4 hv = __ldg(reinterpret_cast<const float4*>(hparam + q));
          HistParam hp;
          hp.lo = hv.x;
          hp.inv_w0 = hv.y;
          hp.w0 = hv.z;
          hp.margin = hv.w;
          // >= k rows with score >= edge(bstar) exist (2 % of a bin + 2e-6 relative absorb the rounding of hist_bin)
          const double e0 = hist_edge(hp, bstar), e1 = hist_edge(hp, bstar + 1);
          const float tn = __double2float_rd(e0 - (double)hp.margin - 0.02 * (e1 - e0) - 2e-6 * fabs(e0));
          const float told = __shfl_sync(0xffffffffu, my_tau, j);
          if (tn > told) {
            if (lane == j) my_tau = tn;
            if (lane == 0) __stcg(tau + q, tn);
            any = true;
          }
        }
        sleep_ns = any ? sleep_min_ns : (sleep_ns * 2 < sleep_max_ns ? sleep_ns * 2 : sleep_max_ns);
        __nanosleep(sleep_ns);
      }
    }
  }
  __syncthreads();
  if (PAIR) cluster_sync();  // the peer's last remote arrivals on this CTA's barriers have landed
}
}  // namespace tc

// ---- host side ------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode(Ctx* ctx) {
  if (!ctx->encode_tiled) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      fn = nullptr;
    ctx->encode_tiled = fn;
  }
  return reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled);
}

static sdb_status make_map(Ctx* ctx, CUtensorMap* map, const void* base, uint64_t rows, uint32_t dim_pad,
                           uint32_t box_rows, bool stream_once, bool int8 = false) {
  EncodeTiledFn enc = get_encode(ctx);
  if (!enc) {
    set_error("cuTensorMapEncodeTiled driver entry point not available");
    return SDB_ECUDA;
  }
  cuuint64_t gdim[2] = {dim_pad, rows};
  cuuint64_t gstride[1] = {(cuuint64_t)dim_pad * (int8 ? 1 : 2)};
  cuuint32_t box[2] = {int8 ? 2 * tc::BLOCK_K : tc::BLOCK_K, box_rows};  // 128 bytes per row either way
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, int8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   stream_once ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d)", (int)r);
    return SDB_ECUDA;
  }
  return SDB_OK;
}

bool screen_tc_available() { return true; }

sdb_status screen_tc_init_device(Ctx* ctx) {
#define SET_SMEM1(SC, I8, MODE, F) \
  SDB_CUDA(cudaFuncSetAttribute(tc::screen_tc_kernel<SC, I8, MODE, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::SMEM_BYTES))
#define SET_SMEM(SC, I8, MODE) SET_SMEM1(SC, I8, MODE, false); SET_SMEM1(SC, I8, MODE, true)
  SET_SMEM(Score::Cosine, false, 0); SET_SMEM(Score::Cosine, false, 1); SET_SMEM(Score::Cosine, false, 2); SET_SMEM(Score::Cosine, false, 3);
  SET_SMEM(Score::Euclid, false, 0); SET_SMEM(Score::Euclid, false, 1); SET_SMEM(Score::Euclid, false, 2); SET_SMEM(Score::Euclid, false, 3);
  SET_SMEM(Score::Dot, false, 0); SET_SMEM(Score::Dot, false, 1); SET_SMEM(Score::Dot, false, 2); SET_SMEM(Score::Dot, false, 3);
  SET_SMEM(Score::EuclidFar, false, 0); SET_SMEM(Score::EuclidFar, false, 1); SET_SMEM(Score::EuclidFar, false, 2);
  SET_SMEM(Score::EuclidFar, false, 3);
  SET_SMEM(Score::Cosine, true, 0); SET_SMEM(Score::Cosine, true, 1); SET_SMEM(Score::Cosine, true, 2); SET_SMEM(Score::Cosine, true, 3);
#undef SET_SMEM
#undef SET_SMEM1
  // how many 2-CTA clusters of the int8 streaming screen are resident at once (pairs must share a GPC, so this can be
  // fewer than half the SMs): the pair launch is persistent only if its grid is all resident
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((uint32_t)ctx->sm_count & ~1u);
  cfg.blockDim = dim3(tc::threads<true, 2>());
  cfg.dynamicSmemBytes = tc::SMEM_BYTES;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int clusters = 0;
  SDB_CUDA(cudaOccupancyMaxActiveClusters(&clusters, tc::screen_tc_kernel<Score::Cosine, true, 2, false>, &cfg));
  ctx->tc_pair_ctas = 2 * clusters;
  return SDB_OK;
}

sdb_status screen_tc_pass(const Corpus* c, Scratch& s, const FiltArg& filt, uint32_t nq, uint32_t k, const PassDesc& p,
                          bool int8, int mode, cudaStream_t st, const View& v) {
  if (p.count == 0) return SDB_OK;
  Ctx* ctx = c->ctx;
  const Score sc = v.sc;
  // (PEARSON corpora hold centred copies (corpus.cu) and centred, negated queries (prep_queries): Score::Cosine)
  if (int8 ? (!c->d_i8 || sc != Score::Cosine || v.cross) : !c->d_bf16) {
    set_error("tensor-core screen: the %s screen copy is not available for this corpus",
              int8 ? "int8 (cosine and pearson scores only)" : "bf16");
    return SDB_EUNSUPPORTED;
  }
  const uint64_t n_pad = (c->n + TILE_ROWS - 1) / TILE_ROWS * TILE_ROWS;
  // refiner pacing: it re-reads its queries' histograms at most every sleep_min ns while thresholds move, backing off
  // to sleep_max when they do not
  const uint32_t sleep_min = 512, sleep_max = 8192;
  const uint32_t k_blocks = int8 ? c->dim_pad8 / (2 * tc::BLOCK_K) : c->dim_pad / tc::BLOCK_K;
  // every launch uses the same grid so that the (CTA, half) slot numbering of the private sub-lists is stable
  const uint32_t chunk_q = tc::MAX_MBLOCKS * tc::BLOCK_M;
  const uint32_t nq0 = nq < chunk_q ? nq : chunk_q;
  const uint32_t mb0 = (nq0 + tc::BLOCK_M - 1) / tc::BLOCK_M;
  const uint32_t mb_last = (nq - (nq - 1) / chunk_q * chunk_q + tc::BLOCK_M - 1) / tc::BLOCK_M;
  uint32_t grid = (uint32_t)ctx->sm_count;
  {
    const uint64_t items0 = (uint64_t)p.count * mb0;
    if (grid > items0) grid = (uint32_t)items0;
  }
  // the int8 streaming launch runs as CTA pairs sharing each corpus tile when every chunk has an even number of
  // query blocks; its grid is the resident pairs
  uint32_t pair = 0;
  if (int8 && mode == 2 && mb0 % 2 == 0 && mb_last % 2 == 0) {
    const uint32_t g2 = (grid < (uint32_t)ctx->tc_pair_ctas ? grid : (uint32_t)ctx->tc_pair_ctas) & ~1u;
    if (g2 >= 2) {
      grid = g2;
      pair = 1;
    }
  }
  CUtensorMap map_b;  // (pair: each CTA loads a 128-row half of the tile)
  if (int8) SDB_TRY(make_map(ctx, &map_b, c->d_i8, n_pad, c->dim_pad8, pair ? tc::BLOCK_N / 2 : tc::BLOCK_N, true, true));
  else SDB_TRY(make_map(ctx, &map_b, c->d_bf16, n_pad, c->dim_pad, tc::BLOCK_N, true));
  if (mode == 3 && p.count * 8 > PROBE_STRIDE) {
    set_error("screen_tc_pass: probe of %u tiles exceeds the probe buffer", p.count);
    return SDB_EINVAL;
  }
  if (mode != 3) s.last_slots = grid * 2;
  const uint32_t slots = grid * 2;
  for (uint32_t q0 = 0; q0 < nq; q0 += chunk_q) {
    const uint32_t nqc = nq - q0 < chunk_q ? nq - q0 : chunk_q;
    const uint32_t nq_pad = (nqc + tc::BLOCK_M - 1) / tc::BLOCK_M * tc::BLOCK_M;
    const uint32_t n_mblocks = nq_pad / tc::BLOCK_M;
    CUtensorMap map_a;
    if (int8) SDB_TRY(make_map(ctx, &map_a, s.d_q8 + (size_t)q0 * c->dim_pad8, nq_pad, c->dim_pad8, tc::BLOCK_M, false, true));
    else SDB_TRY(make_map(ctx, &map_a, s.d_qbf16 + (size_t)q0 * c->dim_pad, nq_pad, c->dim_pad, tc::BLOCK_M, false));
    float* tau = s.d_tau + q0;
    Cand* cand = s.d_cand + (size_t)q0 * s.sc_cap;
    uint32_t* ccnt = s.d_cand_cnt + q0;
    Cand* sub = s.d_sub + (size_t)q0 * slots * tc::SUBCAP;
    uint32_t* scnt = s.d_sub_cnt + (size_t)q0 * slots;
    const HistParam* hp = s.d_hparam + q0;
    uint32_t* hist = s.d_hist + (size_t)q0 * HIST_BINS;
    // the screen is launched at the highest priority: when the previous batch's screen retires, the blocks of THIS
    // launch are placed before the queued blocks of that batch's tail kernels (which fit beside a screen CTA anyway),
    // instead of waiting behind two 13 KB selection blocks per SM
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.dynamicSmemBytes = tc::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributePriority;
    attr[0].val.priority = ctx->prio_high;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = pair ? 2 : 1;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pair ? 2 : 1;
    float* probe_ptr = s.d_probe + (size_t)q0 * PROBE_STRIDE;
    const uint32_t probe_stride = PROBE_STRIDE, cap_arg = s.sc_cap;
    const float* snorm_arg = view_snorm(c, v);
    FiltArg filt_q = filt;
    if (filt_q.bits) filt_q.qf += q0;
#define LAUNCH_TC2(SC, I8, MODE, F)                                                                                  \
  SDB_CUDA(cudaLaunchKernelEx(&cfg, tc::screen_tc_kernel<SC, I8, MODE, F>, map_a, map_b, snorm_arg, k_blocks,        \
                              n_mblocks, nqc, p, tau, cand, ccnt, cap_arg, sub, scnt, k, hp, hist, probe_ptr,        \
                              probe_stride, sleep_min, sleep_max, pair, filt_q))
#define LAUNCH_TC1(SC, I8, MODE)                      \
  do {                                                \
    cfg.blockDim = dim3(tc::threads<I8, MODE>());     \
    if (filt_q.bits) LAUNCH_TC2(SC, I8, MODE, true);  \
    else LAUNCH_TC2(SC, I8, MODE, false);             \
  } while (0)
#define LAUNCH_TC(SC, I8)                   \
  do {                                      \
    if (mode == 0) LAUNCH_TC1(SC, I8, 0);   \
    else if (mode == 1) LAUNCH_TC1(SC, I8, 1); \
    else if (mode == 2) LAUNCH_TC1(SC, I8, 2); \
    else LAUNCH_TC1(SC, I8, 3);             \
  } while (0)
    if (int8) LAUNCH_TC(Score::Cosine, true);
    else if (sc == Score::Cosine) LAUNCH_TC(Score::Cosine, false);
    else if (sc == Score::Euclid) LAUNCH_TC(Score::Euclid, false);
    else if (sc == Score::EuclidFar) LAUNCH_TC(Score::EuclidFar, false);
    else LAUNCH_TC(Score::Dot, false);
#undef LAUNCH_TC
#undef LAUNCH_TC1
#undef LAUNCH_TC2
    count_launch(ctx);
  }
  if (mode == 0) {
    SDB_TRY(cand_set_count(c, s, nq, p.count * TILE_ROWS, st));    // pass 0 wrote fixed slots of the main lists
    s.last_slots = 0;                                              // ... and no private sub-lists
    if (filt.bits) SDB_TRY(cand_filter_list(c, s, filt, nq, st));  // ... of every row, the filtered-out ones included
  }
  SDB_CUDA(cudaGetLastError());
  return SDB_OK;
}

}  // namespace sdb
