// comm.cu -- multi-GPU brute force behind the ABI: row-sharded corpora, ONE NCCL all-gather of the per-shard top-k
// blocks per batch, merge kernel on every rank.  (SURVEY.md section 8e; no reference equivalent -- the reference is
// single-node CPU code.)
//
// NCCL is bound at run time (dlopen of libnccl.so.2) so that single-GPU users need no NCCL at all and a host process
// that already carries its own NCCL (PyTorch) shares that copy instead of loading a second one.
//
// Both deployment shapes are served by the same three phases (local search -> all-gather -> merge):
//   * one process per GPU  : sdb_comm_unique_id / sdb_comm_init_rank, then sdb_knn_sharded_submit* / _wait per rank
//   * one process, N GPUs  : sdb_ctx_create_multi (ncclCommInitAll), then sdb_knn_sharded_multi drives every shard
//                            from one thread inside ncclGroupStart/End
// The exchange itself does NOT go through an NCCL kernel by default.  The screen of the next batch is a persistent
// kernel that owns every SM (one 217 KB CTA per SM), so an NCCL all-gather kernel queued behind the tail of batch i
// cannot become resident until the screen of batch i+1 retires: measured on 8 GPUs, the step time doubled (2.06 ms
// instead of ~0.95 ms).  Instead every rank keeps an exchange ARENA (gather buffers + flag words) that its peers map
// (CUDA IPC between processes, peer access inside one process); after the local search a small kernel stores this
// rank's block straight into every peer's gather buffer over NVLink and publishes a sequence number (release, system
// scope); the merge is preceded by a one-warp kernel that waits for all ranks' sequence numbers, and followed by one
// that acknowledges the slot so a peer can overwrite it four batches later.  These kernels need no shared memory and a
// warp or two, so they run beside the resident screen.  NCCL remains the bootstrap (handle exchange), the fallback
// when peer mapping is unavailable (SDB_EXCHANGE=nccl forces it) and the graph path's all-reduce.
// Everything is enqueued on the batch's stream: no host synchronisation between the local search, the exchange
// and the merge.  Exactness across ranks: every block carries the number of queries its rank still has to repair on
// the host side (failed proof / special queries); since every rank sees every header after the all-gather, all ranks
// take the same decision to run a repair round (local repair, second all-gather + merge) -- no extra collective.
#include <dlfcn.h>
#include <nccl.h>

#include "internal.cuh"

namespace sdb {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;
static std::mutex g_nccl_mu;

static sdb_status nccl_load() {
  std::lock_guard<std::mutex> g(g_nccl_mu);
  if (g_nccl.lib) return SDB_OK;
  void* h = nullptr;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) {
    set_error("NCCL not available: %s", dlerror());
    return SDB_ENCCL;
  }
#define LOAD(field, sym)                                               \
  *(void**)(&g_nccl.field) = dlsym(h, sym);                            \
  if (!g_nccl.field) {                                                 \
    set_error("NCCL symbol %s missing", sym);                          \
    return SDB_ENCCL;                                                  \
  }
  LOAD(GetUniqueId, "ncclGetUniqueId");
  LOAD(CommInitRank, "ncclCommInitRank");
  LOAD(CommInitAll, "ncclCommInitAll");
  LOAD(CommDestroy, "ncclCommDestroy");
  LOAD(AllGather, "ncclAllGather");
  LOAD(AllReduce, "ncclAllReduce");
  LOAD(GroupStart, "ncclGroupStart");
  LOAD(GroupEnd, "ncclGroupEnd");
  LOAD(GetErrorString, "ncclGetErrorString");
#undef LOAD
  g_nccl.lib = h;
  return SDB_OK;
}

#define SDB_NCCL(call)                                                                             \
  do {                                                                                             \
    ncclResult_t r__ = (call);                                                                     \
    if (r__ != ncclSuccess) {                                                                      \
      ::sdb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, g_nccl.GetErrorString(r__));  \
      return SDB_ENCCL;                                                                            \
    }                                                                                              \
  } while (0)

struct Comm {
  ncclComm_t comm = nullptr;
  int nranks = 1, rank = 0;
  bool single_process = false;  // sdb_ctx_create_multi: every rank lives in this process (peer access, no IPC)
};

int comm_size(const Ctx* ctx) { return ctx && ctx->comm ? ctx->comm->nranks : 1; }
int comm_rank(const Ctx* ctx) { return ctx && ctx->comm ? ctx->comm->rank : 0; }

// in-place sum over the ranks of the context's communicator (no-op on a single rank); elem_bytes 4 (u32) or 8 (u64)
sdb_status comm_allreduce_sum(Ctx* ctx, void* d_buf, size_t count, int elem_bytes, cudaStream_t st) {
  if (!ctx->comm || ctx->comm->nranks <= 1 || count == 0) return SDB_OK;
  SDB_TRY(nccl_load());
  SDB_NCCL(g_nccl.AllReduce(d_buf, d_buf, count, elem_bytes == 8 ? ncclUint64 : ncclUint32, ncclSum, ctx->comm->comm, st));
  return SDB_OK;
}

void comm_destroy(Ctx* ctx) {
  if (ctx && ctx->comm) {
    if (ctx->comm->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->comm->comm);
    delete ctx->comm;
    ctx->comm = nullptr;
  }
}

// one rank's block inside the all-gather buffer: rows u64[nq*k] | dist f64[nq*k] | count u32[nq] | hdr u32[4]
struct BlockLayout {
  size_t off_rows, off_dist, off_cnt, off_hdr, bytes;
};
static BlockLayout block_layout(uint32_t nq, uint32_t k) {
  BlockLayout b;
  b.off_rows = 0;
  b.off_dist = (size_t)nq * k * 8;
  b.off_cnt = 2 * (size_t)nq * k * 8;
  b.off_hdr = (b.off_cnt + (size_t)nq * 4 + 15) / 16 * 16;
  b.bytes = b.off_hdr + 16;
  return b;
}

struct ShardSlot {  // per in-flight ticket: this rank's block, the gathered blocks, the headers on the host
  DevBuf<uint8_t> d_block;
  DevBuf<uint8_t> d_gather;      // NCCL path: own allocation
  uint8_t* gather = nullptr;     // where this batch's blocks are merged from (arena slot or d_gather)
  size_t stride = 0;             // distance between two ranks' blocks inside `gather`
  PinnedBuf<uint32_t> h_hdr;     // nranks x 4 + the exchange error word
  int hdr_cap = 0;
  cudaEvent_t ev_done = nullptr;
  uint64_t *d_out_rows = nullptr, *h_out_rows = nullptr;
  double *d_out_dist = nullptr, *h_out_dist = nullptr;
  uint32_t *d_out_count = nullptr, *h_out_count = nullptr;
  ResultBufs res;  // host-buffer entry points: merged result staging
};

}  // namespace sdb

using namespace sdb;

namespace {

struct Arena;
struct ShardState {  // hangs off the corpus through a side table (kept out of internal.cuh: only comm.cu needs it)
  ShardSlot slots[N_TICKETS];
  Arena* arena = nullptr;
};
std::mutex g_state_mu;
std::vector<std::pair<Corpus*, ShardState*>> g_states;

ShardState* state_of(Corpus* c) {
  std::lock_guard<std::mutex> g(g_state_mu);
  for (auto& p : g_states)
    if (p.first == c) return p.second;
  ShardState* s = new ShardState();
  g_states.emplace_back(c, s);
  return s;
}

sdb_status slot_reserve(Corpus* c, ShardSlot& s, uint32_t nq, uint32_t k, bool host_out) {
  const int nranks = c->ctx->comm ? c->ctx->comm->nranks : 1;
  const BlockLayout bl = block_layout(nq, k);
  if (!s.ev_done) SDB_CUDA(cudaEventCreateWithFlags(&s.ev_done, cudaEventDisableTiming));
  SDB_CUDA(s.d_block.reserve(bl.bytes));
  SDB_CUDA(s.d_gather.reserve(bl.bytes * nranks));
  if (s.hdr_cap < nranks) {
    s.hdr_cap = 0;
    SDB_CUDA(s.h_hdr.reserve(4 * nranks + 4));
    memset(s.h_hdr, 0, sizeof(uint32_t) * (4 * nranks + 4));  // [4 * nranks]: exchange error word (peer-to-peer path)
    s.hdr_cap = nranks;
  }
  if (host_out) SDB_CUDA(s.res.reserve((size_t)nq * (k ? k : 1), nq));
  return SDB_OK;
}


// ---- peer-to-peer exchange arena ------------------------------------------------------------------------------------
constexpr int MAX_P2P_RANKS = 16;
struct PeerTable {
  uint8_t* base[MAX_P2P_RANKS];
};
struct Arena {
  DevBuf<uint8_t> base;     // this rank's arena (plain device memory: IPC-exportable)
  size_t block_cap = 0;     // bytes reserved per (slot, rank) block
  size_t flags_off = 0, acks_off = 0, ctr_off = 0, err_off = 0, bytes = 0;
  int nranks = 0;
  PeerTable peers{};        // peers.base[r] = rank r's arena as mapped into this process (own base for r == rank)
  bool mapped[MAX_P2P_RANKS] = {};
  bool ok = false;          // peers mapped: the P2P path is in use
  size_t failed_need = 0;   // a collective attempt for this size failed: stay on NCCL until a larger request retries
  uint32_t seq = 0;                      // exchanges so far (identical on every rank)
  uint32_t slot_seq[N_TICKETS] = {};     // sequence number of the last exchange through each slot
};

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Every wait on a peer is bounded: a rank that never arrives (crashed process, mismatched call sequence) must surface
// as SDB_ENCCL on the host, not as a kernel that spins until the watchdog takes the GPU away.
constexpr uint64_t EXCH_TIMEOUT_NS = 30ull * 1000ull * 1000ull * 1000ull;
// spin until *p has reached `target` (sequence numbers, compared modulo 2^32); false = timed out
__device__ __forceinline__ bool spin_until_reached(const uint32_t* p, uint32_t target) {
  if ((int32_t)(ld_acquire_sys(p) - target) >= 0) return true;
  const uint64_t t0 = global_timer_ns();
  for (;;) {
    __nanosleep(64);
    if ((int32_t)(ld_acquire_sys(p) - target) >= 0) return true;
    if (global_timer_ns() - t0 > EXCH_TIMEOUT_NS) return false;
  }
}

// grid (nranks, S): CTA (p, s) stores its share of this rank's block into peer p's gather slot, the last of the S CTAs
// publishes `seq` in p's flag word.  Before the first store thread 0 makes sure p has consumed the previous content of
// the slot (p's acknowledgement lands in OUR arena).  ctr_off addresses the arrival counters of THIS SLOT (one per
// peer): pushes of different slots run concurrently on the two batch streams and must not share a counter -- with one
// counter per peer a push could publish its flag before its second CTA had copied, and the other push never published
// (a hang of the 50-step 8-GPU run, round 2); two pushes through the same slot are ordered by the ticket's life cycle.
__global__ void __launch_bounds__(256) exch_push_kernel(PeerTable pt, uint8_t* my_base, const uint4* __restrict__ src,
                                                        size_t n16, size_t gather_off, size_t flag_off, size_t ack_off,
                                                        size_t ctr_off, size_t err_off, uint32_t need_ack, uint32_t seq) {
  const uint32_t p = blockIdx.x, S = gridDim.y, sidx = blockIdx.y;
  if (threadIdx.x == 0) {
    const uint32_t* a = reinterpret_cast<const uint32_t*>(my_base + ack_off) + p;
    if (!spin_until_reached(a, need_ack)) atomicMax(reinterpret_cast<uint32_t*>(my_base + err_off), 1u);
  }
  __syncthreads();
  uint4* dst = reinterpret_cast<uint4*>(pt.base[p] + gather_off);
  const size_t per = (n16 + S - 1) / S;
  const size_t lo = per * sidx, hi = lo + per < n16 ? lo + per : n16;
  for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) dst[i] = src[i];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t* ctr = reinterpret_cast<uint32_t*>(my_base + ctr_off) + p;
    const uint32_t old = S > 1 ? atomicAdd(ctr, 1u) : 0u;
    if (old == S - 1) {
      if (S > 1) {
        *ctr = 0;
        __threadfence_system();
      }
      st_release_sys(reinterpret_cast<uint32_t*>(pt.base[p] + flag_off), seq);
    }
  }
}
// one warp: wait until every rank's block of exchange `seq` has landed in this rank's slot
__global__ void exch_wait_kernel(uint8_t* my_base, size_t flags_off, size_t err_off, int nranks, uint32_t seq) {
  if ((int)threadIdx.x < nranks) {
    const uint32_t* f = reinterpret_cast<const uint32_t*>(my_base + flags_off) + threadIdx.x;
    if (!spin_until_reached(f, seq)) atomicMax(reinterpret_cast<uint32_t*>(my_base + err_off), 2u);
  }
}
// one warp: tell every rank that this rank is done with the slot's content of exchange `seq`
__global__ void exch_ack_kernel(PeerTable pt, size_t ack_off, int nranks, uint32_t seq) {
  if ((int)threadIdx.x < nranks) st_release_sys(reinterpret_cast<uint32_t*>(pt.base[threadIdx.x] + ack_off), seq);
}

struct Pending {  // one shard's in-flight sharded batch
  Corpus* c = nullptr;
  ShardSlot* s = nullptr;
  uint32_t ticket = 0, nq = 0, k = 0;
  int slot = -1;
  Ranking rank;  // what the batch ranks: the merges (first and repair round) order the blocks in its direction
};


static bool exchange_forced_nccl() {
  static const bool v = [] {
    const char* e = getenv("SDB_EXCHANGE");
    return e && (e[0] == 'n' || e[0] == 'N');
  }();
  return v;
}

static void arena_unmap(Arena* a, int self) {
  for (int r = 0; r < MAX_P2P_RANKS; r++) {
    if (a->mapped[r] && r != self && a->peers.base[r]) cudaIpcCloseMemHandle(a->peers.base[r]);
    a->mapped[r] = false;
    a->peers.base[r] = nullptr;
  }
  a->ok = false;
}

// (re)allocate this rank's arena for blocks of `need` bytes; the peers are mapped by the callers below
static sdb_status arena_alloc_local(Corpus* c, Arena* a, size_t need) {
  const int R = c->ctx->comm->nranks;
  a->base.reset();
  a->block_cap = (need + 65535) / 65536 * 65536;
  a->nranks = R;
  const size_t gather_bytes = (size_t)N_TICKETS * R * a->block_cap;
  a->flags_off = gather_bytes;
  a->acks_off = a->flags_off + 256 * ((sizeof(uint32_t) * N_TICKETS * R + 255) / 256);
  a->ctr_off = a->acks_off + 256 * ((sizeof(uint32_t) * N_TICKETS * R + 255) / 256);
  a->err_off = a->ctr_off + 256 * ((sizeof(uint32_t) * N_TICKETS * R + 255) / 256);
  a->bytes = a->err_off + 256;
  SDB_CUDA(a->base.reserve(a->bytes));
  SDB_CUDA(cudaMemset(a->base, 0, a->bytes));
  SDB_CUDA(cudaDeviceSynchronize());
  a->seq = 0;
  for (int i = 0; i < N_TICKETS; i++) a->slot_seq[i] = 0;
  return SDB_OK;
}

// one process per GPU: collective (every rank reaches this with the same `need`, because every rank submits the same
// batches in the same order).  IPC handles travel through one NCCL all-gather; a second tiny all-reduce makes the
// outcome unanimous, so either every rank uses the P2P path or every rank stays on NCCL.
static sdb_status arena_ensure_ipc(Corpus* c, ShardState* ss, size_t need) {
  Ctx* ctx = c->ctx;
  Comm* cm = ctx->comm;
  if (!ss->arena) ss->arena = new Arena();
  Arena* a = ss->arena;
  if (a->ok && a->block_cap >= need) return SDB_OK;
  if (!a->ok && a->failed_need && need <= a->failed_need) return SDB_OK;  // stays on NCCL
  const int R = cm->nranks;
  // quiesce: batches in flight still exchange through the old arena
  SDB_CUDA(cudaStreamSynchronize(ctx->stream));
  SDB_CUDA(cudaStreamSynchronize(ctx->stream2));
  arena_unmap(a, cm->rank);
  uint32_t good = 1;
  if (arena_alloc_local(c, a, need) != SDB_OK) good = 0;
  cudaIpcMemHandle_t mine{};
  if (good && cudaIpcGetMemHandle(&mine, a->base) != cudaSuccess) {
    cudaGetLastError();
    good = 0;
  }
  DevBuf<uint8_t> d_h;
  SDB_CUDA(d_h.reserve(sizeof(cudaIpcMemHandle_t) * (R + 1) + 16));
  std::vector<cudaIpcMemHandle_t> all((size_t)R);
  cudaStream_t st = ctx->stream;
  if (cudaMemcpyAsync(d_h + sizeof(mine) * R, &mine, sizeof(mine), cudaMemcpyHostToDevice, st) != cudaSuccess) return SDB_ECUDA;
  if (g_nccl.AllGather(d_h + sizeof(mine) * R, d_h, sizeof(mine), ncclChar, cm->comm, st) != ncclSuccess) {
    set_error("exchange arena: ncclAllGather of the IPC handles failed");
    return SDB_ENCCL;
  }
  if (cudaMemcpyAsync(all.data(), d_h, sizeof(mine) * R, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return SDB_ECUDA;
  if (good) {
    for (int r = 0; r < R && good; r++) {
      if (r == cm->rank) {
        a->peers.base[r] = a->base;
        continue;
      }
      void* ptr = nullptr;
      if (cudaIpcOpenMemHandle(&ptr, all[(size_t)r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        good = 0;
        break;
      }
      a->peers.base[r] = (uint8_t*)ptr;
      a->mapped[r] = true;
    }
  }
  // unanimous?
  uint32_t* d_flag = reinterpret_cast<uint32_t*>(d_h + sizeof(mine) * (R + 1));
  if (cudaMemcpyAsync(d_flag, &good, 4, cudaMemcpyHostToDevice, st) != cudaSuccess) return SDB_ECUDA;
  if (g_nccl.AllReduce(d_flag, d_flag, 1, ncclUint32, ncclMin, cm->comm, st) != ncclSuccess) {
    set_error("exchange arena: ncclAllReduce failed");
    return SDB_ENCCL;
  }
  uint32_t all_good = 0;
  if (cudaMemcpyAsync(&all_good, d_flag, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
    return SDB_ECUDA;
  d_h.reset();
  if (all_good) {
    a->ok = true;
    a->failed_need = 0;
  } else {
    arena_unmap(a, cm->rank);
    a->failed_need = need;
  }
  return SDB_OK;
}

// one process, N GPUs: the arenas of all shards are (re)built together and mapped through peer access
static sdb_status arena_ensure_multi(sdb_corpus* const* shards, int n, size_t need) {
  bool all_ok = true;
  for (int i = 0; i < n; i++) {
    ShardState* ss = state_of(shards[i]);
    if (!ss->arena) ss->arena = new Arena();
    all_ok = all_ok && ss->arena->ok && ss->arena->block_cap >= need;
  }
  if (all_ok) return SDB_OK;
  Arena* a0 = state_of(shards[0])->arena;
  if (!a0->ok && a0->failed_need && need <= a0->failed_need) return SDB_OK;
  bool good = n <= MAX_P2P_RANKS;
  for (int i = 0; i < n; i++) {
    Ctx* ctx = shards[i]->ctx;
    SDB_CUDA(cudaSetDevice(ctx->device));
    SDB_CUDA(cudaStreamSynchronize(ctx->stream));
    SDB_CUDA(cudaStreamSynchronize(ctx->stream2));
  }
  for (int i = 0; i < n && good; i++) {
    Ctx* ctx = shards[i]->ctx;
    SDB_CUDA(cudaSetDevice(ctx->device));
    for (int j = 0; j < n && good; j++) {
      if (j == i || shards[j]->ctx->device == ctx->device) continue;
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, ctx->device, shards[j]->ctx->device) != cudaSuccess || !can) good = false;
      else {
        const cudaError_t e = cudaDeviceEnablePeerAccess(shards[j]->ctx->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) good = false;
        cudaGetLastError();
      }
    }
    Arena* a = state_of(shards[i])->arena;
    for (int r = 0; r < MAX_P2P_RANKS; r++) {
      a->mapped[r] = false;
      a->peers.base[r] = nullptr;
    }
    a->ok = false;
    if (good && arena_alloc_local(shards[i], a, need) != SDB_OK) good = false;
  }
  for (int i = 0; i < n; i++) {
    Arena* a = state_of(shards[i])->arena;
    if (good) {
      for (int j = 0; j < n; j++) a->peers.base[shards[j]->ctx->comm->rank] = state_of(shards[j])->arena->base;
      a->ok = true;
      a->failed_need = 0;
    } else {
      a->failed_need = need;
    }
  }
  return SDB_OK;
}

}  // namespace
namespace sdb {
void comm_corpus_released(Corpus* c) {
  ShardState* ss = nullptr;
  {
    std::lock_guard<std::mutex> g(g_state_mu);
    for (size_t i = 0; i < g_states.size(); i++)
      if (g_states[i].first == c) {
        ss = g_states[i].second;
        g_states.erase(g_states.begin() + (long)i);
        break;
      }
  }
  if (!ss) return;
  for (ShardSlot& s : ss->slots)
    if (s.ev_done) cudaEventDestroy(s.ev_done);
  if (ss->arena) {
    arena_unmap(ss->arena, c->ctx->comm ? c->ctx->comm->rank : 0);
    delete ss->arena;
  }
  delete ss;
}
}  // namespace sdb
namespace {

static bool use_p2p(Corpus* c, ShardState* ss) {
  return c->ctx->comm && c->ctx->comm->nranks > 1 && ss->arena && ss->arena->ok && !exchange_forced_nccl();
}

// phase A: the local search into this rank's block, header = number of queries this rank must repair on the host.
// rf: the call's global row filters (rf.bits == nullptr: unfiltered); the driver slices this shard's rows out of them.
// rank: what the batch ranks (KNN: the default Ranking); the shard's list is its top-k by (order key, global row).
// host_in: queries and bitmaps are host memory (queries may be NULL for SDB_FN_MAGNITUDE, so their pointer cannot tell).
// The slot's buffers belong to the batch's ticket slot, so they are free exactly when the ticket is.
sdb_status phase_local(Corpus* c, const double* queries, bool host_in, uint32_t nq, uint32_t k, const RowFilters& rf,
                       const Ranking& rank, uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                       uint64_t* h_out_rows, double* h_out_dist, uint32_t* h_out_count, Pending* p) {
  if (rf.bits) {  // refused before anything is enqueued
    SDB_TRY(check_filters(nq, rf.bits, rf.n_filters, rf.query_filter));
    if (c->row_base + c->n > rf.n_rows_total) {
      set_error("sharded filtered search: shard rows %llu..%llu outside the bitmaps' %llu rows",
                (unsigned long long)c->row_base, (unsigned long long)(c->row_base + c->n),
                (unsigned long long)rf.n_rows_total);
      return SDB_EINVAL;
    }
  }
  Ticket* t = claim_ticket(c);
  if (!t) return SDB_EOVERFLOW;
  const int slot = (int)(t - c->tickets);
  ShardSlot& s = state_of(c)->slots[slot];
  const BlockLayout bl = block_layout(nq, k);
  const bool host_out = h_out_count != nullptr;
  SDB_TRY(slot_reserve(c, s, nq, k, host_out));
  const KnnCall call{queries, host_in, rf, c->row_base,
                     (uint64_t*)(s.d_block + bl.off_rows), (double*)(s.d_block + bl.off_dist),
                     (uint32_t*)(s.d_block + bl.off_cnt), false, nullptr, rank};
  SDB_TRY(submit_call(c, t, nq, k, call));
  SDB_TRY(knn_shard_header(c, t->id, s.d_block + bl.off_hdr));
  s.d_out_rows = host_out ? s.res.rows : d_out_rows;
  s.d_out_dist = host_out ? s.res.dist : d_out_dist;
  s.d_out_count = host_out ? s.res.count : d_out_count;
  s.h_out_rows = h_out_rows;
  s.h_out_dist = h_out_dist;
  s.h_out_count = h_out_count;
  p->c = c;
  p->s = &s;
  p->ticket = t->id;
  p->nq = nq;
  p->k = k;
  p->slot = slot;
  p->rank = rank;
  return SDB_OK;
}

// phase B: the exchange of the per-shard blocks.  P2P: this rank's block is stored into every peer's arena slot and a
// one-warp kernel waits for everybody else's; NCCL: ONE all-gather (inside the caller's group when one thread drives
// several GPUs).
sdb_status phase_gather(const Pending& p) {
  Corpus* c = p.c;
  ShardSlot& s = *p.s;
  ShardState* ss = state_of(c);
  const BlockLayout bl = block_layout(p.nq, p.k);
  cudaStream_t st = knn_ticket_stream(c, p.ticket);
  if (use_p2p(c, ss)) {
    Arena* a = ss->arena;
    const int R = a->nranks, me = c->ctx->comm->rank;
    const uint32_t seq = ++a->seq;
    const uint32_t need_ack = a->slot_seq[p.slot];
    a->slot_seq[p.slot] = seq;
    const size_t gather_off = ((size_t)p.slot * R + me) * a->block_cap;
    const size_t flag_off = a->flags_off + sizeof(uint32_t) * ((size_t)p.slot * R + me);
    const size_t ack_off = a->acks_off + sizeof(uint32_t) * ((size_t)p.slot * R);
    const size_t n16 = bl.bytes / 16;
    unsigned S = (unsigned)((bl.bytes + (128u << 10) - 1) / (128u << 10));  // 256-thread CTAs: they fit beside a screen CTA
    if (S > 16) S = 16;
    if (S < 1) S = 1;
    const size_t ctr_off = a->ctr_off + sizeof(uint32_t) * ((size_t)p.slot * R);
    exch_push_kernel<<<dim3((unsigned)R, S), 256, 0, st>>>(a->peers, a->base, reinterpret_cast<const uint4*>(s.d_block.get()), n16,
                                                            gather_off, flag_off, ack_off, ctr_off, a->err_off, need_ack, seq);
    exch_wait_kernel<<<1, 32, 0, st>>>(a->base, a->flags_off + sizeof(uint32_t) * ((size_t)p.slot * R), a->err_off, R, seq);
    SDB_CUDA(cudaGetLastError());
    knn_trace_mark(c, p.ticket, "exchanged");
    s.gather = a->base + (size_t)p.slot * R * a->block_cap;
    s.stride = a->block_cap;
    return SDB_OK;
  }
  s.gather = s.d_gather;
  s.stride = bl.bytes;
  if (c->ctx->comm && c->ctx->comm->nranks > 1) {
    SDB_NCCL(g_nccl.AllGather(s.d_block, s.d_gather, bl.bytes, ncclChar, c->ctx->comm->comm, st));
  } else {
    SDB_CUDA(cudaMemcpyAsync(s.d_gather, s.d_block, bl.bytes, cudaMemcpyDeviceToDevice, st));
  }
  return SDB_OK;
}

// phase C: merge on this rank, headers to the host, optional copy of the merged result to host buffers
sdb_status phase_merge(const Pending& p) {
  Corpus* c = p.c;
  ShardSlot& s = *p.s;
  ShardState* ss = state_of(c);
  const int nranks = c->ctx->comm ? c->ctx->comm->nranks : 1;
  const BlockLayout bl = block_layout(p.nq, p.k);
  cudaStream_t st = knn_ticket_stream(c, p.ticket);
  if (p.k)
    SDB_TRY(topk_merge_launch(c->ctx, (uint32_t)nranks, p.nq, p.k, (const uint64_t*)(s.gather + bl.off_rows),
                              (const double*)(s.gather + bl.off_dist), (const uint32_t*)(s.gather + bl.off_cnt),
                              s.stride / 8, s.stride / 8, s.stride / 4, s.d_out_rows, s.d_out_dist, s.d_out_count,
                              p.rank.desc, st));
  else SDB_CUDA(cudaMemsetAsync(s.d_out_count, 0, sizeof(uint32_t) * p.nq, st));
  SDB_CUDA(cudaMemcpy2DAsync(s.h_hdr, 16, s.gather + bl.off_hdr, s.stride, 16, (size_t)nranks, cudaMemcpyDeviceToHost, st));
  if (use_p2p(c, ss)) {  // the slot's blocks have been consumed: peers may overwrite them (four batches from now)
    Arena* a = ss->arena;
    const int R = a->nranks, me = c->ctx->comm->rank;
    exch_ack_kernel<<<1, 32, 0, st>>>(a->peers, a->acks_off + sizeof(uint32_t) * ((size_t)p.slot * R + me), R, a->slot_seq[p.slot]);
    SDB_CUDA(cudaGetLastError());
    SDB_CUDA(cudaMemcpyAsync(s.h_hdr + 4 * nranks, a->base + a->err_off, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  }
  if (s.h_out_count) {
    if (p.k) {
      SDB_CUDA(cudaMemcpyAsync(s.h_out_rows, s.d_out_rows, sizeof(uint64_t) * (size_t)p.nq * p.k, cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaMemcpyAsync(s.h_out_dist, s.d_out_dist, sizeof(double) * (size_t)p.nq * p.k, cudaMemcpyDeviceToHost, st));
    }
    SDB_CUDA(cudaMemcpyAsync(s.h_out_count, s.d_out_count, sizeof(uint32_t) * p.nq, cudaMemcpyDeviceToHost, st));
  }
  SDB_CUDA(cudaEventRecord(s.ev_done, st));
  knn_trace_mark(c, p.ticket, "merged");
  return SDB_OK;
}

// completion of a set of shards driven by this thread (1 in the process-per-GPU shape).  Every rank sees every header,
// so the decision to run the repair round is the same everywhere.
sdb_status finish_all(Pending* ps, int n) {
  bool any = false;
  for (int i = 0; i < n; i++) {
    SDB_CUDA(cudaSetDevice(ps[i].c->ctx->device));
    SDB_CUDA(cudaEventSynchronize(ps[i].s->ev_done));
    const int nranks = ps[i].c->ctx->comm ? ps[i].c->ctx->comm->nranks : 1;
    if (use_p2p(ps[i].c, state_of(ps[i].c)) && ps[i].s->h_hdr[4 * nranks] != 0) {
      set_error("sharded search: a peer did not %s within 30 s (rank %d of %d) -- every rank must submit the same batches in "
                "the same order", ps[i].s->h_hdr[4 * nranks] == 1 ? "acknowledge a slot" : "deliver its block",
                ps[i].c->ctx->comm->rank, nranks);
      for (int j = 0; j < n; j++) knn_release_ticket(ps[j].c, ps[j].ticket);
      return SDB_ENCCL;
    }
    for (int r = 0; r < nranks; r++) any = any || ps[i].s->h_hdr[4 * r] != 0;
  }
  sdb_status rc = SDB_OK;
  if (any) {
    for (int i = 0; i < n && rc == SDB_OK; i++) {
      cudaSetDevice(ps[i].c->ctx->device);
      bool repaired = false;
      rc = knn_finish_for_shard(ps[i].c, ps[i].ticket, &repaired);  // local ladder re-runs / exact fallbacks
    }
    if (rc == SDB_OK) {
      const bool group = n > 1;
      if (group) g_nccl.GroupStart();
      for (int i = 0; i < n && rc == SDB_OK; i++) {
        cudaSetDevice(ps[i].c->ctx->device);
        rc = phase_gather(ps[i]);
      }
      if (group) g_nccl.GroupEnd();
      for (int i = 0; i < n && rc == SDB_OK; i++) {
        cudaSetDevice(ps[i].c->ctx->device);
        rc = phase_merge(ps[i]);
      }
      for (int i = 0; i < n && rc == SDB_OK; i++) {
        cudaSetDevice(ps[i].c->ctx->device);
        if (cudaEventSynchronize(ps[i].s->ev_done) != cudaSuccess) {
          set_error("sharded repair round: %s", cudaGetErrorString(cudaGetLastError()));
          rc = SDB_ECUDA;
        }
      }
    }
  } else {
    for (int i = 0; i < n && rc == SDB_OK; i++) {
      cudaSetDevice(ps[i].c->ctx->device);
      bool repaired = false;
      rc = knn_finish_for_shard(ps[i].c, ps[i].ticket, &repaired);  // nothing flagged: records the statistics
    }
  }
  for (int i = 0; i < n; i++) knn_release_ticket(ps[i].c, ps[i].ticket);
  return rc;
}

// pending sharded tickets of the process-per-GPU shape, keyed by (corpus, ticket)
std::mutex g_pending_mu;
std::vector<Pending> g_pending;

}  // namespace

extern "C" {

sdb_status sdb_comm_unique_id(uint8_t* id128) {
  if (!id128) return SDB_EINVAL;
  SDB_TRY(nccl_load());
  static_assert(sizeof(ncclUniqueId) == SDB_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  SDB_NCCL(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return SDB_OK;
}

sdb_status sdb_comm_init_rank(sdb_ctx* ctx, int nranks, int rank, const uint8_t* id128) {
  if (!ctx || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return SDB_EINVAL;
  SDB_TRY(nccl_load());
  std::lock_guard<std::mutex> g(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  comm_destroy(ctx);
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  Comm* cm = new Comm();
  cm->nranks = nranks;
  cm->rank = rank;
  const ncclResult_t r = g_nccl.CommInitRank(&cm->comm, nranks, id, rank);
  if (r != ncclSuccess) {
    set_error("ncclCommInitRank(%d of %d) failed: %s", rank, nranks, g_nccl.GetErrorString(r));
    delete cm;
    return SDB_ENCCL;
  }
  ctx->comm = cm;
  return SDB_OK;
}

int sdb_comm_size(const sdb_ctx* ctx) { return ctx && ctx->comm ? ctx->comm->nranks : 1; }
int sdb_comm_rank(const sdb_ctx* ctx) { return ctx && ctx->comm ? ctx->comm->rank : 0; }

sdb_status sdb_ctx_create_multi(const int* devices, int ndev, sdb_ctx** out) {
  if (!devices || !out || ndev < 1 || ndev > 64) return SDB_EINVAL;
  for (int i = 0; i < ndev; i++) out[i] = nullptr;
  if (ndev > 1) SDB_TRY(nccl_load());
  for (int i = 0; i < ndev; i++) {
    const sdb_status rc = sdb_ctx_create(devices[i], &out[i]);
    if (rc != SDB_OK) {
      for (int j = 0; j < i; j++) sdb_ctx_destroy(out[j]);
      for (int j = 0; j < ndev; j++) out[j] = nullptr;
      return rc;
    }
  }
  if (ndev > 1) {
    std::vector<ncclComm_t> comms(ndev);
    const ncclResult_t r = g_nccl.CommInitAll(comms.data(), ndev, devices);
    if (r != ncclSuccess) {
      set_error("ncclCommInitAll(%d devices) failed: %s", ndev, g_nccl.GetErrorString(r));
      for (int j = 0; j < ndev; j++) {
        sdb_ctx_destroy(out[j]);
        out[j] = nullptr;
      }
      return SDB_ENCCL;
    }
    for (int i = 0; i < ndev; i++) {
      Comm* cm = new Comm();
      cm->comm = comms[i];
      cm->nranks = ndev;
      cm->rank = i;
      cm->single_process = true;
      out[i]->comm = cm;
    }
  }
  return SDB_OK;
}

sdb_status sdb_corpus_set_row_base(sdb_corpus* c, uint64_t row_base) {
  if (!c) return SDB_EINVAL;
  c->row_base = row_base;
  return SDB_OK;
}

static sdb_status sharded_submit(sdb_corpus* c, const double* d_queries, const double* h_queries, uint32_t nq, uint32_t k,
                                 const RowFilters& rf, const Ranking& rank, uint64_t* d_out_rows, double* d_out_dist,
                                 uint32_t* d_out_count, uint64_t* h_out_rows, double* h_out_dist,
                                 uint32_t* h_out_count, uint32_t* ticket) {
  if (!c || !ticket || !nq) return SDB_EINVAL;
  if (c->ctx->comm && c->ctx->comm->nranks > 1) SDB_TRY(nccl_load());
  Pending p;
  {
    std::lock_guard<std::mutex> g(c->mu);
    SDB_CUDA(cudaSetDevice(c->ctx->device));
    if (c->ctx->comm && c->ctx->comm->nranks > 1 && c->ctx->comm->nranks <= MAX_P2P_RANKS && !exchange_forced_nccl()) {
      if (c->ctx->comm->single_process) {
        set_error("contexts of sdb_ctx_create_multi are driven through sdb_knn_sharded_multi");
        return SDB_EINVAL;
      }
      SDB_TRY(arena_ensure_ipc(c, state_of(c), block_layout(nq, k).bytes));
    }
    // the host entry points hand over host outputs, the device ones device outputs
    SDB_TRY(phase_local(c, h_queries ? h_queries : d_queries, h_out_count != nullptr, nq, k, rf, rank, d_out_rows,
                        d_out_dist, d_out_count, h_out_rows, h_out_dist, h_out_count, &p));
    sdb_status rc = phase_gather(p);
    if (rc == SDB_OK) rc = phase_merge(p);
    if (rc != SDB_OK) {
      cudaStreamSynchronize(c->ctx->stream);
      cudaStreamSynchronize(c->ctx->stream2);
      knn_release_ticket(c, p.ticket);
      return rc;
    }
  }
  {
    std::lock_guard<std::mutex> g(g_pending_mu);
    g_pending.push_back(p);
  }
  *ticket = p.ticket;
  return SDB_OK;
}

sdb_status sdb_knn_sharded_submit_device(sdb_corpus* c, const double* d_queries, uint32_t nq, uint32_t k,
                                         uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                                         uint32_t* ticket) {
  if (!d_queries || !d_out_count || (k && (!d_out_rows || !d_out_dist))) return SDB_EINVAL;
  return sharded_submit(c, d_queries, nullptr, nq, k, RowFilters(), Ranking(), d_out_rows, d_out_dist, d_out_count, nullptr, nullptr,
                        nullptr, ticket);
}

sdb_status sdb_knn_sharded_submit(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k, uint64_t* out_rows,
                                  double* out_dist, uint32_t* out_count, uint32_t* ticket) {
  if (!queries || !out_count || (k && (!out_rows || !out_dist))) return SDB_EINVAL;
  return sharded_submit(c, nullptr, queries, nq, k, RowFilters(), Ranking(), nullptr, nullptr, nullptr, out_rows, out_dist, out_count,
                        ticket);
}

sdb_status sdb_knn_sharded_submit_filtered(sdb_corpus* c, const double* queries, uint32_t nq, uint32_t k,
                                           const uint32_t* filters, uint32_t n_filters, const uint32_t* query_filter,
                                           uint64_t n_rows_total, uint64_t* out_rows, double* out_dist,
                                           uint32_t* out_count, uint32_t* ticket) {
  if (!filters || !queries || !out_count || (k && (!out_rows || !out_dist))) return SDB_EINVAL;
  return sharded_submit(c, nullptr, queries, nq, k, RowFilters{filters, n_filters, query_filter, n_rows_total}, Ranking(),
                        nullptr, nullptr, nullptr, out_rows, out_dist, out_count, ticket);
}

sdb_status sdb_knn_sharded_submit_filtered_device(sdb_corpus* c, const double* d_queries, uint32_t nq, uint32_t k,
                                                  const uint32_t* d_filters, uint32_t n_filters,
                                                  const uint32_t* query_filter, uint64_t n_rows_total,
                                                  uint64_t* d_out_rows, double* d_out_dist, uint32_t* d_out_count,
                                                  uint32_t* ticket) {
  if (!d_filters || !d_queries || !d_out_count || (k && (!d_out_rows || !d_out_dist))) return SDB_EINVAL;
  return sharded_submit(c, d_queries, nullptr, nq, k, RowFilters{d_filters, n_filters, query_filter, n_rows_total},
                        Ranking(), d_out_rows, d_out_dist, d_out_count, nullptr, nullptr, nullptr, ticket);
}

sdb_status sdb_knn_sharded_wait(sdb_corpus* c, uint32_t ticket) {
  if (!c) return SDB_EINVAL;
  Pending p;
  {
    std::lock_guard<std::mutex> g(g_pending_mu);
    size_t i = 0;
    for (; i < g_pending.size(); i++)
      if (g_pending[i].c == c && g_pending[i].ticket == ticket) break;
    if (i == g_pending.size()) {
      set_error("sdb_knn_sharded_wait: unknown or already completed ticket %u", ticket);
      return SDB_EINVAL;
    }
    p = g_pending[i];
    g_pending.erase(g_pending.begin() + (long)i);
  }
  std::lock_guard<std::mutex> g(c->mu);
  return finish_all(&p, 1);
}

// rank: what the batch ranks; queries may be NULL only for SDB_FN_MAGNITUDE, which takes none
static sdb_status sharded_multi(sdb_corpus* const* shards, int n, const double* queries, uint32_t nq, uint32_t k,
                                const RowFilters& rf, const Ranking& rank, uint64_t* out_rows, double* out_dist,
                                uint32_t* out_count) {
  if (!shards || n < 1 || n > 64 || (!queries && rank.fn != SDB_FN_MAGNITUDE) || !nq || !out_count ||
      (k && (!out_rows || !out_dist)))
    return SDB_EINVAL;
  if (n > 1) SDB_TRY(nccl_load());
  std::vector<Pending> ps((size_t)n);
  std::vector<std::unique_lock<std::mutex>> locks;
  for (int i = 0; i < n; i++) {
    if (!shards[i]) return SDB_EINVAL;
    locks.emplace_back(shards[i]->mu);
  }
  sdb_status rc = SDB_OK;
  int started = 0;
  if (n > 1 && shards[0]->ctx->comm && shards[0]->ctx->comm->single_process && !exchange_forced_nccl())
    SDB_TRY(arena_ensure_multi(shards, n, block_layout(nq, k).bytes));
  for (int i = 0; i < n && rc == SDB_OK; i++) {  // every shard searches; shard 0's merged copy goes to the caller
    cudaSetDevice(shards[i]->ctx->device);
    ShardState* ss = state_of(shards[i]);
    (void)ss;
    if (i == 0)
      rc = phase_local(shards[i], queries, true, nq, k, rf, rank, nullptr, nullptr, nullptr, out_rows, out_dist,
                       out_count, &ps[i]);
    else {
      // the other shards keep their merged copy on the device (slot staging buffers)
      rc = phase_local(shards[i], queries, true, nq, k, rf, rank, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                       &ps[i]);
      if (rc == SDB_OK) {
        ShardSlot& s = *ps[i].s;
        rc = slot_reserve(shards[i], s, nq, k, true);
        s.d_out_rows = s.res.rows;
        s.d_out_dist = s.res.dist;
        s.d_out_count = s.res.count;
      }
    }
    if (rc == SDB_OK) started++;
  }
  if (rc == SDB_OK) {
    if (n > 1) g_nccl.GroupStart();
    for (int i = 0; i < n && rc == SDB_OK; i++) {
      cudaSetDevice(shards[i]->ctx->device);
      rc = phase_gather(ps[i]);
    }
    if (n > 1) g_nccl.GroupEnd();
    for (int i = 0; i < n && rc == SDB_OK; i++) {
      cudaSetDevice(shards[i]->ctx->device);
      rc = phase_merge(ps[i]);
    }
  }
  if (rc == SDB_OK) return finish_all(ps.data(), n);
  for (int i = 0; i < started; i++) {
    cudaSetDevice(shards[i]->ctx->device);
    cudaStreamSynchronize(shards[i]->ctx->stream);
    cudaStreamSynchronize(shards[i]->ctx->stream2);
    knn_release_ticket(shards[i], ps[i].ticket);
  }
  return rc;
}

sdb_status sdb_knn_sharded_multi(sdb_corpus* const* shards, int n, const double* queries, uint32_t nq, uint32_t k,
                                 uint64_t* out_rows, double* out_dist, uint32_t* out_count) {
  return sharded_multi(shards, n, queries, nq, k, RowFilters(), Ranking(), out_rows, out_dist, out_count);
}

sdb_status sdb_knn_sharded_multi_filtered(sdb_corpus* const* shards, int n, const double* queries, uint32_t nq,
                                          uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                          const uint32_t* query_filter, uint64_t n_rows_total, uint64_t* out_rows,
                                          double* out_dist, uint32_t* out_count) {
  if (!filters) return SDB_EINVAL;
  return sharded_multi(shards, n, queries, nq, k, RowFilters{filters, n_filters, query_filter, n_rows_total}, Ranking(),
                       out_rows, out_dist, out_count);
}

// ---- ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k on a row-sharded column: the sharded driver with the ranking
// (fn, order).  Every shard returns its top-k by (order key, global row) -- its own order, since a shard's global rows
// are row_base + its scan positions -- so the union of the blocks holds the global top-k, and the merge in the
// ranking's direction returns what sdb_corpus_order_topk returns on the unsharded column.
sdb_status sdb_corpus_order_sharded_submit(sdb_corpus* c, const double* queries, uint32_t nq, int fn, int order,
                                           uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                           const uint32_t* query_filter, uint64_t n_rows_total, uint64_t* out_rows,
                                           double* out_value, uint32_t* out_count, uint32_t* ticket) {
  Ranking rank;
  if (!ticket) return SDB_EINVAL;
  SDB_TRY(order_args(c, queries, nq, fn, order, k, filters, n_filters, query_filter, out_rows, out_value, out_count,
                     &rank));
  return sharded_submit(c, nullptr, queries, nq, k, RowFilters{filters, n_filters, query_filter, n_rows_total}, rank,
                        nullptr, nullptr, nullptr, out_rows, out_value, out_count, ticket);
}

sdb_status sdb_corpus_order_sharded_submit_device(sdb_corpus* c, const double* d_queries, uint32_t nq, int fn,
                                                  int order, uint32_t k, const uint32_t* d_filters,
                                                  uint32_t n_filters, const uint32_t* query_filter,
                                                  uint64_t n_rows_total, uint64_t* d_out_rows, double* d_out_value,
                                                  uint32_t* d_out_count, uint32_t* ticket) {
  Ranking rank;
  if (!ticket) return SDB_EINVAL;
  SDB_TRY(order_args(c, d_queries, nq, fn, order, k, d_filters, n_filters, query_filter, d_out_rows, d_out_value,
                     d_out_count, &rank));
  return sharded_submit(c, d_queries, nullptr, nq, k, RowFilters{d_filters, n_filters, query_filter, n_rows_total},
                        rank, d_out_rows, d_out_value, d_out_count, nullptr, nullptr, nullptr, ticket);
}

sdb_status sdb_corpus_order_sharded_multi(sdb_corpus* const* shards, int n_shards, const double* queries, uint32_t nq,
                                          int fn, int order, uint32_t k, const uint32_t* filters, uint32_t n_filters,
                                          const uint32_t* query_filter, uint64_t n_rows_total, uint64_t* out_rows,
                                          double* out_value, uint32_t* out_count) {
  Ranking rank;
  if (!shards || n_shards < 1) return SDB_EINVAL;
  SDB_TRY(order_args(shards[0], queries, nq, fn, order, k, filters, n_filters, query_filter, out_rows, out_value,
                     out_count, &rank));
  return sharded_multi(shards, n_shards, queries, nq, k, RowFilters{filters, n_filters, query_filter, n_rows_total},
                       rank, out_rows, out_value, out_count);
}

}  // extern "C"
