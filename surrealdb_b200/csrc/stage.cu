// stage.cu -- staging decoders: the reference's persisted HNSW formats -> device-resident arrays (SURVEY 8a row a14).
//
//   He value  = revisioned SerializedVector (idx/trees/vector.rs:32-56): [revision=1][variant][len][elements],
//               elements as raw little-endian fixed-width values (the `specialised-vectors` feature of the
//               `revision` crate, Cargo.toml:70-79).  Variant order F64,F32,I64,I32,I16 (vector.rs:34-41).
//               Byte layout pinned by the five known-answer keys of key/index/hv.rs:72-101 (dim 3).
//   Hn value  = UndirectedGraph::node_to_val (idx/trees/graph.rs:104-115): BE u16 count, then count BE u64 ids;
//               load_node (graph.rs:117-126) inserts them one by one into the node's set, so a repeated id is
//               dropped and the FIRST occurrence keeps its position.
//
// PARITY UNPINNED: the multi-byte length prefix of `revision 0.17.0` (un-vendored) for len >= 251 is recalled
// from upstream (bincode-style: 0xFB + u16 LE, 0xFC + u32 LE, 0xFD + u64 LE); the reference's own KATs only cover
// len = 3.  It is isolated in read_varint() below (and in surrealdb_b200/staging.py for the Hs state).
//
// Both decoders are HBM-bound byte work: one warp per KV value, unaligned payloads read as aligned 32-bit words
// and funnel-shifted, ids byte-swapped with PRMT.
#include "internal.cuh"

namespace sdb {

__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  const uint32_t lo = __ldg(w);
  if (sh == 0) return lo;
  return __funnelshift_r(lo, __ldg(w + 1), sh);  // the blob copy is padded, w+1 is always readable
}
__device__ __forceinline__ uint64_t ld_u64_unaligned(const uint8_t* p) {
  return (uint64_t)ld_u32_unaligned(p) | ((uint64_t)ld_u32_unaligned(p + 4) << 32);
}
__device__ __forceinline__ uint64_t bswap64(uint64_t v) {
  const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
  return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}
// `revision` variable-length unsigned integer.  Returns false on truncated / unsupported input.
__device__ __forceinline__ bool read_varint(const uint8_t*& p, const uint8_t* end, uint64_t& v) {
  if (p >= end) return false;
  const uint8_t b = *p++;
  if (b < 251) {
    v = b;
    return true;
  }
  const int nb = b == 251 ? 2 : b == 252 ? 4 : b == 253 ? 8 : 0;
  if (nb == 0 || p + nb > end) return false;
  v = 0;
  for (int i = 0; i < nb; i++) v |= (uint64_t)p[i] << (8 * i);
  p += nb;
  return true;
}

// ---- He: one warp per value ----------------------------------------------------------------------
// VARIANT < 0: every variant is converted to OUT (f32 / f64; a value OUT cannot represent counts as bad).  VARIANT >= 0:
// OUT is that variant's own element type and only values of that variant are accepted (native typed indexes).
template <typename OUT, int VARIANT = -1>
__global__ void __launch_bounds__(256) stage_vectors_kernel(const uint8_t* __restrict__ blob, uint64_t blob_base,
                                                            const uint64_t* __restrict__ off,
                                                            const uint64_t* __restrict__ ids, uint64_t id0, uint64_t n,
                                                            uint32_t dim, uint64_t n_rows, OUT* __restrict__ out,
                                                            uint8_t* __restrict__ present,
                                                            unsigned long long* __restrict__ n_bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t v = warp0; v < n; v += n_warps) {
    const uint8_t* p = blob + (off[v] - blob_base);
    const uint8_t* end = blob + (off[v + 1] - blob_base);
    const uint64_t row = ids ? ids[v] : id0 + v;
    uint64_t rev = 0, variant = 0, len = 0;
    bool ok = read_varint(p, end, rev) && rev == 1 && read_varint(p, end, variant) && variant <= 4 &&
              (VARIANT < 0 || variant == (uint64_t)VARIANT) && read_varint(p, end, len) && len == dim && row < n_rows;
    const uint32_t esz = (variant == 0 || variant == 2) ? 8u : variant == 4 ? 2u : 4u;
    ok = ok && (uint64_t)(end - p) == (uint64_t)dim * esz;
    if (!ok) {  // uniform across the warp (every lane parsed the same header)
      if (lane == 0) atomicAdd(n_bad, 1ull);
      continue;
    }
    OUT* o = out + row * dim;
    bool inexact = false;
    for (uint32_t c = lane; c < dim; c += 32) {
      OUT r;
      switch ((int)variant) {
        case 0: {  // F64
          const double x = __longlong_as_double((long long)ld_u64_unaligned(p + 8ull * c));
          r = (OUT)x;
          inexact |= ((double)r != x) && (x == x);
        } break;
        case 1: r = (OUT)__uint_as_float(ld_u32_unaligned(p + 4ull * c)); break;  // F32: exact into f32 and f64
        case 2: {  // I64
          const long long x = (long long)ld_u64_unaligned(p + 8ull * c);
          r = (OUT)x;
          inexact |= (long long)r != x;
        } break;
        case 3: {  // I32
          const int x = (int)ld_u32_unaligned(p + 4ull * c);
          r = (OUT)x;
          inexact |= (int)r != x;
        } break;
        default: {  // I16
          const uint32_t w = ld_u32_unaligned(p + 2ull * (c & ~1u));
          r = (OUT)(short)((c & 1u) ? (w >> 16) : (w & 0xFFFFu));
        } break;
      }
      o[c] = r;
    }
    inexact = __any_sync(0xffffffffu, inexact);
    if (lane == 0) {
      if (present) present[row] = 1;
      if (inexact) atomicAdd(n_bad, 1ull);  // value not representable in the requested element type
    }
  }
}

// ---- Hn: one warp per node value; pass 0 counts distinct neighbours, pass 1 writes them ------------------
template <bool FILL>
__global__ void __launch_bounds__(256) stage_nodes_kernel(const uint8_t* __restrict__ blob,
                                                          const uint64_t* __restrict__ off,
                                                          const uint64_t* __restrict__ node_ids, uint64_t n,
                                                          uint64_t n_elems, uint64_t* __restrict__ deg_or_rowptr,
                                                          uint32_t* __restrict__ col_idx,
                                                          unsigned long long* __restrict__ n_bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t v = warp0; v < n; v += n_warps) {
    const uint8_t* p = blob + off[v];
    const uint64_t bytes = off[v + 1] - off[v];
    const uint64_t node = node_ids[v];
    uint32_t cnt = 0;
    bool ok = bytes >= 2 && node < n_elems;
    if (ok) {
      cnt = ((uint32_t)p[0] << 8) | p[1];
      ok = bytes == 2 + 8ull * cnt;
    }
    if (!ok) {
      if (!FILL && lane == 0) atomicAdd(n_bad, 1ull);
      continue;
    }
    const uint8_t* e = p + 2;
    uint64_t base = FILL ? deg_or_rowptr[node] : 0;
    uint32_t kept = 0;
    for (uint32_t c0 = 0; c0 < cnt; c0 += 32) {
      const uint32_t j = c0 + lane;
      const bool valid = j < cnt;
      const uint64_t id = valid ? bswap64(ld_u64_unaligned(e + 8ull * j)) : ~0ull - lane;
      bool keep = valid && id < n_elems;
      if (!FILL && valid && id >= n_elems) atomicAdd(n_bad, 1ull);  // edge to an element the index does not hold
      // first occurrence wins (DynamicSet::insert): inside this group of 32 ...
      const uint32_t same = __match_any_sync(0xffffffffu, id);
      if (same & ((1u << lane) - 1u)) keep = false;
      // ... and against the earlier groups (only for nodes with more than 32 neighbours)
      for (uint32_t t = 0; t < c0 && keep; t++) keep = bswap64(ld_u64_unaligned(e + 8ull * t)) != id;
      const uint32_t km = __ballot_sync(0xffffffffu, keep);
      if (FILL && keep) col_idx[base + kept + __popc(km & ((1u << lane) - 1u))] = (uint32_t)id;
      kept += __popc(km);
    }
    if (!FILL && lane == 0) {
      if (atomicExch((unsigned long long*)&deg_or_rowptr[node], (unsigned long long)kept) != 0ull && kept)
        atomicAdd(n_bad, 1ull);  // the same node key twice (cannot happen in a KV range scan)
    }
  }
}

// host blob (any memory) -> padded device copy
static sdb_status blob_to_device(const uint8_t* blob, uint64_t bytes, DevBuf<uint8_t>* d_out, cudaStream_t st) {
  DevBuf<uint8_t>& d = *d_out;
  cudaError_t e = d.reserve(bytes + 16);
  if (e != cudaSuccess) {
    set_error("staging: cannot allocate %llu bytes for the value blob: %s", (unsigned long long)bytes, cudaGetErrorString(e));
    return SDB_ENOMEM;
  }
  if (bytes) SDB_CUDA(cudaMemcpyAsync(d, blob, bytes, cudaMemcpyHostToDevice, st));
  SDB_CUDA(cudaMemsetAsync(d + bytes, 0, 16, st));
  return SDB_OK;
}

sdb_status stage_decode_vectors(Ctx* ctx, const uint8_t* blob, const uint64_t* off, const uint64_t* ids, uint64_t n,
                                uint32_t dim, sdb_dtype out_dtype, uint64_t n_rows, void* d_out, uint8_t* d_present,
                                uint64_t* n_bad, cudaStream_t st, int native) {
  DevBuf<unsigned long long> d_bad;
  SDB_CUDA(d_bad.reserve(1));
  SDB_CUDA(cudaMemsetAsync(d_bad, 0, 8, st));
  // chunked so that the staging copy stays small next to a 10M x 768 index (30 GB of He values)
  const uint64_t CHUNK_BYTES = 512ull << 20, CHUNK_VALS = 4ull << 20;
  DevBuf<uint8_t> d_blob;
  DevBuf<uint64_t> d_off, d_ids;
  sdb_status rc = SDB_OK;
  for (uint64_t v0 = 0; v0 < n && rc == SDB_OK;) {
    uint64_t v1 = v0 + 1;
    while (v1 < n && v1 - v0 < CHUNK_VALS && off[v1 + 1] - off[v0] <= CHUNK_BYTES) v1++;
    const uint64_t bytes = off[v1] - off[v0], nv = v1 - v0;
    if (d_blob.reserve(bytes + 16) != cudaSuccess) {
      set_error("staging: cannot allocate the %llu-byte staging chunk", (unsigned long long)(bytes + 16));
      rc = SDB_ENOMEM;
      break;
    }
    if (d_off.reserve(nv + 1) != cudaSuccess || d_ids.reserve(nv) != cudaSuccess) {
      rc = SDB_ENOMEM;
      break;
    }
    auto chk = [&](cudaError_t e) {
      if (e != cudaSuccess && rc == SDB_OK) {
        set_error("staging: %s", cudaGetErrorString(e));
        rc = SDB_ECUDA;
      }
    };
    chk(cudaMemcpyAsync(d_blob, blob + off[v0], bytes, cudaMemcpyHostToDevice, st));
    chk(cudaMemsetAsync(d_blob + bytes, 0, 16, st));
    chk(cudaMemcpyAsync(d_off, off + v0, 8 * (nv + 1), cudaMemcpyHostToDevice, st));
    if (ids) chk(cudaMemcpyAsync(d_ids, ids + v0, 8 * nv, cudaMemcpyHostToDevice, st));
    if (rc != SDB_OK) break;
    const unsigned grid = (unsigned)std::min<uint64_t>((nv + 7) / 8, (uint64_t)ctx->sm_count * 16);
    const uint64_t* d_ids_or_null = ids ? d_ids.get() : nullptr;
    switch (native) {  // sdb_vector_type numbers = SerializedVector variants
      case 0: stage_vectors_kernel<double, 0><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, d_ids_or_null, v0, nv, dim, n_rows, (double*)d_out, d_present, d_bad); break;
      case 1: stage_vectors_kernel<float, 1><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, d_ids_or_null, v0, nv, dim, n_rows, (float*)d_out, d_present, d_bad); break;
      case 2: stage_vectors_kernel<long long, 2><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, d_ids_or_null, v0, nv, dim, n_rows, (long long*)d_out, d_present, d_bad); break;
      case 3: stage_vectors_kernel<int, 3><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, d_ids_or_null, v0, nv, dim, n_rows, (int*)d_out, d_present, d_bad); break;
      case 4: stage_vectors_kernel<short, 4><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, d_ids_or_null, v0, nv, dim, n_rows, (short*)d_out, d_present, d_bad); break;
      default:
        if (out_dtype == SDB_F32)
          stage_vectors_kernel<float><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, ids ? d_ids.get() : nullptr, v0, nv, dim, n_rows,
                                                            (float*)d_out, d_present, d_bad);
        else
          stage_vectors_kernel<double><<<grid, 256, 0, st>>>(d_blob, off[v0], d_off, ids ? d_ids.get() : nullptr, v0, nv, dim,
                                                             n_rows, (double*)d_out, d_present, d_bad);
    }
    count_launch(ctx);
    chk(cudaGetLastError());
    chk(cudaStreamSynchronize(st));  // the host source of the next chunk's copy may be pageable: keep it simple
    v0 = v1;
  }
  unsigned long long h_bad = 0;
  if (rc == SDB_OK && cudaMemcpy(&h_bad, d_bad, 8, cudaMemcpyDeviceToHost) != cudaSuccess) rc = SDB_ECUDA;
  if (n_bad) *n_bad = h_bad;
  return rc;
}

sdb_status stage_decode_nodes(Ctx* ctx, const uint8_t* blob, const uint64_t* off, const uint64_t* node_ids, uint64_t n,
                              uint64_t n_elems, DevBuf<uint64_t>* d_row_ptr_out, DevBuf<uint32_t>* d_col_idx_out,
                              uint64_t* n_edges, uint64_t* n_bad, cudaStream_t st) {
  DevBuf<uint8_t> d_blob;
  DevBuf<uint64_t> d_off, d_ids, d_rp, d_tot;
  DevBuf<uint32_t> d_ci;
  DevBuf<unsigned long long> d_bad;
  const uint64_t bytes = n ? off[n] : 0;
  SDB_TRY(blob_to_device(blob, bytes, &d_blob, st));
  cudaError_t e = d_off.reserve(n + 1);
  if (e == cudaSuccess) e = d_ids.reserve(n ? n : 1);
  if (e == cudaSuccess) e = d_rp.reserve(n_elems + 1);
  if (e == cudaSuccess) e = d_tot.reserve(1);
  if (e == cudaSuccess) e = d_bad.reserve(1);
  if (e != cudaSuccess) {
    set_error("staging: device allocation failed: %s", cudaGetErrorString(e));
    return SDB_ENOMEM;
  }
  if (n) {
    SDB_CUDA(cudaMemcpyAsync(d_off, off, 8 * (n + 1), cudaMemcpyHostToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(d_ids, node_ids, 8 * n, cudaMemcpyHostToDevice, st));
  }
  SDB_CUDA(cudaMemsetAsync(d_rp, 0, 8 * (n_elems + 1), st));
  SDB_CUDA(cudaMemsetAsync(d_bad, 0, 8, st));
  const unsigned grid = (unsigned)std::min<uint64_t>((n + 7) / 8 + 1, (uint64_t)ctx->sm_count * 16);
  if (n) {
    stage_nodes_kernel<false><<<grid, 256, 0, st>>>(d_blob, d_off, d_ids, n, n_elems, d_rp, nullptr, d_bad);
    count_launch(ctx);
  }
  SDB_TRY(exclusive_scan(ctx, d_rp, d_rp, n_elems + 1, d_tot, st));
  uint64_t total = 0;
  SDB_CUDA(cudaMemcpyAsync(&total, d_tot, 8, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (d_ci.reserve(total ? total : 1) != cudaSuccess) {
    set_error("staging: cannot allocate col_idx for %llu edges", (unsigned long long)total);
    return SDB_ENOMEM;
  }
  if (n) {
    stage_nodes_kernel<true><<<grid, 256, 0, st>>>(d_blob, d_off, d_ids, n, n_elems, d_rp, d_ci, d_bad);
    count_launch(ctx);
  }
  unsigned long long h_bad = 0;
  SDB_CUDA(cudaMemcpyAsync(&h_bad, d_bad, 8, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  SDB_CUDA(cudaGetLastError());
  *d_row_ptr_out = std::move(d_rp);
  *d_col_idx_out = std::move(d_ci);
  if (n_edges) *n_edges = total;
  if (n_bad) *n_bad = h_bad;
  return SDB_OK;
}

}  // namespace sdb

using namespace sdb;

extern "C" {

sdb_status sdb_stage_decode_vectors(sdb_ctx* ctx, const uint8_t* blob, const uint64_t* off, const uint64_t* elem_ids,
                                    uint64_t n, uint32_t dim, sdb_dtype out_dtype, uint64_t n_rows, void* d_out_rows,
                                    uint8_t* d_present, uint64_t* n_bad) {
  if (!ctx || (n && (!blob || !off)) || !dim || !d_out_rows || (out_dtype != SDB_F32 && out_dtype != SDB_F64)) {
    set_error("sdb_stage_decode_vectors: bad argument");
    return SDB_EINVAL;
  }
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  return stage_decode_vectors(ctx, blob, off, elem_ids, n, dim, out_dtype, n_rows, d_out_rows, d_present, n_bad,
                              ctx->stream);
}

sdb_status sdb_stage_decode_nodes(sdb_ctx* ctx, const uint8_t* blob, const uint64_t* off, const uint64_t* node_ids,
                                  uint64_t n, uint64_t n_elems, uint64_t** out_row_ptr, uint32_t** out_col_idx,
                                  uint64_t* n_bad) {
  if (!ctx || (n && (!blob || !off || !node_ids)) || !out_row_ptr || !out_col_idx || n_elems >= 0xFFFFFFF0ull) {
    set_error("sdb_stage_decode_nodes: bad argument");
    return SDB_EINVAL;
  }
  std::lock_guard<std::mutex> guard(ctx->mu);
  SDB_CUDA(cudaSetDevice(ctx->device));
  DevBuf<uint64_t> d_rp;
  DevBuf<uint32_t> d_ci;
  uint64_t total = 0;
  SDB_TRY(stage_decode_nodes(ctx, blob, off, node_ids, n, n_elems, &d_rp, &d_ci, &total, n_bad, ctx->stream));
  uint64_t* h_rp = (uint64_t*)malloc(8 * (n_elems + 1));
  uint32_t* h_ci = (uint32_t*)malloc(4 * (total ? total : 1));
  cudaError_t e = cudaSuccess;
  if (h_rp && h_ci) {
    e = cudaMemcpy(h_rp, d_rp, 8 * (n_elems + 1), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && total) e = cudaMemcpy(h_ci, d_ci, 4 * total, cudaMemcpyDeviceToHost);
  }
  if (!h_rp || !h_ci || e != cudaSuccess) {
    free(h_rp);
    free(h_ci);
    set_error("sdb_stage_decode_nodes: %s", e != cudaSuccess ? cudaGetErrorString(e) : "host allocation failed");
    return e != cudaSuccess ? SDB_ECUDA : SDB_ENOMEM;
  }
  *out_row_ptr = h_rp;
  *out_col_idx = h_ci;
  return SDB_OK;
}

}  // extern "C"
