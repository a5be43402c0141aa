"""Batch construction of an HNSW-shaped index on the GPU (SURVEY.md section 8f-2, "next" row).

The reference builds its graph by serial insertion under a write lock (idx/trees/hnsw/mod.rs:230-394); that is not a
data-parallel algorithm, so instead of porting it this builder works layer by layer on whole batches:

  * levels follow the reference's law floor(-ln U * ml), ml = 1/ln m (hnsw/mod.rs:263-266); layer l holds the elements
    of level >= l;
  * candidates of an element = its efc (150) nearest elements of the layer, from the brute-force engine in approximate
    mode -- the reference selects among the efc results of its insertion search (layer.rs:352-358); with prefix=True the
    candidates come from the id prefix [0, 2^ceil(log2 i)) only, which emulates insertion order and keeps the long-range
    links early elements get in the incremental algorithm;
  * Heuristic::select (heuristic.rs:61-81,201-216) on the GPU (sdb_hnsw_select_neighbors) picks <= m_max of them;
  * every selected edge is mirrored (graph.rs:52-64) and a node that ends up with more than m_max edges is re-selected
    among its own picks plus up to (rev_factor-1)*m_max reverse edges ordered by distance (layer.rs:362-378);
  * a candidate at a NaN distance (a zero row under cosine, a row with a NaN) is dropped before the selection, in every
    builder: nothing links to such a row, because a NaN neighbour is never rejected and stalls the searches that meet it.

The result is a valid input for the layer-walk kernel (the same CSR the reference's Hn records decode to).  It is NOT
the graph the reference would have built, so parity claims apply to the walk on a given graph; quality is measured as
recall against exact brute force next to a reference-style (oracle) graph: tests/dev/hnsw_quality.py, DESIGN.md section 6.
"""
import math

import numpy as np

from .engine import VectorColumn


def assign_levels(n, m, seed):
    rng = np.random.default_rng(seed)
    ml = 1.0 / math.log(m)
    u = rng.random(n)
    u[u == 0.0] = 0.5
    return np.floor(-np.log(u) * ml).astype(np.int64)


def _merge_reverse(fwd, cnt, m_max, cap=None):
    """bidirectional linking (graph.rs:52-64): every selected edge u->v also adds v->u; a node keeps its own
    selection first (nearest first) and fills up with reverse edges until m_max."""
    n = fwd.shape[0]
    valid = np.arange(fwd.shape[1])[None, :] < cnt[:, None]
    src = np.repeat(np.arange(n, dtype=np.int64), cnt)
    dst = fwd[valid].astype(np.int64)
    order = np.argsort(dst, kind="stable")
    dst_s, src_s = dst[order], src[order]
    start = np.searchsorted(dst_s, np.arange(n + 1))
    rank = np.arange(dst_s.size) - start[dst_s]
    cap = cap or 2 * m_max
    rev_cols = max(cap - m_max, m_max)  # reverse edges kept per node before the re-selection
    keep = rank < rev_cols
    rev = np.full((n, rev_cols), -1, np.int64)
    rev[dst_s[keep], rank[keep]] = src_s[keep]
    f = np.where(valid, fwd.astype(np.int64), -2)
    for j in range(rev_cols):  # drop reverse edges that duplicate a forward edge
        col = rev[:, j]
        dup = (f == col[:, None]).any(1)
        rev[dup, j] = -1
    allc = np.concatenate([np.where(valid, fwd.astype(np.int64), -1), rev], axis=1)
    ok = allc >= 0
    order2 = np.argsort(~ok, axis=1, kind="stable")[:, :cap]
    out = np.take_along_axis(allc, order2, axis=1)
    out_cnt = np.minimum(ok.sum(1), cap)
    return out, out_cnt


def _drop_nan(cand, dist, cnt, also=None):
    """candidate lists (CUDA (b, kc) ids and f64 distances, cnt valid entries per row) without the entries at a NaN
    distance (a zero row under cosine, a row with a NaN) or marked in `also`, order kept -> (cand, cnt).  The selection
    never rejects a NaN candidate (no comparison with NaN holds), and a linked one stops every search whose result set
    fills up with it last (no distance is < NaN): such a row is left unlinked."""
    import torch
    kc = cand.shape[1]
    pos = torch.arange(kc, device=cand.device)[None, :]
    live = pos < cnt[:, None]
    out = torch.isnan(dist) & live
    if also is not None:
        out |= also & live
    elif not bool(out.any()):
        return cand, cnt
    cand = torch.gather(cand, 1, torch.argsort(pos + out.to(torch.int64) * kc, dim=1, stable=True)).contiguous()
    return cand, (cnt - out.sum(1).to(cnt.dtype)).contiguous()


VT_TORCH = {"F64": "float64", "F32": "float32", "I64": "int64", "I32": "int32", "I16": "int16"}


def _legacy(metric, vector_type):
    """F32 COSINE / EUCLIDEAN keep the original builder: brute-force candidates and the f32 selection kernel
    (sdb_hnsw_select_neighbors), so the graphs they make do not change.  Every other combination ranks candidates
    with sdb_hnsw_knn_exact_device and selects with sdb_hnsw_select_device, both in the index's own arithmetic."""
    return vector_type.upper() == "F32" and metric.upper() in ("COSINE", "EUCLIDEAN")


def _check_x(x, n, dim, vector_type):
    import torch
    vt = vector_type.upper()
    if vt not in VT_TORCH:
        raise ValueError(f"unknown vector type {vector_type!r}")
    want = getattr(torch, VT_TORCH[vt])
    if not x.is_cuda or x.dtype != want or tuple(x.shape) != (n, dim) or not x.is_contiguous():
        raise ValueError(f"vectors must be a contiguous CUDA {want} tensor of shape ({n}, {dim}) for vector type {vt}")


def load_device(ctx, x, layers_dev, entry, metric, vector_type="F32", minkowski_order=3.0):
    """sdb_hnsw_load_device_typed: a handle that borrows x (torch CUDA (n, dim) of the type) and the device CSR layers
    [(row_ptr int64 (n+1), col_idx int32)] (layer 0 first).  The caller keeps the tensors alive."""
    import ctypes as C
    from . import _lib as L
    nl = len(layers_dev)
    h = C.c_void_p()
    L.check(L.lib().sdb_hnsw_load_device_typed(ctx.h, int(x.shape[1]), L.METRIC[metric.upper()], L.VTYPE[vector_type.upper()],
                                               int(x.shape[0]), C.c_void_p(x.data_ptr()), nl,
                                               (C.c_void_p * nl)(*[t[0].data_ptr() for t in layers_dev]),
                                               (C.c_void_p * nl)(*[t[1].data_ptr() for t in layers_dev]), int(entry), C.byref(h)))
    if metric.upper() == "MINKOWSKI":
        L.check(L.lib().sdb_hnsw_set_minkowski_order(h, float(minkowski_order)))
    return h


def set_layers(h, layers_dev, entry):
    """sdb_hnsw_set_layers_device: point a borrowed handle at other device CSR layers (its element state is kept)"""
    import ctypes as C
    from . import _lib as L
    nl = len(layers_dev)
    L.check(L.lib().sdb_hnsw_set_layers_device(h, nl, (C.c_void_p * nl)(*[t[0].data_ptr() for t in layers_dev]),
                                               (C.c_void_p * nl)(*[t[1].data_ptr() for t in layers_dev]), int(entry)))


def knn_exact(h, queries, k, members=None):
    """sdb_hnsw_knn_exact_device: for every row of `queries` (torch CUDA, the index's type) the k nearest elements of
    the handle (or of `members`, a CUDA int32 tensor of element ids) in the index's own arithmetic, ordered by
    (distance, id).  -> (ids int64 (nq, k), dist float64 (nq, k), count int32 (nq,)), CUDA tensors."""
    import ctypes as C
    import torch
    from . import _lib as L
    nq, dev = int(queries.shape[0]), queries.device
    ids = torch.zeros((nq, k), dtype=torch.int64, device=dev)
    dist = torch.zeros((nq, k), dtype=torch.float64, device=dev)
    cnt = torch.zeros((nq,), dtype=torch.int32, device=dev)
    q = queries.contiguous()
    mem = None if members is None else members.to(torch.int32).contiguous()
    torch.cuda.current_stream(dev).synchronize()  # torch wrote the inputs on ITS stream; the library runs on its own
    L.check(L.lib().sdb_hnsw_knn_exact_device(h, C.c_void_p(q.data_ptr()), nq, int(k),
                                              None if mem is None else C.c_void_p(mem.data_ptr()),
                                              0 if mem is None else int(mem.numel()), C.c_void_p(ids.data_ptr()),
                                              C.c_void_p(dist.data_ptr()), C.c_void_p(cnt.data_ptr())))
    return ids, dist, cnt


def select(h, cand, cnt, m_max, presorted, elem_ids=None, row0=0):
    """sdb_hnsw_select_device: Heuristic::select for elements elem_ids (CUDA int32) or row0 + i, from the candidate
    lists cand (CUDA int64 (n, kc) element ids) with cnt (CUDA int32 (n,)) valid entries.
    -> (picks int32 (n, m_max), count int32 (n,)), CUDA tensors."""
    import ctypes as C
    import torch
    from . import _lib as L
    cand = cand.to(torch.int64).contiguous()
    cnt = cnt.to(torch.int32).contiguous()
    n, kc = int(cand.shape[0]), int(cand.shape[1])
    ids = None if elem_ids is None else elem_ids.to(torch.int32).contiguous()
    out = torch.zeros((n, m_max), dtype=torch.int32, device=cand.device)
    ocnt = torch.zeros((n,), dtype=torch.int32, device=cand.device)
    torch.cuda.current_stream(cand.device).synchronize()
    L.check(L.lib().sdb_hnsw_select_device(h, None if ids is None else C.c_void_p(ids.data_ptr()), int(row0), n,
                                           C.c_void_p(cand.data_ptr()), C.c_void_p(cnt.data_ptr()), kc, int(m_max),
                                           int(presorted), C.c_void_p(out.data_ptr()), C.c_void_p(ocnt.data_ptr())))
    return out, ocnt


def _build_layers_typed(ctx, x, n, dim, metric, vector_type, minkowski_order, levels, m, m0, batch, progress, heuristic,
                        prefix, efc, rev_factor):
    """build_layers for every metric and type but F32 COSINE / EUCLIDEAN: the same steps, with candidates from
    sdb_hnsw_knn_exact_device over the layer's members (element ids throughout) and Heuristic::select from
    sdb_hnsw_select_device, on one handle whose adjacency is never read"""
    import torch
    dev = x.device
    top = int(levels.max()) if n else 0
    layers = []
    empty = [(torch.zeros(n + 1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))]
    h = load_device(ctx, x, empty, -1, metric, vector_type, minkowski_order)
    try:
        for l in range(top + 1):
            members = np.nonzero(levels >= l)[0].astype(np.int64)
            k_nb = m0 if l == 0 else m
            row_ptr = np.zeros(n + 1, np.uint64)
            if members.size <= 1:
                layers.append((row_ptr, np.zeros(0, np.uint32)))
                continue
            local = np.full(n, -1, np.int64)
            local[members] = np.arange(members.size)
            mem_dev = torch.from_numpy(members.astype(np.int32)).to(dev)
            kc_full = (max(2 * k_nb, min(efc, 255)) if heuristic else k_nb) + 1
            nbrs = np.zeros((members.size, k_nb), np.int64)  # member-local ids
            counts = np.zeros(members.size, np.int64)
            seg_lo = 0
            seg_hi = min(members.size, 4096) if (heuristic and prefix) else members.size
            while seg_lo < members.size:
                kc = min(kc_full, seg_hi)
                for b0 in range(seg_lo, seg_hi, batch):
                    b1 = min(seg_hi, b0 + batch)
                    q = x.index_select(0, mem_dev[b0:b1].to(torch.int64))
                    ids, dist, cnt = knn_exact(h, q, kc, mem_dev[:seg_hi])
                    ids, cnt = _drop_nan(ids, dist, cnt)
                    if heuristic:
                        s_o, s_c = select(h, ids, cnt, k_nb, 1, elem_ids=mem_dev[b0:b1])
                        sel, sc = s_o.cpu().numpy().astype(np.int64), s_c.cpu().numpy().astype(np.int64)
                        nbrs[b0:b1] = np.where(np.arange(k_nb)[None, :] < sc[:, None], local[np.maximum(sel, 0)], 0)
                        counts[b0:b1] = sc
                    else:
                        r = ids.cpu().numpy()
                        c = cnt.cpu().numpy().astype(np.int64)
                        valid = np.arange(kc)[None, :] < c[:, None]
                        keep = valid & (r != members[b0:b1][:, None])  # drop self, keep nearest-first order
                        order = np.argsort(~keep, axis=1, kind="stable")[:, :k_nb]
                        nbrs[b0:b1, : order.shape[1]] = local[np.take_along_axis(r, order, axis=1)]
                        counts[b0:b1] = np.minimum(keep.sum(1), k_nb)
                    if progress:
                        progress(l, b1, members.size)
                seg_lo, seg_hi = seg_hi, min(members.size, 2 * seg_hi)
            if heuristic:
                if progress:
                    progress(l, -1, float(counts.mean()))
                union, ucnt = _merge_reverse(nbrs, counts, k_nb, cap=rev_factor * k_nb)
                if progress:
                    progress(l, -2, float(ucnt.mean()))
                u_dev = torch.from_numpy(members[np.maximum(union, 0)]).to(dev)
                r_o, r_c = select(h, u_dev, torch.from_numpy(ucnt.astype(np.int32)).to(dev), k_nb, 0, elem_ids=mem_dev)
                nbrs = local[np.maximum(r_o.cpu().numpy().astype(np.int64), 0)]
                counts = r_c.cpu().numpy().astype(np.int64)
            deg = np.zeros(n, np.int64)
            deg[members] = counts
            row_ptr[1:] = np.cumsum(deg)
            flat = members[np.maximum(nbrs, 0)]  # local -> global element ids
            mask = np.arange(k_nb)[None, :] < counts[:, None]
            layers.append((row_ptr, flat[mask].astype(np.uint32)))
    finally:
        from . import _lib as L
        L.lib().sdb_hnsw_destroy(h)
    entry = int(np.argmax(levels)) if n else -1
    return layers, entry, levels


def build_layers(ctx, vectors_dev, n, dim, metric="EUCLIDEAN", m=16, m0=32, seed=1, batch=4096, progress=None,
                 heuristic=True, prefix=False, efc=150, rev_factor=4, levels=None, vector_type="F32", minkowski_order=3.0):
    """vectors_dev: torch CUDA tensor (n, dim) of the vector type's dtype (F64 float64, F32 float32, I64 int64, I32
    int32, I16 int16).  -> (layers, entry_point, levels) with layers = [(row_ptr u64[n+1], col_idx u32[e]), ...]
    (layer 0 first), element id = row index.  metric: any Distance; minkowski_order: p of MINKOWSKI.
    heuristic=True: candidates = 2*m_max nearest, pruned by Heuristic::select on the GPU, then bidirectional linking and
    re-selection of over-full nodes; False: plain exact m_max-NN lists.  prefix=True additionally restricts element i's
    candidates to the id prefix [0, 2^ceil(log2 i)), emulating insertion order (better cross-cluster links on strongly
    clustered data, worse on diffuse data).  F32 COSINE / EUCLIDEAN rank candidates with the brute-force engine and select
    with sdb_hnsw_select_neighbors; every other combination ranks with the exact kNN and selects with
    sdb_hnsw_select_device, in the index's own arithmetic (see _legacy)."""
    import ctypes as C
    import torch
    from . import _lib as L
    levels = assign_levels(n, m, seed) if levels is None else np.asarray(levels, np.int64)
    if not _legacy(metric, vector_type):
        _check_x(vectors_dev, n, dim, vector_type)
        return _build_layers_typed(ctx, vectors_dev, n, dim, metric, vector_type, minkowski_order, levels, m, m0, batch,
                                   progress, heuristic, prefix, efc, rev_factor)
    top = int(levels.max()) if n else 0
    layers = []
    dev = vectors_dev.device
    for l in range(top + 1):
        members = np.nonzero(levels >= l)[0].astype(np.int64)
        k_nb = m0 if l == 0 else m
        row_ptr = np.zeros(n + 1, np.uint64)
        if members.size <= 1:
            layers.append((row_ptr, np.zeros(0, np.uint32)))
            continue
        midx = torch.from_numpy(members).to(dev)
        sub = vectors_dev if members.size == n else vectors_dev.index_select(0, midx).contiguous()
        # candidates per element: efc nearest (the reference selects among the efc results of its insertion search,
        # layer.rs:352-358), +1 because the element itself comes back too
        kc_full = (max(2 * k_nb, min(efc, 255)) if heuristic else k_nb) + 1
        nbrs = np.zeros((members.size, k_nb), np.int64)
        counts = np.zeros(members.size, np.int64)
        o_r = torch.zeros((batch, kc_full), dtype=torch.int64, device=dev)
        o_d = torch.zeros((batch, kc_full), dtype=torch.float64, device=dev)
        o_c = torch.zeros((batch,), dtype=torch.int32, device=dev)
        s_o = torch.zeros((batch, k_nb), dtype=torch.int32, device=dev)
        s_c = torch.zeros((batch,), dtype=torch.int32, device=dev)
        # "insertion order" emulation: element i (ids are assumed shuffled) draws its candidates from the prefix
        # [0, 2^ceil(log2 i)) only, like an element inserted when the index held that many points -- early elements
        # therefore keep long-range links, which is what makes the incremental HNSW navigable across clusters.
        seg_lo = 0
        seg_hi = min(members.size, 4096) if (heuristic and prefix) else members.size
        while seg_lo < members.size:
            torch.cuda.current_stream().synchronize()
            col = VectorColumn(ctx, dim, metric, "F32", capacity=seg_hi)
            col.append_device(sub.data_ptr(), seg_hi)
            col.finalize()
            col.set_exact(False)  # candidate generation does not need the exactness proof
            kc = min(kc_full, seg_hi)
            for b0 in range(seg_lo, seg_hi, batch):
                b1 = min(seg_hi, b0 + batch)
                q = sub[b0:b1].to(torch.float64).contiguous()
                torch.cuda.current_stream().synchronize()  # torch wrote q on ITS stream; the library runs on its own
                o_rv = o_r.view(-1)[: batch * kc].view(batch, kc)
                o_dv = o_d.view(-1)[: batch * kc].view(batch, kc)
                col.knn_device(q.data_ptr(), b1 - b0, kc, 0, o_rv.data_ptr(), o_dv.data_ptr(), o_c.data_ptr())
                c_r, c_c = _drop_nan(o_rv[: b1 - b0], o_dv[: b1 - b0], o_c[: b1 - b0])
                torch.cuda.current_stream().synchronize()
                if heuristic:
                    L.check(L.lib().sdb_hnsw_select_neighbors(ctx.h, C.c_void_p(sub.data_ptr()), dim, L.METRIC[metric.upper()],
                                                              b0, b1 - b0, C.c_void_p(c_r.data_ptr()), C.c_void_p(c_c.data_ptr()),
                                                              kc, k_nb, 1, C.c_void_p(s_o.data_ptr()), C.c_void_p(s_c.data_ptr())))
                    nbrs[b0:b1] = s_o[: b1 - b0].cpu().numpy()
                    counts[b0:b1] = s_c[: b1 - b0].cpu().numpy()
                else:
                    r = c_r.cpu().numpy()
                    cnt = c_c.cpu().numpy().astype(np.int64)
                    valid = np.arange(kc)[None, :] < cnt[:, None]
                    keep = valid & (r != (b0 + np.arange(b1 - b0))[:, None])  # drop self, keep nearest-first order
                    order = np.argsort(~keep, axis=1, kind="stable")[:, :k_nb]
                    nbrs[b0:b1, : order.shape[1]] = np.take_along_axis(r, order, axis=1)
                    counts[b0:b1] = np.minimum(keep.sum(1), k_nb)
                if progress:
                    progress(l, b1, members.size)
            col.close()
            seg_lo, seg_hi = seg_hi, min(members.size, 2 * seg_hi)
        if heuristic:
            # bidirectional edges, then re-select every over-full node among (own selection + reverse edges) ordered by
            # distance -- layer.rs:362-378
            if progress:
                progress(l, -1, float(counts.mean()))
            union, ucnt = _merge_reverse(nbrs, counts, k_nb, cap=rev_factor * k_nb)
            if progress:
                progress(l, -2, float(ucnt.mean()))
            u_dev = torch.from_numpy(np.maximum(union, 0).astype(np.int64)).to(dev)
            c_dev = torch.from_numpy(ucnt.astype(np.int32)).to(dev)
            r_o = torch.zeros((members.size, k_nb), dtype=torch.int32, device=dev)
            r_c = torch.zeros((members.size,), dtype=torch.int32, device=dev)
            torch.cuda.current_stream().synchronize()
            L.check(L.lib().sdb_hnsw_select_neighbors(ctx.h, C.c_void_p(sub.data_ptr()), dim, L.METRIC[metric.upper()], 0,
                                                      members.size, C.c_void_p(u_dev.data_ptr()), C.c_void_p(c_dev.data_ptr()),
                                                      rev_factor * k_nb, k_nb, 0, C.c_void_p(r_o.data_ptr()), C.c_void_p(r_c.data_ptr())))
            nbrs = r_o.cpu().numpy().astype(np.int64)
            counts = r_c.cpu().numpy().astype(np.int64)
        deg = np.zeros(n, np.int64)
        deg[members] = counts
        row_ptr[1:] = np.cumsum(deg)
        col_idx = np.zeros(int(row_ptr[-1]), np.uint32)
        flat = members[np.maximum(nbrs, 0)]  # local -> global element ids
        mask = np.arange(k_nb)[None, :] < counts[:, None]
        col_idx[:] = flat[mask].astype(np.uint32)
        layers.append((row_ptr, col_idx))
    entry = int(np.argmax(levels)) if n else -1
    return layers, entry, levels


def build_incremental(ctx, x, metric="COSINE", m=16, m0=32, efc=150, seed=1, growth=0.25, boot_min=65536,
                      search_chunk=1 << 16, rev_extra=32, progress=None, settle=True, vector_type="F32",
                      minkowski_order=3.0):
    """Batched TRUE insertion (SURVEY 8f-2): the reference inserts one element at a time -- search the current graph
    with efc, select <= m_max neighbours with the heuristic, link both ways, re-select over-full neighbours
    (hnsw/mod.rs:297-377, hnsw/layer.rs:342-387).  Here the same four steps run for a whole BATCH of new elements
    against the graph built so far, with the layer-walk kernel itself as the insertion search
    (sdb_hnsw_load_device + sdb_hnsw_search_device), Heuristic::select on the GPU (sdb_hnsw_select_neighbors[_ids]) and
    the linking as a handful of device-side scatter operations.  Batches grow geometrically (`growth` x the current
    size), so every element is inserted into a graph at least 1 / (1 + growth) of the size it would have seen in the
    serial algorithm; elements of one batch do not see each other.

    Elements are first re-ordered by level (highest first, random inside a level -- ids are assumed exchangeable), so
    the upper layers and a bootstrap prefix are complete before the bulk of layer 0 arrives; that prefix (every element
    of level >= 1, at least `boot_min`) is built by the kNN batch builder above.

    F32 COSINE / EUCLIDEAN re-wrap the growing graph with sdb_hnsw_load_device for every search and select with
    sdb_hnsw_select_neighbors[_ids]; every other metric and type keeps one handle (sdb_hnsw_load_device_typed), re-points
    it at the grown graph with sdb_hnsw_set_layers_device, so the elements' metric state is computed once, and selects
    with sdb_hnsw_select_device in the index's arithmetic.

    x: torch CUDA (n, dim) of the vector type's dtype (see build_layers).  Returns a dict: x (re-ordered copy, device), order (new -> original index, numpy),
    layers_dev [(row_ptr int64 (n+1), col_idx int32)] layer 0 first (device tensors, CSR over NEW ids), entry (new id),
    levels (new order)."""
    import ctypes as C
    import torch
    from . import _lib as L
    n, dim = x.shape
    dev = x.device
    levels = assign_levels(n, m, seed)
    order = np.argsort(-levels, kind="stable")
    levels = levels[order]
    x = x.index_select(0, torch.from_numpy(order).to(dev)).contiguous()
    n_up = int((levels >= 1).sum())
    n_boot = min(n, max(n_up, boot_min))
    torch.cuda.synchronize()
    boot_layers, entry, _ = build_layers(ctx, x[:n_boot], n_boot, dim, metric, m=m, m0=m0, seed=seed, prefix=True, efc=efc,
                                         levels=levels[:n_boot], progress=progress, vector_type=vector_type,
                                         minkowski_order=minkowski_order)
    n_layers = len(boot_layers)
    # upper layers are final: CSR over all n ids (rows >= n_boot are empty)
    upper = []
    for l in range(1, n_layers):
        rp, ci = boot_layers[l]
        rp_full = np.full(n + 1, rp[-1], np.int64)
        rp_full[: n_boot + 1] = rp.astype(np.int64)
        upper.append((torch.from_numpy(rp_full).to(dev), torch.from_numpy(ci.astype(np.int32) if ci.size else np.zeros(1, np.int32)).to(dev)))
    # layer 0 as fixed-width adjacency while it grows
    adj0 = torch.full((n, m0), -1, dtype=torch.int32, device=dev)
    deg0 = torch.zeros(n, dtype=torch.int32, device=dev)
    rp0, ci0 = boot_layers[0]
    d0 = np.diff(rp0.astype(np.int64))
    rows = np.repeat(np.arange(n_boot), d0)
    cols = np.arange(ci0.size) - np.repeat(rp0[:-1].astype(np.int64), d0)
    adj0[torch.from_numpy(rows).to(dev), torch.from_numpy(cols).to(dev)] = torch.from_numpy(ci0.astype(np.int32)).to(dev)
    deg0[:n_boot] = torch.from_numpy(d0.astype(np.int32)).to(dev)
    mcode = L.METRIC[metric.upper()]
    col_ids = torch.arange(m0, device=dev, dtype=torch.int32)[None, :]

    def csr0():
        rp = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        rp[1:] = torch.cumsum(deg0.to(torch.int64), 0)
        ci = adj0[col_ids < deg0[:, None]]
        if ci.numel() == 0:
            ci = torch.zeros(1, dtype=torch.int32, device=dev)
        return rp, ci.contiguous()

    typed = not _legacy(metric, vector_type)
    held = [[csr0()] + upper]  # the adjacency the typed handle borrows
    th = load_device(ctx, x, held[0], entry, metric, vector_type, minkowski_order) if typed else None

    def search_select(lo, hi, drop_self):
        """insertion search of elements [lo, hi) on the current graph + Heuristic::select -> (sel (b, m0) int32, count)"""
        b = hi - lo
        rp, ci = csr0()
        lay = [(rp, ci)] + upper
        torch.cuda.synchronize()
        if typed:
            set_layers(th, lay, entry)
            held[0] = lay
            h = th
        else:
            RP = (C.c_void_p * n_layers)(*[t[0].data_ptr() for t in lay])
            CI = (C.c_void_p * n_layers)(*[t[1].data_ptr() for t in lay])
            h = C.c_void_p()
            L.check(L.lib().sdb_hnsw_load_device(ctx.h, dim, mcode, n, C.c_void_p(x.data_ptr()), n_layers, RP, CI, int(entry), C.byref(h)))
        sel = torch.empty((b, m0), dtype=torch.int32, device=dev)
        scnt = torch.empty((b,), dtype=torch.int32, device=dev)
        try:
            for c0 in range(0, b, search_chunk):
                c1 = min(b, c0 + search_chunk)
                nqc = c1 - c0
                cand = torch.empty((nqc, efc), dtype=torch.int64, device=dev)
                cdist = torch.empty((nqc, efc), dtype=torch.float64, device=dev)
                ccnt = torch.empty((nqc,), dtype=torch.int32, device=dev)
                torch.cuda.synchronize()
                L.check(L.lib().sdb_hnsw_search_device(h, C.c_void_p(x[lo + c0].data_ptr()), nqc, efc, efc,
                                                       C.c_void_p(cand.data_ptr()), C.c_void_p(cdist.data_ptr()),
                                                       C.c_void_p(ccnt.data_ptr())))
                # candidates at a NaN distance leave the list (_drop_nan); second pass: the element is part of the graph
                # by now and leaves its own list too
                me = torch.arange(lo + c0, lo + c1, device=dev, dtype=torch.int64)[:, None]
                cand, ccnt = _drop_nan(cand, cdist, ccnt, (cand == me) if drop_self else None)
                torch.cuda.synchronize()
                if typed:
                    L.check(L.lib().sdb_hnsw_select_device(h, None, lo + c0, nqc, C.c_void_p(cand.data_ptr()),
                                                           C.c_void_p(ccnt.data_ptr()), efc, m0, 1,
                                                           C.c_void_p(sel[c0:c1].data_ptr()), C.c_void_p(scnt[c0:c1].data_ptr())))
                else:
                    L.check(L.lib().sdb_hnsw_select_neighbors(ctx.h, C.c_void_p(x.data_ptr()), dim, mcode, lo + c0, nqc,
                                                              C.c_void_p(cand.data_ptr()), C.c_void_p(ccnt.data_ptr()), efc, m0, 1,
                                                              C.c_void_p(sel[c0:c1].data_ptr()), C.c_void_p(scnt[c0:c1].data_ptr())))
                del cand, cdist, ccnt
        finally:
            if not typed:
                L.lib().sdb_hnsw_destroy(h)
        return sel, scnt

    def link(lo, hi, sel, scnt, dedup):
        """forward edges of [lo, hi) := sel; reverse edges into the targets, re-selecting the nodes that overflow m0"""
        b = hi - lo
        valid = col_ids < scnt[:, None]
        adj0[lo:hi] = torch.where(valid, sel, torch.full_like(sel, -1))
        deg0[lo:hi] = scnt
        src = torch.arange(lo, hi, device=dev, dtype=torch.int32)[:, None].expand(b, m0)[valid]
        dst = sel[valid].to(torch.int64)
        if dedup and dst.numel():  # the target may hold this edge already (second pass over the same elements)
            keep = torch.ones(dst.numel(), dtype=torch.bool, device=dev)
            for e0 in range(0, dst.numel(), 1 << 22):
                e1 = min(dst.numel(), e0 + (1 << 22))
                keep[e0:e1] = ~(adj0[dst[e0:e1]] == src[e0:e1, None]).any(1)
            src, dst = src[keep], dst[keep]
        if not dst.numel():
            return
        dst_s, perm = torch.sort(dst, stable=True)
        src_s = src[perm]
        uniq, counts = torch.unique_consecutive(dst_s, return_counts=True)
        start = torch.cumsum(counts, 0) - counts
        rank = torch.arange(dst_s.numel(), device=dev) - torch.repeat_interleave(start, counts)
        pos = deg0[dst_s].to(torch.int64) + rank
        ok = pos < m0
        adj0[dst_s[ok], pos[ok]] = src_s[ok]
        new_deg = deg0[uniq].to(torch.int64) + counts
        deg0[uniq] = torch.clamp(new_deg, max=m0).to(torch.int32)
        over = new_deg > m0
        ov_nodes = uniq[over]
        n_ov = int(ov_nodes.numel())
        if n_ov:
            # re-select the over-full nodes among their m0 current edges + the reverse edges that did not fit
            kc = m0 + rev_extra
            union = torch.full((n_ov, kc), 0, dtype=torch.int64, device=dev)
            union[:, :m0] = adj0[ov_nodes].to(torch.int64)
            node_slot = torch.full((n,), -1, dtype=torch.int64, device=dev)
            node_slot[ov_nodes] = torch.arange(n_ov, device=dev)
            ex_dst, ex_src, ex_rank = dst_s[~ok], src_s[~ok], (pos[~ok] - m0)
            keep = ex_rank < rev_extra
            union[node_slot[ex_dst[keep]], m0 + ex_rank[keep]] = ex_src[keep].to(torch.int64)
            ucnt = (m0 + torch.clamp(new_deg[over] - m0, max=rev_extra)).to(torch.int32)
            out = torch.empty((n_ov, m0), dtype=torch.int32, device=dev)
            ocnt = torch.empty((n_ov,), dtype=torch.int32, device=dev)
            ids32 = ov_nodes.to(torch.int32).contiguous()
            torch.cuda.synchronize()
            if typed:
                L.check(L.lib().sdb_hnsw_select_device(th, C.c_void_p(ids32.data_ptr()), 0, n_ov, C.c_void_p(union.data_ptr()),
                                                       C.c_void_p(ucnt.data_ptr()), kc, m0, 0, C.c_void_p(out.data_ptr()),
                                                       C.c_void_p(ocnt.data_ptr())))
            else:
                L.check(L.lib().sdb_hnsw_select_neighbors_ids(ctx.h, C.c_void_p(x.data_ptr()), dim, mcode, C.c_void_p(ids32.data_ptr()),
                                                              n_ov, C.c_void_p(union.data_ptr()), C.c_void_p(ucnt.data_ptr()), kc, m0, 0,
                                                              C.c_void_p(out.data_ptr()), C.c_void_p(ocnt.data_ptr())))
            v2 = col_ids < ocnt[:, None]
            adj0[ov_nodes] = torch.where(v2, out, torch.full_like(out, -1))
            deg0[ov_nodes] = ocnt

    n_cur = n_boot
    try:
        while n_cur < n:
            b = int(min(n - n_cur, max(4096, int(n_cur * growth))))
            sel, scnt = search_select(n_cur, n_cur + b, False)
            link(n_cur, n_cur + b, sel, scnt, False)
            if settle:
                # Elements of one batch did not see each other.  Second pass: the same insertion search on the graph that
                # now holds the whole batch, so close neighbours that arrived together get linked (serial insertion would
                # have linked the later one to the earlier one).
                sel, scnt = search_select(n_cur, n_cur + b, True)
                link(n_cur, n_cur + b, sel, scnt, True)
            if progress:
                progress(0, n_cur + b, n)
            n_cur += b
    finally:
        if typed:
            L.lib().sdb_hnsw_destroy(th)
    rp, ci = csr0()
    return {"x": x, "order": order, "layers_dev": [(rp, ci)] + upper, "entry": int(entry), "levels": levels}
