#!/usr/bin/env python
"""Secondary measurements for the other rows of SURVEY.md section 8 (NOT the driver's headline line):

  python bench_extra.py hnsw  [--rows N --dim D --queries Q --ef 64 --k 10 --metric M --graph-metric G --vector-type T
                               --build-in-type]
  python bench_extra.py graph [--log2-nodes 24 --edges E --sources 1024 --hops 3]

Each prints one JSON line with the metric, a roofline object computed from in-kernel counters
(HNSW: visited*(4D+4) + expanded*deg*4 bytes; graph: 16|F| + 8|E_h| per hop), and a cpu_baseline obtained by
timing the oracle (port of the reference algorithm) on the host cores for the same inputs (bounded sample).
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], "measured"
    return 6650.0, "fallback"


def dev_time_ms(ctx, fn):
    import torch
    st = torch.cuda.ExternalStream(ctx.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record(st)
    out = fn()
    e1.record(st)
    e1.synchronize()
    return out, e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3


def bench_hnsw(a):
    import torch
    from surrealdb_b200 import Context, HnswIndex
    from surrealdb_b200.hnsw_build import build_layers
    ctx = Context(0)
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0x5DB00003)
    n, dim = a.rows, a.dim
    gm = (a.graph_metric or a.metric).upper()  # metric the graph is linked with
    centers = torch.nn.functional.normalize(torch.randn((4096, dim), generator=g, device=dev), dim=1)
    def sample(cnt):
        # sigma = TOTAL noise norm relative to the unit-norm centroid (per-coordinate sigma / sqrt(dim)); a per-coordinate
        # 0.15 would bury the centroids under isotropic noise in high dimension and make every ANN method degenerate
        out = torch.empty((cnt, dim), dtype=torch.float32, device=dev)
        for r0 in range(0, cnt, 1 << 20):  # in slabs: 10M x 768 would otherwise need three 31 GB temporaries
            r1 = min(cnt, r0 + (1 << 20))
            c = torch.randint(0, 4096, (r1 - r0,), generator=g, device=dev)
            out[r0:r1] = centers[c] + (a.sigma / dim ** 0.5) * torch.randn((r1 - r0, dim), generator=g, device=dev)
        return out
    x = sample(n)
    queries = sample(a.queries)
    x0h = x.cpu().numpy() if a.build_in_type else None  # the data in its original order (the incremental builder re-orders)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tl = [time.perf_counter()]
    def prog(l, a1, b1):
        if a1 < 0 or a1 == b1:
            now = time.perf_counter()
            print(f"[build] layer {l} stage {a1} value {b1} +{now - tl[0]:.1f}s", file=sys.stderr, flush=True)
            tl[0] = now
    INT_SCALE = 8192.0
    from surrealdb_b200.hnsw import VT_DTYPE, to_vector_type

    def convert(h, vt):  # in slabs: 1M x 768 f64 temporaries would need ~20 GB of host memory
        scale = INT_SCALE if vt[0] == "I" else 1.0
        out = np.empty(h.shape, VT_DTYPE[vt])
        for r0 in range(0, h.shape[0], 1 << 16):
            out[r0:r0 + (1 << 16)] = to_vector_type(h[r0:r0 + (1 << 16)].astype(np.float64) * scale, vt)
        return out

    def build(xb, vt):
        """builds the graph from xb (device, vector type vt) in metric gm -> (index walked in a.metric, its vectors
        on the device, host layers or None, entry, layer count, mean layer-0 degree, build seconds)"""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if a.builder == "incremental":
            from surrealdb_b200.hnsw_build import build_incremental
            res = build_incremental(ctx, xb, gm, m=a.m, m0=2 * a.m, efc=a.efc, seed=7, growth=a.growth, progress=prog,
                                    settle=not a.no_settle, vector_type=vt, minkowski_order=a.minkowski_order)
            torch.cuda.synchronize()
            build_s = time.perf_counter() - t0
            xb = res["x"]  # re-ordered by level: element ids below are the NEW ids (rows of this tensor)
            layers = [(rp.cpu().numpy().astype(np.uint64), ci.cpu().numpy().astype(np.uint32)) for rp, ci in res["layers_dev"]] if not a.no_cpu else None
            idx = HnswIndex.from_device(ctx, xb, res["layers_dev"], res["entry"], a.metric.upper(),
                                        minkowski_order=a.minkowski_order, vector_type=vt)
            out = (idx, xb, layers, res["entry"], len(res["layers_dev"]), float(res["layers_dev"][0][1].numel()) / n, build_s)
        else:
            layers, entry, levels = build_layers(ctx, xb, n, dim, gm, m=a.m, m0=2 * a.m, seed=7, progress=prog,
                                                 prefix=a.prefix, vector_type=vt, minkowski_order=a.minkowski_order)
            build_s = time.perf_counter() - t0
            idx = HnswIndex(ctx, xb.cpu().numpy(), layers, entry, a.metric.upper(), minkowski_order=a.minkowski_order,
                            vector_type=vt)
            out = (idx, xb, layers, entry, len(layers), float(np.diff(layers[0][0].astype(np.int64)).mean()), build_s)
        print(f"[build] {vt} done {build_s:.1f}s", file=sys.stderr, flush=True)
        return out

    vts = a.vector_type.split(",")
    idx = layers = entry = n_layers = deg0 = build_s = xh = None
    if not a.build_in_type or "F32" in vts:  # the F32 graph (the one every type is walked on without --build-in-type)
        idx, x, layers, entry, n_layers, deg0, build_s = build(x, "F32")
        xh = x.cpu().numpy() if not a.no_cpu or a.vector_type != "F32" else None
        if a.vector_type != "F32" and layers is None:
            layers = [(rp.cpu().numpy().astype(np.uint64), ci.cpu().numpy().astype(np.uint32)) for rp, ci in idx._keep[1]]
    qh0, q_dev0, idx0 = queries.cpu().numpy(), queries, idx
    for vt in vts:  # one JSON line per vector type
        # another vector type: the index holds the data in the type (integers: scaled by INT_SCALE and truncated toward
        # zero) and is walked in that type's arithmetic, on the F32 graph above or (--build-in-type) on a graph built in
        # the type
        esz = {"F64": 8, "F32": 4, "I64": 8, "I32": 4, "I16": 2}[vt]
        qh, queries, idx, vt_build_s, vt_layers, vt_deg0 = qh0, q_dev0, idx0, build_s, n_layers, deg0
        if vt != "F32":
            qh = convert(qh0, vt)
            queries = torch.from_numpy(qh).to(dev)
            if a.build_in_type:  # the graph is built in the type's own arithmetic, from the same data in the type
                idx, _, _, _, vt_layers, vt_deg0, vt_build_s = build(torch.from_numpy(convert(x0h, vt)).to(dev), vt)
            else:
                idx = HnswIndex(ctx, convert(xh, vt), layers, entry, a.metric.upper(), minkowski_order=a.minkowski_order,
                                vector_type=vt)
        print(f"[load] index on device {time.perf_counter() - t0:.1f}s", file=sys.stderr, flush=True)
        idx.search_graph(qh[:256], a.k, a.ef)  # warm-up
        (ids, dist, cnt, ctr), ms_call, wall = dev_time_ms(ctx, lambda: idx.search_graph(qh, a.k, a.ef, counters=True))
        visited, expanded = int(ctr[:, 0].sum()), int(ctr[:, 1].sum())
        byts = visited * (esz * dim + 4.0) + expanded * vt_deg0 * 4.0
        # `value`: queries and results resident in HBM (sdb_hnsw_search_device); the host-buffer call above is the e2e figure
        import ctypes as C
        from surrealdb_b200 import _lib as L
        d_ids = torch.empty((a.queries, a.k), dtype=torch.int64, device=dev)
        d_dist = torch.empty((a.queries, a.k), dtype=torch.float64, device=dev)
        d_cnt = torch.empty((a.queries,), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        def dev_search():
            L.check(L.lib().sdb_hnsw_search_device(idx.h, C.c_void_p(queries.data_ptr()), a.queries, a.k, a.ef, C.c_void_p(d_ids.data_ptr()),
                                                   C.c_void_p(d_dist.data_ptr()), C.c_void_p(d_cnt.data_ptr())))
        dev_search()
        best = None
        for _ in range(3):
            _, m1, w1 = dev_time_ms(ctx, dev_search)
            best = m1 if best is None or m1 < best else best
        ms = best
        same_dev = bool(np.array_equal(d_ids.cpu().numpy()[:, :1].astype(np.uint64), ids[:, :1]))
        # recall@k against the exact kNN in the index's own arithmetic (sdb_hnsw_knn_exact_device)
        from surrealdb_b200.hnsw_build import knn_exact
        nr = min(a.queries, a.recall_queries)
        t_ids, _, t_cnt = knn_exact(idx.h, queries[:nr], a.k)
        t_ids, t_cnt = t_ids.cpu().numpy(), t_cnt.cpu().numpy()
        recall = float(np.mean([len(set(t_ids[i, : t_cnt[i]].tolist()) & set(ids[i, : cnt[i]].tolist())) / a.k
                                for i in range(nr)]))
        peak, src = peaks()
        out = {"bench": "hnsw_search", "metric": f"HNSW KNN queries/sec (M={a.m}, M0={2*a.m}, ef={a.ef}, k={a.k})",
               "value": a.queries / (ms * 1e-3), "unit": "queries/s", "device_ms": ms,
               "e2e": {"value": a.queries / (wall * 1e-3), "unit": "queries/s", "call_wall_ms": wall, "api": "sdb_hnsw_search (pageable host queries and results)",
                       "h2d_bytes": int(a.queries * dim * esz), "d2h_bytes": int(a.queries * a.k * 16 + a.queries * 20)},
               "device_results_equal_host_call": same_dev,
               "recall_at_k": recall, "recall_queries": nr, "build_s": vt_build_s, "config": {"rows": n, "dim": dim, "queries": a.queries, "metric": a.metric.lower(), "graph_metric": gm.lower(),
                                                  "vector_type": vt, "graph_vector_type": vt if a.build_in_type else "F32", **({"int_scale": INT_SCALE, "data_to_int": f"x * {INT_SCALE:g}, truncated toward zero"} if vt[0] == "I" else {}),
                                                  **({"minkowski_order": a.minkowski_order} if a.metric.upper() == "MINKOWSKI" else {}), "data": f"4096 unit-norm centroids + gaussian noise of total norm {a.sigma}",
                                                  "graph": ("GPU batched true insertion (hnsw_build.build_incremental): walk kernel as insertion search (efc=%d), Heuristic::select, bidirectional linking, re-selection of over-full nodes; batches grow by %.2fx" % (a.efc, a.growth)) if a.builder == "incremental" else "GPU batch-built layers (hnsw_build.py): kNN candidates" + (" from id prefixes" if a.prefix else "") + " + Heuristic::select + bidirectional re-selection", "build_s": vt_build_s,
                                                  "recall_truth": "sdb_hnsw_knn_exact_device (exact kNN in the index's arithmetic)",
                                                  "layers": vt_layers, "visited_per_query": visited / a.queries,
                                                  "expanded_per_query": expanded / a.queries},
               "roofline": {"bound": "hbm", "kernel": "hnsw_search_kernel", "achieved": byts / (ms * 1e-3) / 1e9, "peak": peak,
                            "unit": "GB/s", "frac": byts / (ms * 1e-3) / 1e9 / peak, "peak_source": src,
                            "algorithmic_bytes": byts, "traffic": None}}
        if a.metric in ("minkowski", "pearson", "jaccard") or vt != "F32":  # the CPU oracle's walk does not restate these
            out["cpu_baseline"] = None
        elif not a.no_cpu:
            from oracle import pyoracle as O
            if xh is None:
                xh = x.cpu().numpy()
            graph = {"vectors": xh, "layers": layers, "entry_point": entry, "metric": a.metric.lower()}
            threads = os.cpu_count() or 1
            nqc = min(a.queries, 8 * threads)
            t0 = time.perf_counter()
            with ThreadPoolExecutor(threads) as ex:
                res = list(ex.map(lambda i: O.hnsw_search_csr(graph, qh[i], a.k, a.ef), range(nqc)))
            dt = time.perf_counter() - t0
            same = all(list(res[i][0]) == list(ids[i, : cnt[i]]) for i in range(nqc))
            out["cpu_baseline"] = {"value": nqc / dt, "unit": "queries/s", "cores": threads, "kind": "port",
                                   "sample": f"{nqc} of the same queries, same graph, {threads} threads, {dt:.2f}s; "
                                             f"results identical to the GPU walk: {same}"}
        print(json.dumps(out), flush=True)


def bench_graph(a):
    """BASELINE config 5: R-MAT graph, 3-hop ->edge->node multiset expansion (+ one +collect BFS).  Under torchrun
    (WORLD_SIZE > 1) the CSR is row-sharded (1-D source ranges) and every hop is the library's collective:
    all-reduce of the degree array, local expansion into global positions, all-reduce of the level."""
    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200.graph import CsrGraph, CsrGraphShard, collect, device_free, expand, expand_device
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    ctx = Context(local)
    if world > 1:
        import torch.distributed as dist
        if os.environ.get("NCCL_DEBUG", "VERSION").upper() == "VERSION":
            os.environ["NCCL_DEBUG"] = "WARN"
        os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")  # the version banner / warnings must not land on stdout
        dist.init_process_group("nccl", device_id=dev)
        uid = torch.zeros(128, dtype=torch.uint8, device=dev)
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(Context.comm_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        ctx.comm_init_rank(world, rank, bytes(uid.cpu().numpy().tobytes()))
    g = torch.Generator(device=dev).manual_seed(0x5DB00005)
    n_nodes = a.nodes if a.nodes else (1 << a.log2_nodes)
    bits = max(1, int(np.ceil(np.log2(n_nodes))))
    E = a.edges
    t_gen = time.perf_counter()
    keys = []
    chunk = 1 << 27
    for e0 in range(0, E, chunk):  # R-MAT a,b,c,d = .57,.19,.19,.05, generated in chunks (identical on every rank)
        ne = min(chunk, E - e0)
        src = torch.zeros(ne, dtype=torch.int64, device=dev)
        dst = torch.zeros(ne, dtype=torch.int64, device=dev)
        for b in range(bits):
            r = torch.rand(ne, generator=g, device=dev)
            src = (src << 1) | (r >= 0.76).long()
            dst = (dst << 1) | (((r >= 0.57) & (r < 0.76)) | (r >= 0.95)).long()
        if n_nodes != (1 << bits):
            src, dst = src % n_nodes, dst % n_nodes
        keys.append(src * n_nodes + dst)
        del src, dst, r
    key = torch.unique(torch.cat(keys))  # one edge per (src,dst); edge ids in (src,dst) order => KV order
    del keys
    src, dst = key // n_nodes, key % n_nodes
    E = int(key.numel())
    del key
    row_ptr = torch.zeros(n_nodes + 1, dtype=torch.int64, device=dev)
    row_ptr[1:] = torch.cumsum(torch.bincount(src, minlength=n_nodes), 0)
    del src
    # contiguous source ranges with (roughly) equal edge counts per rank
    cuts = [0]
    for r in range(1, world):
        cuts.append(int(torch.searchsorted(row_ptr, torch.tensor(E * r // world, device=dev)).item()))
    cuts.append(n_nodes)
    cuts = [min(max(c, 0), n_nodes) for c in cuts]
    lo, hi = cuts[rank], cuts[rank + 1]
    rp = row_ptr.cpu().numpy().astype(np.uint64)
    e0, e1 = int(rp[lo]), int(rp[hi])
    ci_local = dst[e0:e1].to(torch.int32).cpu().numpy().astype(np.uint32)
    t_gen = time.perf_counter() - t_gen
    if world == 1:
        ci = ci_local
        graph = CsrGraph(ctx, rp, ci)
    else:
        graph = CsrGraphShard.__new__(CsrGraphShard)  # (the full col_idx never exists on the host: hand the slice over)
        import ctypes as C
        from surrealdb_b200 import _lib as L
        graph.ctx, graph.n_rows, graph.row_lo, graph.row_hi, graph.h = ctx, n_nodes, lo, hi, C.c_void_p()
        rps = np.ascontiguousarray(rp[lo:hi + 1] - np.uint64(e0))
        L.check(L.lib().sdb_graph_load_csr_shard(ctx.h, n_nodes, lo, hi, C.c_void_p(rps.ctypes.data),
                                                 C.c_void_p(ci_local.ctypes.data) if ci_local.size else None, C.byref(graph.h)))
    del dst
    torch.cuda.empty_cache()
    deg = np.diff(rp.astype(np.int64))
    rng = np.random.default_rng(11)
    sources = rng.choice(np.nonzero(deg > 0)[0], a.sources, replace=False).astype(np.uint32)

    def tmax(x):
        if world == 1:
            return x
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0])

    d_src = torch.from_numpy(sources.astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    p0, _ = expand_device(ctx, [graph] * a.hops, d_src.data_ptr(), sources.size, a.limit)  # warm-up at full size
    device_free(ctx, p0)
    ms_dev = None
    for _ in range(3):
        if world > 1:
            dist.barrier()
        (pd, nd), m1, _w = dev_time_ms(ctx, lambda: expand_device(ctx, [graph] * a.hops, d_src.data_ptr(), sources.size, a.limit))
        device_free(ctx, pd)
        m1 = tmax(m1)
        ms_dev = m1 if ms_dev is None or m1 < ms_dev else ms_dev
    # end to end with host buffers (result copied back), and the per-hop sizes for the algorithmic byte count
    best = None
    for _ in range(2):
        out_ids, ms, wall = dev_time_ms(ctx, lambda: expand([graph] * a.hops, sources, a.limit))
        wall = tmax(wall)
        best = wall if best is None or wall < best else best
    wall = best
    sizes = [int(sources.size)]
    fr = sources
    for h in range(a.hops - 1):
        fr = expand([graph], fr, a.limit)
        sizes.append(int(fr.size))
    sizes.append(int(out_ids.size))
    byts = sum(16.0 * sizes[h] + 8.0 * sizes[h + 1] for h in range(a.hops))
    collect(graph, sources[:1], 1, a.hops, False)  # warm-up: allocates the per-graph BFS state
    (coll, cms, cwall) = dev_time_ms(ctx, lambda: collect(graph, sources[:a.collect_sources], 1, a.hops, False))
    cms = tmax(cms)
    if rank != 0:
        dist.barrier()
        dist.destroy_process_group()
        return
    peak, srcp = peaks()
    res = {"bench": "graph_expand", "metric": f"{a.hops}-hop ->edge->node multiset expansion, traversed edges/sec",
           "value": sum(sizes[1:]) / (ms_dev * 1e-3), "unit": "edges/s", "device_ms": ms_dev, "n_gpus": world,
           "e2e": {"value": sum(sizes[1:]) / (wall * 1e-3), "unit": "edges/s", "call_wall_ms": wall,
                   "h2d_bytes": int(sources.size * 4), "d2h_bytes": int(out_ids.size * 4)},
           "config": {"nodes": n_nodes, "edges": E, "sources": int(sources.size), "hops": a.hops, "per_source_limit": a.limit, "frontier_sizes": sizes,
                      "graph": "R-MAT (.57,.19,.19,.05), integer ids, adjacency in (src,dst)=edge-id order",
                      "sharding": "none" if world == 1 else f"1-D source ranges, {world} shards with equal edge counts; one all-reduce pair per hop",
                      "generation_s": t_gen,
                      "collect_bfs": {"sources": a.collect_sources, "device_ms": cms, "nodes": int(coll.size)}},
           "roofline": {"bound": "hbm", "kernel": "expand_kernel (+degree/scan)", "achieved": byts / (ms_dev * 1e-3) / 1e9,
                        "peak": peak, "unit": "GB/s", "frac": byts / (ms_dev * 1e-3) / 1e9 / peak, "peak_source": srcp,
                        "algorithmic_bytes": byts, "traffic": None,
                        "note": "device_ms = hops x (degree, scan, expand [+ 2 all-reduces when sharded]) incl. one 8-byte size "
                                "read-back per hop; frontier and result resident in HBM; max over ranks"}}
    if not a.no_cpu and world == 1:
        from oracle import pyoracle as O
        t0 = time.perf_counter()
        fr = sources
        for h in range(a.hops):
            fr = O.graph_hop(rp, ci, fr, a.limit)
        dt = time.perf_counter() - t0
        res["cpu_baseline"] = {"value": sum(sizes[1:]) / dt, "unit": "edges/s", "cores": 1, "kind": "port",
                               "sample": f"same frontier, {a.hops} hops, single thread (the reference expands one "
                                         f"lookup chain per task), {dt:.3f}s; identical output: {bool(np.array_equal(fr, out_ids))}"}
    if a.checksum:
        res["result_checksum"] = {"n": int(out_ids.size), "sum": int(out_ids.astype(np.uint64).sum()),
                                  "xor_fold": int(np.bitwise_xor.reduce(out_ids.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.arange(out_ids.size, dtype=np.uint64))),
                                  "collect_sum": int(coll.astype(np.uint64).sum())}
    print(json.dumps(res), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def bench_stage(a):
    """a14 staging: raw He / Hn KV values -> device arrays.  Algorithmic bytes = value bytes read + decoded bytes
    written; the host->device copy of the blob is inside the timed call (pageable numpy memory), so the number to
    compare with is PCIe, not HBM; the kernel-only time is reported from CUDA events of a second call on a blob
    that is already device-resident ... (not exposed: the ABI takes host blobs), so we report the whole call."""
    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200 import staging as S
    ctx = Context(0)
    n, dim = a.rows, a.dim
    rng = np.random.default_rng(1)
    hdr = b"\x01\x01" + (bytes([dim]) if dim < 251 else b"\xfb" + dim.to_bytes(2, "little"))
    vb = len(hdr) + 4 * dim
    import ctypes as C
    from surrealdb_b200 import _lib as L
    def host_buffer(shape):  # pinned (sdb_pinned_alloc) unless --pageable: what a Rust shim would scan the KV range into
        nbytes = int(np.prod(shape))
        if a.pageable:
            return np.empty(shape, np.uint8)
        ptr = L.lib().sdb_pinned_alloc(nbytes)
        assert ptr, "pinned allocation failed"
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), (nbytes,)).reshape(shape)
    blob = host_buffer((n, vb))
    blob[:, :len(hdr)] = np.frombuffer(hdr, np.uint8)
    payload = rng.standard_normal((n, dim), dtype=np.float32)
    blob[:, len(hdr):] = payload.view(np.uint8).reshape(n, 4 * dim)
    off = (np.arange(n + 1, dtype=np.uint64) * np.uint64(vb))
    out = torch.empty((n, dim), dtype=torch.float32, device="cuda")
    bad = C.c_uint64(0)
    def call():
        L.check(L.lib().sdb_stage_decode_vectors(ctx.h, C.c_void_p(blob.ctypes.data), C.c_void_p(off.ctypes.data), None, n,
                                                 dim, L.DTYPE["F32"], n, C.c_void_p(out.data_ptr()), None, C.byref(bad)))
    call()
    t0 = time.perf_counter(); call(); dt_v = time.perf_counter() - t0
    ok = bool(np.array_equal(out[: min(n, 4096)].cpu().numpy(), payload[: min(n, 4096)])) and bad.value == 0
    # Hn: n nodes x m0 neighbours
    m0 = 2 * a.m
    nb = rng.integers(0, n, (n, m0), dtype=np.uint64)
    node = host_buffer((n, 2 + 8 * m0))
    node[:, 0] = m0 >> 8
    node[:, 1] = m0 & 255
    node[:, 2:] = nb.astype(">u8").view(np.uint8).reshape(n, 8 * m0)
    noff = np.arange(n + 1, dtype=np.uint64) * np.uint64(2 + 8 * m0)
    nid = np.arange(n, dtype=np.uint64)
    rp, ci, nbad = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    def call_n():
        L.check(L.lib().sdb_stage_decode_nodes(ctx.h, C.c_void_p(node.ctypes.data), C.c_void_p(noff.ctypes.data),
                                               C.c_void_p(nid.ctypes.data), n, n, C.byref(rp), C.byref(ci), C.byref(nbad)))
    call_n(); L.lib().sdb_free(rp); L.lib().sdb_free(ci)
    t0 = time.perf_counter(); call_n(); dt_n = time.perf_counter() - t0
    L.lib().sdb_free(rp); L.lib().sdb_free(ci)
    res = {"metric": "staging_values_per_s", "value": n / dt_v, "unit": "He values/s", "rows": n, "dim": dim,
           "he_bytes": int(blob.nbytes), "he_seconds": dt_v, "he_gb_per_s_in": blob.nbytes / dt_v / 1e9, "he_correct": ok,
           "hn_values_per_s": n / dt_n, "hn_bytes": int(node.nbytes), "hn_seconds": dt_n,
           "hn_gb_per_s_in": node.nbytes / dt_n / 1e9, "hn_edges": int(n * m0),
           "host_memory": "pageable" if a.pageable else "pinned",
           "note": "whole C-ABI call (H2D copy of the raw values + decode kernel [+ D2H of the CSR for Hn]); PCIe-bound"}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("which", choices=["hnsw", "graph", "stage"])
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--ef", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--m", type=int, default=16)
    metrics = ["euclidean", "cosine", "manhattan", "chebyshev", "hamming", "minkowski", "pearson", "jaccard"]
    ap.add_argument("--metric", default="euclidean", choices=metrics, help="metric of the walk (and of the recall)")
    ap.add_argument("--graph-metric", default=None, choices=metrics,
                    help="metric the GPU builder links the graph with (default: --metric)")
    ap.add_argument("--minkowski-order", type=float, default=3.0)
    ap.add_argument("--vector-type", default="F32",
                    help="element type(s) of the index, F64 F32 I64 I32 I16, comma-separated (the graph is built once, in "
                         "F32, from the same data, unless --build-in-type; one result line per type)")
    ap.add_argument("--build-in-type", action="store_true",
                    help="build every --vector-type index's graph in that type's own arithmetic, from the data in the type")
    ap.add_argument("--recall-queries", type=int, default=1000, help="queries of the recall@k against the exact kNN")
    ap.add_argument("--sigma", type=float, default=0.15)
    ap.add_argument("--prefix", action="store_true", help="insertion-order (prefix) candidate sets in the batch builder")
    ap.add_argument("--builder", default="batch", choices=["batch", "incremental"])
    ap.add_argument("--efc", type=int, default=150)
    ap.add_argument("--growth", type=float, default=0.25)
    ap.add_argument("--no-settle", action="store_true", help="incremental builder without the second pass per batch")
    ap.add_argument("--log2-nodes", type=int, default=24)
    ap.add_argument("--edges", type=int, default=160_000_000)
    ap.add_argument("--nodes", type=int, default=0, help="node count (not a power of two: R-MAT ids are folded mod nodes)")
    ap.add_argument("--checksum", action="store_true", help="print order-sensitive checksums of the result (1 vs N GPUs)")
    ap.add_argument("--sources", type=int, default=1024)
    ap.add_argument("--hops", type=int, default=3)
    ap.add_argument("--collect-sources", type=int, default=1, help="start nodes of the +collect BFS")
    ap.add_argument("--limit", type=int, default=32, help="GraphEdgeScan per-source limit (0 = none)")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--pageable", action="store_true", help="stage: keep the value blobs in pageable host memory")
    a = ap.parse_args()
    {"hnsw": bench_hnsw, "graph": bench_graph, "stage": bench_stage}[a.which](a)
