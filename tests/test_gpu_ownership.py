"""Every device and pinned buffer the library allocates is released again.  Each case reads the process-wide count of
live buffers (sdb_debug_live_allocations), does its work, closes every handle it made and expects count and bytes back
at the start.  Buffers a context keeps growing (its pinned staging buffer) belong to the context, so the cases measure
around the context's whole life.  Refused calls must leave nothing behind either."""
import contextlib
import ctypes as C
import gc

import numpy as np
import pytest

from oracle import kvformats as K
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu


def live():
    from surrealdb_b200 import _lib as L
    n, b = C.c_uint64(), C.c_uint64()
    L.lib().sdb_debug_live_allocations(C.byref(n), C.byref(b))
    return n.value, b.value


@contextlib.contextmanager
def no_leaks():
    gc.collect()
    before = live()
    yield before
    gc.collect()
    assert live() == before


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def column(ctx, corpus, metric, screen=None):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, corpus.shape[1], metric, "F32" if corpus.dtype == np.float32 else "F64",
                       capacity=corpus.shape[0])
    col.append(corpus)
    col.finalize()
    if screen:
        col.set_screen(screen)
    return col


def check(col, corpus, queries, metric, k, skip=None):
    rows, dist, cnt = col.knn(queries, k)
    for q in range(queries.shape[0]):
        r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=skip)
        assert list(rows[q, : cnt[q]]) == list(r) and dist[q, : cnt[q]].tobytes() == d.tobytes(), q


def ring(n, deg=4):
    """one CSR layer: element i links to i+1 .. i+deg (mod n)"""
    rp = (np.arange(n + 1) * deg).astype(np.uint64)
    ci = ((np.arange(n)[:, None] + np.arange(1, deg + 1)[None, :]) % n).astype(np.uint32).ravel()
    return rp, ci


def test_context_and_corpus_release_every_buffer():
    import torch
    from surrealdb_b200 import Context
    rng = np.random.default_rng(31)
    with no_leaks():
        ctx = Context(0)
        dim, n = 64, 3000
        for metric in ("COSINE", "EUCLIDEAN"):  # COSINE: int8 and bf16 screen copies; EUCLIDEAN: bf16 only
            corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
            corpus[5] = 0.0                          # a special row: ranked by the exact kernel on every query
            queries = rng.uniform(-1, 1, (6, dim))
            queries[2] = 0.0                         # a zero query: the exact path and the fallback buffers
            col = column(ctx, corpus, metric)
            check(col, corpus, queries, metric, 10)
            # host entry points on both ticket parities (two batches in flight), then the device entry points
            q = np.ascontiguousarray(queries)
            outs = [(np.zeros((6, 10), np.uint64), np.zeros((6, 10)), np.zeros(6, np.uint32)) for _ in range(2)]
            tickets = [col.submit_host(q.ctypes.data, 6, 10, *[a.ctypes.data for a in o]) for o in outs]
            for t in tickets:
                col.wait(t)
            want_rows, want_dist, _ = col.knn(queries, 10)
            for o in outs:
                assert o[0].tobytes() == want_rows.tobytes() and o[1].tobytes() == want_dist.tobytes()
            dq = dev(q)
            dr = torch.zeros((6, 10), dtype=torch.int64, device="cuda")
            dd = torch.zeros((6, 10), dtype=torch.float64, device="cuda")
            dc = torch.zeros(6, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            col.knn_device(dq.data_ptr(), 6, 10, 0, dr.data_ptr(), dd.data_ptr(), dc.data_ptr())
            tickets = [col.submit_device(dq.data_ptr(), 6, 10, 0, dr.data_ptr(), dd.data_ptr(), dc.data_ptr())
                       for _ in range(2)]
            for t in tickets:
                col.wait(t)
            assert dr.cpu().numpy().astype(np.uint64).tobytes() == want_rows.tobytes()
            got = col.project("EUCLIDEAN", queries[0])
            assert got[7] == O.f64_metric("euclidean", corpus[7].astype(np.float64), queries[0])
            skip = np.zeros(n, np.uint8)
            skip[::3] = 1
            col.set_skip(skip)
            col.remove([1, 2, 4])
            col.finalize()
            skip[[1, 2, 4]] = 1
            check(col, corpus, queries, metric, 10, skip=skip)
            col.set_skip(None)
            col.close()
        corpus = rng.uniform(-20, 20, (2000, 24))    # an F64 corpus
        col = column(ctx, corpus, "COSINE")
        check(col, corpus, rng.uniform(-20, 20, (3, 24)), "COSINE", 7)
        col.close()
        ctx.close()


def test_the_repair_ladder_releases_its_buffers():
    # near-duplicate rows (test_gpu_knn.py's adversarial cluster): the proof fails for some queries, which climb the
    # remaining rungs as a repair batch of their own
    from surrealdb_b200 import Context
    rng = np.random.default_rng(8)
    center = rng.uniform(-1, 1, 64).astype(np.float32)
    corpus = (center[None, :] + rng.normal(0, 1e-6, (30000, 64))).astype(np.float32)
    queries = (center[None, :] + rng.normal(0, 1e-3, (12, 64))).astype(np.float64)
    with no_leaks():
        ctx = Context(0)
        repaired = 0
        for screen in ("SIMT_F32", "TC_BF16", "TC_INT8"):
            col = column(ctx, corpus, "COSINE", screen)
            check(col, corpus, queries, "COSINE", 10)
            st = col.stats()
            repaired += st["n_repaired"] + st["n_fallback"]
            col.close()
        assert repaired > 0
        ctx.close()


def test_refused_screen_batch_leaves_the_corpus_usable():
    # a candidate list of 2^30 slots per query needs about 1 TB: the allocation is refused before any device work, the
    # batch scratch is left empty, and the next ordinary batch allocates it again
    from surrealdb_b200 import Context, _lib as L
    rng = np.random.default_rng(5)
    corpus = rng.uniform(-1, 1, (5000, 32)).astype(np.float32)
    queries = rng.uniform(-1, 1, (4, 32))
    with no_leaks():
        ctx = Context(0)
        col = column(ctx, corpus, "COSINE")
        check(col, corpus, queries, "COSINE", 10)
        q = np.ascontiguousarray(queries[:1])
        rc = L.lib().sdb_debug_screen_batch(col.h, C.c_void_p(q.ctypes.data), 1, 10, L.SCREEN["TC_INT8"], 1, 1 << 30, 0,
                                            *([None] * 8))
        assert rc == L.SDB_ECUDA, rc
        check(col, corpus, queries, "COSINE", 10)
        col.close()
        ctx.close()


@pytest.mark.parametrize("metric", ["COSINE", "PEARSON", "JACCARD"])
@pytest.mark.parametrize("vt", ["F32", "I32"])
def test_hnsw_owned_load_and_searches(metric, vt):
    from surrealdb_b200 import Context
    from surrealdb_b200.hnsw import HnswIndex
    from surrealdb_b200.hnsw_build import knn_exact, select
    rng = np.random.default_rng(3)
    n, dim = 800, 12
    data = rng.integers(0, 6, (n, dim)) if metric == "JACCARD" else rng.uniform(-20, 20, (n, dim))
    data = np.trunc(data).astype(np.int32) if vt == "I32" else data.astype(np.float32)
    with no_leaks():
        ctx = Context(0)
        idx = HnswIndex(ctx, data, [ring(n, 8), ring(n, 2)], 0, metric, vector_type=vt)
        q = data[:10]
        ids, dist, cnt = idx.search_graph(q, 5, 32)
        assert cnt.min() > 0
        idx.search_graph(q, 5, 32, truthy=(np.arange(n) % 2).astype(np.uint8))
        idx.search_graph(q, 5, 32, all_docs_pending=(np.arange(n) % 3 == 0).astype(np.uint8))
        idx._typed_distances(data[0], data[:50])
        e_ids, e_dist, e_cnt = knn_exact(idx.h, dev(q), 16)
        knn_exact(idx.h, dev(q), 16, dev(np.arange(0, n, 2, dtype=np.int32)))
        select(idx.h, e_ids, e_cnt, 6, 1, row0=0)
        import torch
        torch.cuda.synchronize()
        idx.close()
        ctx.close()


def test_hnsw_borrowed_handle_owns_only_its_layer_tables():
    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200.hnsw_build import load_device, set_layers
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(4)
    n, dim = 600, 16
    x = dev(rng.uniform(-1, 1, (n, dim)).astype(np.float32))
    lay = [tuple(dev(a.astype(np.int64 if a.dtype == np.uint64 else np.int32)) for a in ring(n, d)) for d in (6, 2)]
    torch.cuda.synchronize()
    with no_leaks():
        ctx = Context(0)
        base = live()
        h = load_device(ctx, x, lay, 0, "EUCLIDEAN")  # EUCLIDEAN carries no per-vector state
        # the caller's vectors and CSR arrays are not the library's: only the two device tables of layer pointers are
        assert live() == (base[0] + 2, base[1] + 2 * 8 * len(lay))
        set_layers(h, lay[:1], 0)
        assert live() == (base[0] + 2, base[1] + 2 * 8)
        L.lib().sdb_hnsw_destroy(h)
        ctx.close()


def test_hnsw_staged_loads():
    from surrealdb_b200 import Context
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(11)
    dim, n = 16, 400
    data = rng.uniform(-20, 20, (n, dim)).astype(np.float32)
    rp, ci = ring(n, 6)
    he = [(e, K.ser_vector("F32", data[e])) for e in range(n)]
    hn = [[(e, K.node_to_val(ci[rp[e]:rp[e + 1]])) for e in range(n)]]
    state = K.hnsw_state(0, n, (n, 0), ())
    with no_leaks():
        ctx = Context(0)
        idx = HnswIndex.from_kv(ctx, dim, state, he, hn, "COSINE")
        assert idx.n_bad == 0
        idx.search_graph(data[:4], 5, 20)
        idx.close()
        # bad values: a truncated He value and a node value naming an element outside the index
        bad_he = he[:7] + [(7, he[7][1][:-3])] + he[8:]
        bad_hn = [hn[0][:9] + [(9, K.node_to_val([1, 2, n + 5]))] + hn[0][10:]]
        idx = HnswIndex.from_kv(ctx, dim, state, bad_he, bad_hn, "COSINE")
        assert idx.n_bad > 0
        idx.close()
        ctx.close()


def test_refused_hnsw_load_releases_the_half_built_handle():
    from surrealdb_b200 import Context, _lib as L
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(2)
    n = 300
    data = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
    rp, ci = ring(n, 4)
    ci[17] = n + 3  # a neighbour id out of range: refused after the arrays were allocated and copied
    with no_leaks():
        ctx = Context(0)
        with pytest.raises(L.SdbError, match="SDB_EINVAL"):
            HnswIndex(ctx, data, [ring(n, 4), (rp, ci)], 0, "COSINE")
        ctx.close()


def test_graph_and_staging_release_every_buffer():
    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200 import graph as G
    from surrealdb_b200 import staging as S
    rng = np.random.default_rng(9)
    n = 3000
    rp, ci = ring(n, 5)
    with no_leaks():
        ctx = Context(0)
        g = G.CsrGraph(ctx, rp, ci)
        frontier = np.array([0, 5, 9], np.uint32)
        out = G.expand([g, g], frontier)
        assert out.size == 3 * 25
        big = G.expand([g, g, g], np.arange(n, dtype=np.uint32))  # > 1 MB: through the context's pinned staging buffer
        assert big.size == n * 125
        col = G.collect(g, [0], 1, 3)
        assert col.size > 0
        d_f = dev(frontier)
        torch.cuda.synchronize()
        ptr, cnt = G.expand_device(ctx, [g], d_f.data_ptr(), 3)
        assert cnt == 15 and ptr
        G.device_free(ctx, ptr)
        g.close()
        dim = 8
        items = [(e, K.ser_vector("F32", rng.uniform(-1, 1, dim).astype(np.float32))) for e in range(50)]
        items.append((50, items[0][1][:-2]))  # a truncated value
        out_v = torch.zeros((60, dim), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        assert S.decode_vectors(ctx, items, dim, out_v.data_ptr(), 60, "F32") >= 1
        nodes = [(e, K.node_to_val([int(x) for x in rng.integers(0, 40, 5)])) for e in range(40)]
        nodes.append((45, K.node_to_val([1])))  # node id out of range
        row_ptr, col_idx, bad = S.decode_nodes(ctx, nodes, 40)
        assert bad >= 1 and row_ptr.size == 41
        ctx.close()
