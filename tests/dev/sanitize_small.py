"""Small end-to-end exercise of every kernel family, meant to run under compute-sanitizer (memcheck / racecheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
from oracle import pyoracle as O
from surrealdb_b200 import Context, VectorColumn, HnswIndex
from surrealdb_b200.graph import CsrGraph, expand, collect
from surrealdb_b200.synthetic import gen_f32

ctx = Context(0)
n, dim, nq, k = 3000, 96, 40, 5
corpus = gen_f32(1, 0, n * dim).reshape(n, dim)
corpus[17] = 0.0
queries = gen_f32(2, 0, nq * dim).reshape(nq, dim).astype(np.float64)
for metric in ("COSINE", "EUCLIDEAN"):
    for screen in ("SIMT_F32", "TC_BF16", "TC_INT8", "NONE_EXACT"):
        col = VectorColumn(ctx, dim, metric, "F32", capacity=n)
        col.append(corpus); col.finalize(); col.set_screen(screen)
        nqq = 3 if screen == "NONE_EXACT" else nq
        rows, dist, cnt = col.knn(queries[:nqq], k)
        for q in range(0, nqq, 7):
            r, d = O.knn_topk(corpus, queries[q], metric.lower(), k)
            assert list(rows[q]) == list(r) and dist[q].tobytes() == d.tobytes(), (metric, screen, q)
        print("knn ok", metric, screen, col.stats()["n_fallback"], flush=True)
        col.close()
data = gen_f32(3, 0, 600 * 16).reshape(600, 16) * 20
h = O.Hnsw(16, "euclidean", m=6, efc=40, seed=5)
for v in data:
    h.insert(v)
g = h.export()
idx = HnswIndex(ctx, g["vectors"], g["layers"], g["entry_point"], "EUCLIDEAN")
qs = gen_f32(4, 0, 20 * 16).reshape(20, 16) * 20
ids, dist, cnt, ctr = idx.search_graph(qs, 5, 24, counters=True)
for q in range(20):
    oi, od, oc = O.hnsw_search_csr(g, qs[q], 5, 24)
    assert list(ids[q, :cnt[q]]) == list(oi)
print("hnsw ok", flush=True)
rp = np.array([0, 3, 3, 5, 9], np.uint64)
ci = np.array([1, 2, 2, 0, 1, 3, 0, 1, 2], np.uint32)
gr = CsrGraph(ctx, rp, ci)
assert list(expand([gr, gr], [0, 3, 0])) == list(O.graph_hop(rp, ci, O.graph_hop(rp, ci, [0, 3, 0])))
assert list(collect(gr, [0], 1, 0, False)) == list(O.graph_collect(rp, ci, [0], 1, 0, False))
print("graph ok", flush=True)
# ---- kernels added later in round 1: other metrics (exact kernel), projection, filtered walk, staging decoders
from oracle import kvformats as K
from surrealdb_b200 import staging as S
import torch
for metric in ("MANHATTAN", "CHEBYSHEV", "HAMMING", "PEARSON"):
    col = VectorColumn(ctx, dim, metric, "F32", capacity=n)
    col.append(corpus); col.finalize()
    rows, dist, cnt = col.knn(queries[:2], k)
    r, d = O.knn_topk(corpus, queries[0], metric.lower(), k)
    assert list(rows[0]) == list(r) and dist[0].tobytes() == d.tobytes(), metric
    col.close()
col = VectorColumn(ctx, dim, "COSINE", "F32", capacity=n)
col.append(corpus); col.finalize()
for fn in ("SIMILARITY_COSINE", "DOT", "MAGNITUDE", "PEARSON"):
    col.project(fn, queries[0])
big = VectorColumn(ctx, dim, "COSINE", "F32", capacity=n)
big.append(corpus); big.finalize(); big.set_screen("TC_INT8")
qq = np.tile(queries, (15, 1))[:600]                      # batch >= 512: the R=4 schedule + radix-select compaction
rows, dist, cnt = big.knn(qq, k)
r, d = O.knn_topk(corpus, qq[599], "cosine", k)
assert list(rows[599]) == list(r)
print("metrics/project/large-batch ok", flush=True)
truthy = (np.arange(600) % 3 == 0).astype(np.uint8)
ids, dist, cnt, ctr = idx.search_graph(qs, 5, 24, counters=True, truthy=truthy)
for q in range(20):
    oi, od, oc = O.hnsw_search_csr(g, qs[q], 5, 24, truthy=truthy)
    assert list(ids[q, :cnt[q]]) == list(oi)
he = [(e, K.ser_vector("F32", g["vectors"][e])) for e in range(600)]
hn = [[(e, K.node_to_val(ci_[rp_[e]:rp_[e + 1]])) for e in range(600) if rp_[e + 1] > rp_[e]] for rp_, ci_ in g["layers"]]
state = K.hnsw_state(int(g["entry_point"]), 600, (1, 0), tuple((1, 0) for _ in g["layers"][1:]))
idx2 = HnswIndex.from_kv(ctx, 16, state, he, hn, "EUCLIDEAN")
ids2, dist2, cnt2 = idx2.search_graph(qs, 5, 24)
ids1, dist1, cnt1 = idx.search_graph(qs, 5, 24)
assert ids1.tobytes() == ids2.tobytes() and idx2.n_bad == 0
out = torch.zeros((4, 7), dtype=torch.float64, device="cuda")
items = [(i, K.ser_vector(v, np.arange(7) + i)) for i, v in enumerate(("F64", "I64", "I32", "I16"))]
assert S.decode_vectors(ctx, items, 7, out.data_ptr(), 4, "F64") == 0
torch.cuda.synchronize()
assert out.cpu().numpy()[3].tolist() == [3, 4, 5, 6, 7, 8, 9]
print("filtered walk / staging ok", flush=True)
# every handle and the context are closed, so that --leak-check full sees what the library failed to release
for handle in (col, big, idx, idx2, gr):
    handle.close()
ctx.close()
print("closed", flush=True)
