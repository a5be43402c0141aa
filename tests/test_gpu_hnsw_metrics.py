"""The HNSW walk in the metrics beyond cosine / euclidean (MANHATTAN, CHEBYSHEV, HAMMING, MINKOWSKI, PEARSON,
JACCARD), through the C ABI, against the oracle's restatement of the reference on the same graphs: the typed F32
distances of sdb_hnsw_distance, and the ids, f64 distances and visit counters of the plain, filtered and pending walks,
for every loader.  MANHATTAN, CHEBYSHEV and HAMMING are checked against the CPU oracle (oracle/), which builds and walks
graphs in them; MINKOWSKI, PEARSON and JACCARD against tests/hnsw_metric_ref.py, walking graphs the oracle links in
euclidean (manhattan for Jaccard's integer data)."""
import math

import numpy as np
import pytest

import hnsw_metric_ref as R
from oracle import kvformats as K
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

NEW = ["manhattan", "chebyshev", "hamming", "minkowski", "pearson", "jaccard"]
IN_ORACLE = ("manhattan", "chebyshev", "hamming")
GRAPH_METRIC = {"minkowski": "euclidean", "pearson": "euclidean", "jaccard": "manhattan"}


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def gen(rng, metric, shape):
    """the reference's test generator (idx/trees/knn.rs:630-641): integers in [0, 2) for Hamming, in [0, dim/2) for
    Jaccard, uniform(-20, 20) otherwise"""
    dim = shape[-1]
    if metric == "hamming":
        return rng.integers(0, 2, shape).astype(np.float32)
    if metric == "jaccard":
        return rng.integers(0, max(dim // 2, 1), shape).astype(np.float32)
    return rng.uniform(-20, 20, shape).astype(np.float32)


def build(data, metric, m=8, efc=60, seed=1):
    """an oracle-built graph (Hnsw::insert restated) for walking in `metric`"""
    h = O.Hnsw(data.shape[1], GRAPH_METRIC.get(metric, metric), m=m, efc=efc, seed=seed)
    for v in data:
        h.insert(v)
    assert h.check_props()
    return h.export()


def ref_distance(metric, a, b, order=3.0):
    return O.vec_distance_f32(metric, a, b) if metric in IN_ORACLE else R.distance(metric, a, b, order)


def ref_search(g, q, k, ef, metric, order=3.0, **kw):
    if metric in IN_ORACLE:
        return O.hnsw_search_csr(g, q, k, ef, **kw)
    return R.search_csr(g, q, k, ef, metric, order=order, **kw)


def same(metric, got, want):
    """bit-equal (NaN: NaN-ness only, the payload of a computed NaN is the hardware's); Minkowski within 1e-12"""
    if math.isnan(want):
        return math.isnan(got)
    if metric == "minkowski":
        return math.isclose(got, want, rel_tol=1e-12, abs_tol=0.0) or got == want
    return np.float64(got).tobytes() == np.float64(want).tobytes()


def check_walk(metric, idx, g, queries, k, ef, order=3.0, **kw):
    ids, dist, cnt, ctr = idx.search_graph(queries, k, ef, counters=True, **kw)
    for q in range(queries.shape[0]):
        oi, od, oc = ref_search(g, queries[q], k, ef, metric, order, **kw)
        assert cnt[q] == oi.size, (metric, k, ef, q)
        assert list(ids[q, : cnt[q]]) == list(oi), (metric, k, ef, q)
        assert (int(ctr[q, 0]), int(ctr[q, 1])) == oc, (metric, k, ef, q)
        if metric == "minkowski":
            assert all(same(metric, a, b) for a, b in zip(dist[q, : cnt[q]], od)), (k, ef, q)
        else:
            assert dist[q, : cnt[q]].tobytes() == od.tobytes(), (metric, k, ef, q)


@pytest.mark.parametrize("metric", NEW)
def test_hnsw_distance_parity(ctx, metric):
    # sdb_hnsw_distance = Distance::calculate(&query, &vector) (hnsw/index.rs:407), the pending-log order
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(len(metric))
    nan = np.float32("nan")
    orders = (2.0, 3.0) if metric == "minkowski" else (3.0,)
    for dim in (1, 3, 7, 8, 20, 129, 768, 1536):
        vecs = gen(rng, metric, (40, dim))
        vecs[1] = 0.0
        vecs[2] = -0.0
        vecs[3] = 5.0                                   # constant rows
        vecs[4, :: 3] = nan
        vecs[5, : (dim + 1) // 2] = -0.0
        vecs[6] = np.array([0x7FC00001], np.uint32).view(np.float32)[0]   # a NaN payload
        queries = [gen(rng, metric, (dim,)), np.zeros(dim, np.float32), np.full(dim, -0.0, np.float32), vecs[7].copy()]
        q_nan = gen(rng, metric, (dim,))
        q_nan[0] = nan
        queries.append(q_nan)
        layers = [(np.zeros(41, np.uint64), np.zeros(0, np.uint32))]
        for p in orders:
            idx = HnswIndex(ctx, vecs, layers, 0, metric, minkowski_order=p)
            for q in queries:
                got = idx._typed_distances(q, vecs)
                for r in range(vecs.shape[0]):
                    want = ref_distance(metric, q, vecs[r], p)
                    assert same(metric, got[r], want), (metric, dim, p, r, got[r], want)
            idx.close()


@pytest.mark.parametrize("metric", NEW)
@pytest.mark.parametrize("dim", [7, 20, 129])
def test_walk_parity_random_graphs(ctx, metric, dim):
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(dim * 7 + len(metric))
    data = gen(rng, metric, (900, dim))
    queries = gen(rng, metric, (40, dim))
    g = build(data, metric)
    for order in ((2.0, 3.0) if metric == "minkowski" else (3.0,)):
        idx = HnswIndex(ctx, g["vectors"], g["layers"], g["entry_point"], metric, minkowski_order=order)
        for k, ef in ((10, 10), (10, 40), (1, 1), (25, 64)):
            check_walk(metric, idx, g, queries, k, ef, order=order)
        idx.close()


@pytest.mark.parametrize("metric", ["manhattan", "pearson", "jaccard"])
def test_filtered_and_pending_walk_parity(ctx, metric):
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(91)
    dim, n = 24, 1500
    data = gen(rng, metric, (n, dim))
    g = build(data, metric)
    idx = HnswIndex(ctx, g["vectors"], g["layers"], g["entry_point"], metric)
    queries = gen(rng, metric, (32, dim))
    for sel in (1.0, 0.5, 0.25):
        truthy = (rng.random(n) < sel).astype(np.uint8)
        for k, ef in ((10, 40), (3, 8)):
            try:
                check_walk(metric, idx, g, queries, k, ef, truthy=truthy)
            except Exception as e:  # documented: a filter too selective for the on-chip window -> caller's CPU path
                assert "SDB_EOVERFLOW" in str(e) and sel < 1.0, (sel, k, ef, str(e))
    pending = (rng.random(n) < 0.1).astype(np.uint8)
    check_walk(metric, idx, g, queries, 10, 40, all_docs_pending=pending)
    # HnswIndex.knn_search with a pending log: pending vectors ranked with calculate(&query, &vector)
    q = queries[0]
    ids0, _, _ = idx.search_graph(q, 30, 64)
    near = [int(e) for e in ids0[0][:30]]
    moved = {e: gen(rng, metric, (dim,)) for e in near[::2]}
    for e, v in moved.items():
        idx.add_pending(e, [data[e]], [v])
    idx.add_pending("person:new", [], [q.copy()])
    k, ef = 10, 40
    got = idx.knn_search(q, k, ef)
    entries = set()
    key = HnswIndex._vid_key

    def offer(d, vid):
        if len(entries) >= k and d > max(e[0] for e in entries):
            return
        entries.add((d, key(vid), vid))
        while len(entries) > k:
            entries.remove(max(entries, key=lambda e: (e[0], e[1])))
    for vid, v in list(moved.items()) + [("person:new", q)]:
        offer(ref_distance(metric, q, v), vid)
    mask = np.zeros(n, np.uint8)
    mask[list(moved)] = 1
    oi, od, _ = ref_search(g, q, k, ef, metric, all_docs_pending=mask)
    for e, d in zip(oi, od):
        offer(float(d), int(e))
    want = [(vid, d) for d, _, vid in sorted(entries, key=lambda e: (e[0], e[1]))]
    assert got == want, (metric, got, want)


@pytest.mark.parametrize("metric", ["pearson", "jaccard"])
def test_device_and_staged_loaders_build_the_element_state(ctx, metric):
    import torch
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(17)
    dim, n = 20, 700
    data = gen(rng, metric, (n, dim))
    g = build(data, metric)
    queries = gen(rng, metric, (24, dim))
    x = torch.from_numpy(g["vectors"]).cuda()
    layers_dev = [(torch.from_numpy(rp.astype(np.int64)).cuda(), torch.from_numpy(ci.astype(np.int32)).cuda())
                  for rp, ci in g["layers"]]
    dev = HnswIndex.from_device(ctx, x, layers_dev, g["entry_point"], metric)
    he = [(e, K.ser_vector("F32", g["vectors"][e])) for e in range(n)]
    hn = [[(e, K.node_to_val(ci[rp[e]:rp[e + 1]])) for e in range(n) if rp[e + 1] > rp[e]] for rp, ci in g["layers"]]
    state = K.hnsw_state(int(g["entry_point"]), n, (n, 0), tuple((1, 0) for _ in g["layers"][1:]))
    staged = HnswIndex.from_kv(ctx, dim, state, he, hn, metric)
    assert staged.n_bad == 0
    for idx in (dev, staged):
        for k, ef in ((10, 40), (4, 4)):
            check_walk(metric, idx, g, queries, k, ef)


def test_minkowski_order_setter(ctx):
    from surrealdb_b200 import SdbError
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.hnsw import HnswIndex
    data = np.arange(12, dtype=np.float32).reshape(4, 3)
    layers = [(np.zeros(5, np.uint64), np.zeros(0, np.uint32))]
    idx = HnswIndex(ctx, data, layers, 0, "minkowski")
    assert idx._typed_distances([1, 2, 3], [[2, 3, 4]])[0] == 1.4422495703074083   # default order 3
    assert L.lib().sdb_hnsw_set_minkowski_order(idx.h, float("nan")) == L.SDB_EINVAL
    assert idx._typed_distances([1, 2, 3], [[2, 3, 4]])[0] == 1.4422495703074083   # unchanged
    L.check(L.lib().sdb_hnsw_set_minkowski_order(idx.h, 1.0))
    # CUDA's pow is within an ulp or two of the platform libm's (DESIGN section 8): 3.0 up to 1e-12 relative
    assert math.isclose(idx._typed_distances([1, 2, 3], [[2, 3, 4]])[0], 3.0, rel_tol=1e-12)
    with pytest.raises(SdbError, match="SDB_EINVAL"):
        HnswIndex(ctx, data, layers, 0, "minkowski", minkowski_order=float("nan"))
