"""HNSW indexes of the vector types F64, I64, I32 and I16 through the C ABI, against tests/hnsw_types_ref.py's
restatement of the reference's typed arithmetic (idx/trees/vector.rs:206-451) on the same graphs: the distances of
sdb_hnsw_distance, the ids, f64 distances and visit counters of the plain, filtered and pending walks, the typed staged
loader, and the loaders' refusals.  Graphs are linked by the CPU oracle on the f32 copy of the data and walked in the
type's own metric."""
import ctypes as C
import math

import numpy as np
import pytest

import hnsw_types_ref as R
from oracle import kvformats as K
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

TYPES = ["F64", "I64", "I32", "I16"]
METRICS = ["chebyshev", "cosine", "euclidean", "hamming", "jaccard", "manhattan", "minkowski", "pearson"]
GRAPH_METRIC = {"cosine": "cosine", "hamming": "hamming", "jaccard": "manhattan"}


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def gen(rng, metric, vt, shape):
    """the reference's test generator (idx/trees/knn.rs:630-641) in the type: integers in [0, 2) for Hamming, in
    [0, dim/2) for Jaccard, uniform(-20, 20) otherwise (truncated toward zero for the integer types)"""
    dim = shape[-1]
    if metric == "hamming":
        v = rng.integers(0, 2, shape).astype(np.float64)
    elif metric == "jaccard":
        v = rng.integers(0, max(dim // 2, 1), shape).astype(np.float64)
    else:
        v = rng.uniform(-20, 20, shape)
    return v if vt == "F64" else np.trunc(v).astype(R.DTYPES[vt])


def same(metric, got, want):
    """bit-equal (NaN: NaN-ness only); Minkowski within 1e-12 relative"""
    if math.isnan(want):
        return math.isnan(got)
    if metric == "minkowski":
        return math.isclose(got, want, rel_tol=1e-12, abs_tol=0.0) or got == want
    return np.float64(got).tobytes() == np.float64(want).tobytes()


def wrap_rows(rng, vt, vecs):
    """rows whose arithmetic wraps in the type (I16 near +-30000: the dot, the Manhattan difference; I32 squares past
    2^31; I64 the minimum, whose abs stays negative) and, for F64, NaN / +-0 / constant / non-f32 rows"""
    dim = vecs.shape[1]
    if vt == "F64":
        vecs[1] = 0.0
        vecs[2] = -0.0
        vecs[3] = 5.0
        vecs[4, ::3] = np.nan
        vecs[5, : (dim + 1) // 2] = -0.0
        vecs[6] = 0.1
    elif vt == "I16":
        vecs[1] = rng.choice([-30000, 30000], dim) + rng.integers(-50, 50, dim)
        vecs[2] = 30000
        vecs[3] = -30000
        vecs[4] = 7
    elif vt == "I32":
        vecs[1] = rng.choice([-50000, 50000], dim)
        vecs[2] = 2 ** 31 - 1
        vecs[3] = 7
    else:
        vecs[1] = np.iinfo(np.int64).min
        vecs[2] = rng.integers(-2 ** 40, 2 ** 40, dim)
        vecs[3] = 7
        vecs[4] = 2 ** 53 + 1
    return vecs


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vt", TYPES)
def test_hnsw_distance_parity(ctx, vt, metric):
    # sdb_hnsw_distance = Distance::calculate(&query, &vector) (hnsw/index.rs:407) in the index's type
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(METRICS.index(metric) * 4 + TYPES.index(vt))
    orders = (2.0, 3.0) if metric == "minkowski" else (3.0,)
    for dim in (1, 3, 7, 8, 20, 129, 768, 1536):
        vecs = wrap_rows(rng, vt, gen(rng, metric, vt, (24, dim)))
        queries = [gen(rng, metric, vt, (dim,)), np.zeros(dim, R.DTYPES[vt]), vecs[1].copy(), vecs[7].copy()]
        if vt == "F64":
            qn = gen(rng, metric, vt, (dim,))
            qn[0] = np.nan
            queries += [np.full(dim, -0.0), qn]
        layers = [(np.zeros(25, np.uint64), np.zeros(0, np.uint32))]
        for p in orders:
            idx = HnswIndex(ctx, vecs, layers, 0, metric, minkowski_order=p, vector_type=vt)
            for q in queries:
                got = idx._typed_distances(q, vecs)
                for r in range(vecs.shape[0]):
                    want = R.distance(metric, q, vecs[r], p, vector_type=vt)
                    assert same(metric, got[r], want), (vt, metric, dim, p, r, got[r], want)
            idx.close()


def build(data32, metric, seed=1):
    h = O.Hnsw(data32.shape[1], GRAPH_METRIC.get(metric, "euclidean"), m=8, efc=60, seed=seed)
    for v in data32:
        h.insert(v)
    return h.export()


def check_walk(vt, metric, idx, g, queries, k, ef, **kw):
    ids, dist, cnt, ctr = idx.search_graph(queries, k, ef, counters=True, **kw)
    for q in range(queries.shape[0]):
        oi, od, oc = R.search_csr(g, queries[q], k, ef, metric, vector_type=vt, **kw)
        assert cnt[q] == oi.size, (vt, metric, k, ef, q)
        assert list(ids[q, : cnt[q]]) == list(oi), (vt, metric, k, ef, q)
        assert (int(ctr[q, 0]), int(ctr[q, 1])) == oc, (vt, metric, k, ef, q)
        assert all(same(metric, a, b) for a, b in zip(dist[q, : cnt[q]], od)), (vt, metric, k, ef, q)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vt", TYPES)
def test_walk_parity(ctx, vt, metric):
    # plain, filtered and pending walks: ids, f64 distances and both visit counters
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(100 + METRICS.index(metric) * 4 + TYPES.index(vt))
    dim, n = 20, 700
    data = gen(rng, metric, vt, (n, dim))
    queries = gen(rng, metric, vt, (24, dim))
    g = dict(build(data.astype(np.float32), metric), vectors=data)
    idx = HnswIndex(ctx, data, g["layers"], g["entry_point"], metric, vector_type=vt)
    for k, ef in ((10, 40), (4, 8)):
        check_walk(vt, metric, idx, g, queries, k, ef)
    truthy = (rng.random(n) < 0.5).astype(np.uint8)
    try:
        check_walk(vt, metric, idx, g, queries, 10, 40, truthy=truthy)
    except Exception as e:  # a filter too selective for the on-chip window -> the caller's CPU path
        assert "SDB_EOVERFLOW" in str(e), str(e)
    pending = (rng.random(n) < 0.1).astype(np.uint8)
    check_walk(vt, metric, idx, g, queries, 10, 40, all_docs_pending=pending)
    idx.close()


@pytest.mark.parametrize("metric", ["euclidean", "manhattan", "cosine", "pearson", "chebyshev"])
def test_i16_walk_wraps_inside_the_walk(ctx, metric):
    # values near +-30000: the i16 difference of Manhattan and the i16 dot of cosine wrap on most pairs
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(7 + len(metric))
    dim, n = 16, 600
    data = (rng.choice([-30000, 30000], (n, dim)) + rng.integers(-400, 400, (n, dim))).astype(np.int16)
    queries = (rng.choice([-30000, 30000], (16, dim)) + rng.integers(-400, 400, (16, dim))).astype(np.int16)
    g = dict(build(data.astype(np.float32), metric, seed=2), vectors=data)
    idx = HnswIndex(ctx, data, g["layers"], g["entry_point"], metric, vector_type="I16")
    for k, ef in ((10, 40), (3, 6)):
        check_walk("I16", metric, idx, g, queries, k, ef)


def kv_index(vt, vectors, g):
    he = [(e, K.ser_vector(vt, vectors[e])) for e in range(vectors.shape[0])]
    hn = [[(e, K.node_to_val(ci[rp[e]:rp[e + 1]])) for e in range(vectors.shape[0]) if rp[e + 1] > rp[e]]
          for rp, ci in g["layers"]]
    state = K.hnsw_state(int(g["entry_point"]), vectors.shape[0], (len(he), 0), tuple((1, 0) for _ in g["layers"][1:]))
    return state, he, hn


@pytest.mark.parametrize("vt", TYPES)
@pytest.mark.parametrize("metric", ["euclidean", "jaccard", "pearson", "cosine"])
def test_staged_typed_loader_equals_the_host_loader(ctx, vt, metric):
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(31 + TYPES.index(vt))
    dim, n = 12, 500
    data = gen(rng, metric, vt, (n, dim))
    queries = gen(rng, metric, vt, (16, dim))
    g = dict(build(data.astype(np.float32), metric), vectors=data)
    host = HnswIndex(ctx, data, g["layers"], g["entry_point"], metric, vector_type=vt)
    state, he, hn = kv_index(vt, data, g)
    staged = HnswIndex.from_kv(ctx, dim, state, he, hn, metric, vector_type=vt)
    assert staged.n_bad == 0
    for k, ef in ((10, 40), (3, 5)):
        a = host.search_graph(queries, k, ef, counters=True)
        b = staged.search_graph(queries, k, ef, counters=True)
        for x, y in zip(a, b):
            assert x.tobytes() == y.tobytes(), (vt, metric, k, ef)
    check_walk(vt, metric, staged, g, queries, 10, 40)


def two_element_graph():
    return [(np.array([0, 1, 2], np.uint64), np.array([1, 0], np.uint32))]


def test_staged_values_keep_their_native_precision(ctx):
    from surrealdb_b200.hnsw import HnswIndex
    g = {"layers": two_element_graph(), "entry_point": 0}
    # I64 2^53 + 1 is not an f64: it must not become 2^53
    big = 2 ** 53 + 1
    data = np.array([[big, 0], [big - 1, 0]], np.int64)
    state, he, hn = kv_index("I64", data, g)
    idx = HnswIndex.from_kv(ctx, 2, state, he, hn, "hamming", vector_type="I64")
    ids, dist, cnt = idx.search_graph(np.array([[big, 0]], np.int64), 2, 4)
    assert list(ids[0, :2]) == [0, 1] and list(dist[0, :2]) == [0.0, 1.0]
    # F64 0.1 is not an f32
    data = np.array([[0.1, 0.0], [float(np.float32(0.1)), 0.0]])
    state, he, hn = kv_index("F64", data, g)
    idx = HnswIndex.from_kv(ctx, 2, state, he, hn, "hamming", vector_type="F64")
    ids, dist, cnt = idx.search_graph(np.array([[0.1, 0.0]]), 2, 4)
    assert list(ids[0, :2]) == [0, 1] and list(dist[0, :2]) == [0.0, 1.0]


def test_staged_value_of_another_type_is_counted_bad(ctx):
    from surrealdb_b200.hnsw import HnswIndex
    g = {"layers": [(np.array([0, 1, 2, 2], np.uint64), np.array([1, 0], np.uint32))], "entry_point": 0}
    data = np.array([[1, 2], [3, 4], [5, 6]], np.int32)
    state, he, hn = kv_index("I32", data, g)
    he[2] = (2, K.ser_vector("F32", data[2]))  # an F32 value in an I32 index
    idx = HnswIndex.from_kv(ctx, 2, state, he, hn, "euclidean", vector_type="I32")
    assert idx.n_bad == 1
    ids, dist, cnt = idx.search_graph(np.array([[5, 6]], np.int32), 3, 4)
    assert cnt[0] == 2 and 2 not in list(ids[0, :2])


def test_load_typed_f32_equals_load(ctx):
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.hnsw import HnswIndex
    rng = np.random.default_rng(5)
    data = rng.uniform(-20, 20, (600, 24)).astype(np.float32)
    queries = rng.uniform(-20, 20, (32, 24)).astype(np.float32)
    g = build(data, "cosine")
    for metric in ("cosine", "euclidean", "pearson"):
        typed = HnswIndex(ctx, data, g["layers"], g["entry_point"], metric, vector_type="F32")
        nl = len(g["layers"])
        rps = [np.ascontiguousarray(l[0], np.uint64) for l in g["layers"]]
        cis = [np.ascontiguousarray(l[1] if len(l[1]) else np.zeros(1, np.uint32), np.uint32) for l in g["layers"]]
        h = C.c_void_p()
        L.check(L.lib().sdb_hnsw_load(ctx.h, 24, L.METRIC[metric.upper()], 600, C.c_void_p(data.ctypes.data), nl,
                                      (C.c_void_p * nl)(*[a.ctypes.data for a in rps]),
                                      (C.c_void_p * nl)(*[a.ctypes.data for a in cis]), int(g["entry_point"]), C.byref(h)))
        ids = np.zeros((32, 10), np.uint64)
        dist = np.zeros((32, 10), np.float64)
        cnt = np.zeros(32, np.uint32)
        ctr = np.zeros((32, 2), np.uint64)
        L.check(L.lib().sdb_hnsw_search(h, C.c_void_p(queries.ctypes.data), 32, 10, 40, C.c_void_p(ids.ctypes.data),
                                        C.c_void_p(dist.ctypes.data), C.c_void_p(cnt.ctypes.data),
                                        C.c_void_p(ctr.ctypes.data)))
        L.lib().sdb_hnsw_destroy(h)
        for x, y in zip(typed.search_graph(queries, 10, 40, counters=True), (ids, dist, cnt, ctr)):
            assert x.tobytes() == y.tobytes(), metric


def test_refusals(ctx):
    from surrealdb_b200 import _lib as L
    cis = np.zeros(1, np.uint32)
    CI = (C.c_void_p * 1)(cis.ctypes.data)
    rp = np.zeros(2, np.uint64)
    RP = (C.c_void_p * 1)(rp.ctypes.data)
    h = C.c_void_p()
    v = np.zeros(32768, np.int16)
    assert L.lib().sdb_hnsw_load_typed(ctx.h, 4, L.METRIC["EUCLIDEAN"], 7, 1, C.c_void_p(v.ctypes.data), 1, RP, CI, 0,
                                       C.byref(h)) == L.SDB_EINVAL
    assert L.lib().sdb_hnsw_load_typed(ctx.h, 32768, L.METRIC["PEARSON"], L.VTYPE["I16"], 1, C.c_void_p(v.ctypes.data), 1,
                                       RP, CI, 0, C.byref(h)) == L.SDB_EUNSUPPORTED
    assert "i16" in L.lib().sdb_last_error().decode()
    # I16 PEARSON up to the reference's limit, and other metrics beyond it, load
    L.check(L.lib().sdb_hnsw_load_typed(ctx.h, 32767, L.METRIC["PEARSON"], L.VTYPE["I16"], 1, C.c_void_p(v.ctypes.data), 1,
                                        RP, CI, 0, C.byref(h)))
    L.lib().sdb_hnsw_destroy(h)
    L.check(L.lib().sdb_hnsw_load_typed(ctx.h, 32768, L.METRIC["EUCLIDEAN"], L.VTYPE["I16"], 1, C.c_void_p(v.ctypes.data), 1,
                                        RP, CI, 0, C.byref(h)))
    L.lib().sdb_hnsw_destroy(h)
    # the staged typed loader refuses the same way
    NB = (C.c_void_p * 1)(np.zeros(1, np.uint8).ctypes.data)
    NO = (C.c_void_p * 1)(np.zeros(1, np.uint64).ctypes.data)
    NN = (C.c_uint64 * 1)(0)
    assert L.lib().sdb_hnsw_load_staged_typed(ctx.h, 4, L.METRIC["EUCLIDEAN"], 9, 1, None, None, None, 0, 1, NB, NO, NO,
                                              NN, -1, C.byref(h), None) == L.SDB_EINVAL


def test_f64_pearson_negative_zero_distance(ctx):
    # F64 PEARSON underflows to -0.0 for element 1 ([1e10, -1e10, 1e-320] against [0, 0, -1]).  The walk, the exact kNN
    # and the document-level result order by FloatKey (total_cmp: -0.0 before 0.0) and return -0.0 with its sign; the
    # walk still expands a 0.0 candidate when its f is -0.0 (cq_dist > fq_dist compares f64s).  Compared by bits.
    import torch
    import hnsw_select_ref as S
    from surrealdb_b200.hnsw import HnswIndex
    from surrealdb_b200.hnsw_build import knn_exact
    rng = np.random.default_rng(0)
    special = np.array([[1.0, -1.0, 0.0], [1e10, -1e10, 1e-320], [5.0, 5.0, 5.0], [-2.0, 2.0, 0.0]])
    data = np.concatenate([rng.uniform(0, 1, (6, 3)) * np.array([1.0, 1.0, -1.0]), special, rng.uniform(-1, 1, (4, 3))])
    q = np.array([[0.0, 0.0, -1.0]])
    n = data.shape[0]
    full = np.array([j for i in range(n) for j in range(n) if j != i], np.uint32)  # every element links every other
    layers = [(np.arange(n + 1, dtype=np.uint64) * (n - 1), full)]
    wi, wd = S.knn("pearson", data, q[0], n, vector_type="F64")
    zero = [int(i) for i, d in zip(wi, wd) if d == 0.0]
    assert len(zero) == 4 and zero[0] == 7 and np.signbit(wd[list(wi).index(7)])  # -0.0 first among the zeros
    first = list(wi).index(7)
    g = dict(vectors=data, layers=layers, entry_point=0)
    for entry in (0, 7, 6):
        g["entry_point"] = entry
        idx = HnswIndex(ctx, data, layers, entry, "pearson", vector_type="F64")
        for k, ef in ((first + 1, first + 1), (first + 2, first + 2), (first + 1, n), (n, n), (1, 1)):
            ids, dist, cnt, ctr = idx.search_graph(q, k, ef, counters=True)
            oi, od, oc = R.search_csr(g, q[0], k, ef, "pearson", vector_type="F64")
            assert cnt[0] == oi.size and list(ids[0, : cnt[0]]) == list(oi), (entry, k, ef)
            assert dist[0, : cnt[0]].tobytes() == od.tobytes(), (entry, k, ef)
            assert (int(ctr[0, 0]), int(ctr[0, 1])) == oc, (entry, k, ef)
        res = idx.knn_search(q[0], first + 2, n)
        assert [int(v) for v, _ in res] == list(wi[: first + 2])
        assert np.array([d for _, d in res]).tobytes() == wd[: first + 2].tobytes()
        for k in (first + 1, first + 2, n):
            ids, dist, cnt = knn_exact(idx.h, torch.from_numpy(q).cuda(), k)
            ids, dist, cnt = ids.cpu().numpy(), dist.cpu().numpy(), cnt.cpu().numpy()
            assert cnt[0] == k and list(ids[0, :k]) == list(wi[:k]), k
            assert dist[0, :k].tobytes() == wd[:k].tobytes(), k
        idx.close()
