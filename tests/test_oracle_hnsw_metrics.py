"""The typed F32 metrics that the HNSW walk serves beyond cosine / euclidean (idx/trees/vector.rs:218-451), restated in
tests/hnsw_metric_ref.py: the reference's known-answer vectors, hand-worked Jaccard cases, the tests_hnsw invariants,
and the restated walk checked against the CPU oracle's wherever the oracle restates the metric too."""
import math

import numpy as np
import pytest

import hnsw_metric_ref as R
from oracle import pyoracle as O

A, B = [1.0, 2.0, 3.0], [2.0, 3.0, 4.0]


@pytest.mark.parametrize("metric,want", [
    # vector.rs:723-772 (test_distance_* on [1,2,3] / [2,3,4]); the typed F32 values
    ("chebyshev", 1.0), ("euclidean", 1.7320508075688772), ("hamming", 3.0), ("jaccard", 0.5), ("manhattan", 3.0),
    ("minkowski", 1.4422495703074083), ("pearson", 1.0),
])
def test_reference_known_answers(metric, want):
    assert R.distance(metric, A, B) == want


def test_jaccard_argument_order_and_duplicates():
    # calculate(a, b): union = distinct(a); every b_i already in the set counts, so b's duplicates count too
    assert R.distance("jaccard", [1, 2, 3], [1, 1, 1]) == 1.0          # inter 3, |union| 3
    assert R.distance("jaccard", [1, 1, 1], [1, 2, 3]) == 1.0 / 3.0    # inter 1, |union| 3
    assert R.distance("jaccard", [1, 2], [3, 3]) == 1.0 / 3.0          # the 2nd 3 hits the inserted 3
    assert R.distance("jaccard", [5, 6, 7], [8, 9, 10]) == 0.0


def test_jaccard_compares_bit_patterns():
    nan1 = np.array([0x7FC00001], np.uint32).view(np.float32)[0]
    nan2 = np.array([0x7FC00002], np.uint32).view(np.float32)[0]
    assert R.distance("jaccard", [0.0], [-0.0]) == 0.0                 # -0.0 and 0.0 differ by their bits
    assert R.distance("jaccard", [0.0, 1.0], [0.0, 1.0]) == 1.0
    assert R.distance("jaccard", [nan1], [nan1]) == 1.0                # the same NaN payload is one pattern
    assert R.distance("jaccard", [nan1], [nan2]) == 0.0


def test_pearson_of_a_constant_vector_is_zero():
    assert R.distance("pearson", [4.0, 4.0, 4.0, 4.0], [1.0, 5.0, 2.0, 7.0]) == 0.0
    assert R.distance("pearson", [1.0, 5.0, 2.0, 7.0], [-3.0] * 4) == 0.0
    assert R.distance("pearson", [1.0, 2.0, 3.0], [3.0, 2.0, 1.0]) == -1.0


def test_pearson_restated_in_scalar_arithmetic():
    # the vectorised restatement against a plain per-element loop of vector.rs:412-451
    rng = np.random.default_rng(11)
    for n in (1, 7, 8, 9, 20, 129):
        x, y = rng.uniform(-20, 20, (2, n)).astype(np.float32)
        means = []
        for v in (x, y):
            p = [np.float32(0)] * 8
            for i in range(n // 8 * 8):
                p[i % 8] = np.float32(p[i % 8] + v[i])
            s = np.float32(0)
            for j in range(4):
                s = np.float32(s + np.float32(p[j] + p[j + 4]))
            for c in v[n // 8 * 8:]:
                s = np.float32(s + c)
            assert R.nd_sum_f32(v)[0] == s
            means.append(float(np.float32(s / np.float32(n))))
        sxy = sx2 = sy2 = 0.0
        for a, b in zip(x, y):
            dx, dy = float(a) - means[0], float(b) - means[1]
            sxy += dx * dy
            sx2 += dx * dx
            sy2 += dy * dy
        den = math.sqrt(sx2 * sy2)
        assert R.distance("pearson", x, y) == (0.0 if den == 0.0 else sxy / den)


@pytest.mark.parametrize("p", [1.0, 2.0, 3.0])
def test_minkowski_orders(p):
    assert R.distance("minkowski", A, B, p) == {1.0: 3.0, 2.0: 1.7320508075688772, 3.0: 1.4422495703074083}[p]
    rng = np.random.default_rng(int(p))
    a, b = rng.uniform(-20, 20, (2, 64)).astype(np.float32)
    want = sum(abs(float(x) - float(y)) ** p for x, y in zip(a, b)) ** (1.0 / p)
    assert math.isclose(R.distance("minkowski", a, b, p), want, rel_tol=1e-12)


@pytest.mark.parametrize("metric", ["euclidean", "manhattan", "chebyshev", "hamming"])
def test_restated_distances_equal_the_oracle(metric):
    rng = np.random.default_rng(3)
    for dim in (1, 7, 8, 20, 129):
        X = (rng.integers(0, 2, (30, dim)) if metric == "hamming" else rng.uniform(-20, 20, (30, dim))).astype(np.float32)
        X[1, ::2] = np.nan
        X[2] = -0.0
        q = X[5].copy() if dim > 1 else X[5] + 1
        got = R.distances(metric, X, q)
        for r in range(30):
            want = O.vec_distance_f32(metric, X[r], q)
            assert (math.isnan(want) and math.isnan(got[r])) or got[r] == want, (metric, dim, r)


@pytest.mark.parametrize("metric", ["euclidean", "manhattan", "hamming"])
def test_restated_walk_equals_the_oracle(metric):
    # plain, filtered and pending walks, ids + distances + both visit counters, on oracle-built graphs
    rng = np.random.default_rng(8)
    dim, n = 12, 500
    data = (rng.integers(0, 2, (n, dim)) if metric == "hamming" else rng.uniform(-20, 20, (n, dim))).astype(np.float32)
    h = O.Hnsw(dim, metric, m=8, efc=60, seed=2)
    for v in data:
        h.insert(v)
    g = h.export()
    truthy = (rng.random(n) < 0.4).astype(np.uint8)
    pending = (rng.random(n) < 0.2).astype(np.uint8)
    for q in data[:5] + np.float32(0.5) if metric != "hamming" else data[:5]:
        for k, ef in ((10, 40), (1, 1), (5, 8)):
            for kw in ({}, {"truthy": truthy}, {"all_docs_pending": pending}):
                oi, od, oc = O.hnsw_search_csr(g, q, k, ef, **kw)
                ri, rd, rc = R.search_csr(g, q, k, ef, metric, **kw)
                assert list(ri) == list(oi) and rd.tobytes() == od.tobytes() and rc == oc, (k, ef, kw.keys())


def test_hamming_small_collections_invariants():
    # tests_hnsw (hnsw/mod.rs:752-791) for Hamming: 30 unique vectors of integers in [0, 2) (knn.rs:630-641), dim 20,
    # m=24, efc=500; insert, then search each -> itself is found at distance 0
    rng = np.random.default_rng(4)
    rows = {}
    while len(rows) < 30:
        v = rng.integers(0, 2, 20).astype(np.float32)
        rows.setdefault(v.tobytes(), v)
    data = np.stack(list(rows.values()))
    for ext, keep in ((False, False), (True, False), (False, True), (True, True)):
        h = O.Hnsw(20, "hamming", m=24, efc=500, extend_candidates=ext, keep_pruned_connections=keep, seed=9)
        for v in data:
            h.insert(v)
            assert h.check_props()
        for i, v in enumerate(data):
            ids, dist = h.search(v, 1, 500)
            assert ids[0] == i and dist[0] == 0.0


def test_minkowski2_small_collections_invariants():
    # tests_hnsw for Minkowski(2): 30 uniform(-20, 20) vectors of dim 5, m=24, efc=500.  The restated walk in
    # Minkowski(2) over the graph the oracle links (in euclidean: the same neighbour order) finds every vector itself.
    rng = np.random.default_rng(5)
    data = rng.uniform(-20, 20, (30, 5)).astype(np.float32)
    h = O.Hnsw(5, "euclidean", m=24, efc=500, seed=9)
    for v in data:
        h.insert(v)
    g = h.export()
    for i, v in enumerate(data):
        ids, dist, _ = R.search_csr(g, v, 1, 500, "minkowski", order=2.0)
        assert ids[0] == i and dist[0] == 0.0
