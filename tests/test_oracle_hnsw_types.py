"""The HNSW metrics of the vector types other than F32 (VectorType F64, I64, I32, I16; idx/trees/vector.rs:206-451),
restated in tests/hnsw_types_ref.py: the reference's known answers, the F64 restatement against the CPU oracle, the
wrapping and quirks of each type worked by hand, the reference's distance-collection and simple-HNSW tests, and the
conversion of query numbers to the index's type."""
import math

import numpy as np
import pytest

import hnsw_types_ref as R
from oracle import pyoracle as O

A, B = [1.0, 2.0, 3.0], [2.0, 3.0, 4.0]
METRICS = ["chebyshev", "cosine", "euclidean", "hamming", "jaccard", "manhattan", "minkowski", "pearson"]


@pytest.mark.parametrize("metric,want", [
    # vector.rs:723-772 (test_distance on [1,2,3] / [2,3,4] with VectorType::F64)
    ("chebyshev", 1.0), ("cosine", 0.007416666029069652), ("euclidean", 1.7320508075688772), ("hamming", 3.0),
    ("jaccard", 0.5), ("manhattan", 3.0), ("minkowski", 1.4422495703074083), ("pearson", 1.0),
])
def test_reference_known_answers_f64(metric, want):
    assert R.distance(metric, A, B, vector_type="F64") == want


def test_f64_cosine_and_euclid_equal_the_oracle():
    rng = np.random.default_rng(21)
    for dim in (1, 3, 7, 8, 9, 20, 129, 768):
        X = rng.uniform(-20, 20, (24, dim))
        X[1] = 0.0
        X[2] = -0.0
        X[3] = 5.0
        X[4, ::3] = np.nan
        X[5, : (dim + 1) // 2] = -0.0
        X[6] = rng.uniform(-1e-300, 1e-300, dim)
        X[7] = rng.uniform(-1e300, 1e300, dim)
        for q in (X[0], X[8] + 0.5, np.zeros(dim)):
            for metric in ("cosine", "euclidean"):
                got = R.distances(metric, X, q, vector_type="F64")
                for r in range(X.shape[0]):
                    want = O.vec_distance_f64(metric, X[r], q)
                    assert (math.isnan(want) and math.isnan(got[r])) or got[r] == want, (metric, dim, r, got[r], want)


def test_f64_jaccard_is_a_distance():
    # jaccard_f64 returns 1 - inter / union (vector.rs:316-327), the other types the similarity
    assert R.distance("jaccard", [1, 2, 3], [1, 1, 1], vector_type="F64") == 0.0
    assert R.distance("jaccard", [1, 2, 3], [1, 1, 1]) == 1.0
    assert R.distance("jaccard", [1, 2, 3], [1, 1, 1], vector_type="I32") == 1.0
    assert R.distance("jaccard", [0.0], [-0.0], vector_type="F64") == 1.0  # bit patterns: 0.0 and -0.0 differ


def test_i16_cosine_dot_wraps_in_i16():
    # dot = 200*200 = 40000 wraps to 40000 - 65536 = -25536 in i16; the norms are exact f64
    got = R.distance("cosine", [200], [200], vector_type="I16")
    assert got == 1.0 - (-25536.0) / (200.0 * 200.0)
    assert R.distance("cosine", [200], [200], vector_type="I32") == 0.0
    # at dim 1536 with |x| <= 20 the dot passes 32767
    x = np.full(1536, 20, np.int16)
    assert R.distance("cosine", x, x, vector_type="I16") == 1.0 - float(np.int16(1536 * 400 - 65536 * 9)) / (
        math.sqrt(1536 * 400.0) ** 2)


def test_i16_manhattan_subtraction_wraps():
    # 30000 - (-30000) = 60000 wraps to -5536 in i16, |f64(-5536)| = 5536
    assert R.distance("manhattan", [30000], [-30000], vector_type="I16") == 5536.0
    assert R.distance("manhattan", [30000], [-30000], vector_type="I32") == 60000.0
    # chebyshev and euclidean convert before subtracting: no wrap
    assert R.distance("chebyshev", [30000], [-30000], vector_type="I16") == 60000.0
    assert R.distance("euclidean", [30000], [-30000], vector_type="I16") == 60000.0


def test_i32_euclid_square_sum_wraps():
    # 50000^2 = 2.5e9 wraps to 2.5e9 - 2^32 < 0 in i32: the sqrt of that negative f64 is NaN
    assert math.isnan(R.distance("euclidean", [50000], [0], vector_type="I32"))
    # three squares of 40000^2: 4.8e9 wraps to 4.8e9 - 2^32 = 505032704
    assert R.distance("euclidean", [40000] * 3, [0] * 3, vector_type="I32") == math.sqrt(505032704.0)
    assert R.distance("euclidean", [40000] * 3, [0] * 3, vector_type="I64") == math.sqrt(4.8e9)


def test_i64_abs_of_min_stays_negative():
    mn = np.iinfo(np.int64).min
    # 0 - MIN wraps to MIN; abs(MIN) = MIN
    assert R.distance("manhattan", [0], [mn], vector_type="I64") == float(mn)
    assert R.distance("manhattan", [0, 0], [mn, 1], vector_type="I64") == float(mn + 1)  # MIN + 1, wrapping
    assert R.distance("chebyshev", [0], [mn], vector_type="I64") == 0.0                 # MIN never wins from 0
    assert R.distance("chebyshev", [0, 0], [mn, 5], vector_type="I64") == 5.0


def test_integer_pearson_mean_truncates_toward_zero():
    # x = [-3, 0]: sum -3, mean -3 / 2 = -1 in i32 (truncation toward zero, not floor's -2)
    x, y = [-3, 0], [1, 4]
    mx, my = -1.0, 2.0
    dx = [-3.0 - mx, 0.0 - mx]
    dy = [1.0 - my, 4.0 - my]
    sxy = dx[0] * dy[0] + dx[1] * dy[1]
    den = math.sqrt((dx[0] ** 2 + dx[1] ** 2) * (dy[0] ** 2 + dy[1] ** 2))
    for vt in ("I64", "I32", "I16"):
        assert R.distance("pearson", x, y, vector_type=vt) == sxy / den
    assert R.distance("pearson", x, y, vector_type="F64") == 1.0
    with pytest.raises(ValueError):
        R.distance("pearson", np.zeros(32768), np.ones(32768), vector_type="I16")


def gen_typed(rng, metric, vt, dim):
    """new_random_vec (idx/trees/knn.rs:630-641 + Vector::try_from_vector): integers in [0, 2) for Hamming, in [0, dim/2)
    for Jaccard, uniform(-20, 20) otherwise, truncated toward zero for the integer types"""
    if metric == "hamming":
        v = rng.integers(0, 2, dim).astype(np.float64)
    elif metric == "jaccard":
        v = rng.integers(0, max(dim // 2, 1), dim).astype(np.float64)
    else:
        v = rng.uniform(-20, 20, dim)
    return v if vt == "F64" else np.trunc(v).astype(R.DTYPES[vt])


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vt", ["F64", "F32", "I64", "I32", "I16"])
def test_distance_collection(metric, vt):
    # test_distance_collection (vector.rs:697-720): 100 pairs, dim 1536 (768 for Jaccard): finite, < 10 % zeros
    if vt == "F32" and metric == "cosine":
        pytest.skip("F32 cosine is the oracle's (tests/test_oracle_metrics.py)")
    rng = np.random.default_rng(METRICS.index(metric) * 8 + ["F64", "F32", "I64", "I32", "I16"].index(vt))
    dim = 768 if metric == "jaccard" else 1536
    zeros = 0
    for _ in range(100):
        a, b = gen_typed(rng, metric, vt, dim), gen_typed(rng, metric, vt, dim)
        if vt == "F32":
            a, b = a.astype(np.float32), b.astype(np.float32)
        d = R.distance(metric, a, b, vector_type=vt)
        assert math.isfinite(d), (metric, vt, d)
        zeros += d == 0.0
    assert zeros / 100 < 0.1, (metric, vt, zeros)


def test_simple_hnsw_i16():
    # test_simple_hnsw (hnsw/mod.rs:1002-1037): 11 I16 points of dim 2, m=3, efc=500, EUCLIDEAN; search (-2, -3) with
    # k=10, ef=501 returns 10 results.  The graph is linked by the oracle on the f32 copy (the same values).
    pts = np.array([(-2, -3), (-2, 1), (-4, 3), (-3, 1), (-1, 1), (-2, 3), (3, 0), (-1, -2), (-2, 2), (-4, -2), (0, 3)],
                   np.int16)
    h = O.Hnsw(2, "euclidean", m=3, efc=500, seed=1)
    for v in pts.astype(np.float32):
        h.insert(v)
    g = h.export()
    g16 = dict(g, vectors=pts)
    ids, dist, _ = R.search_csr(g16, np.array([-2, -3], np.int16), 10, 501, "euclidean", vector_type="I16")
    assert ids.size == 10
    assert ids[0] == 0 and dist[0] == 0.0
    want = sorted(math.sqrt(float((int(x) + 2) ** 2 + (int(y) + 3) ** 2)) for x, y in pts)[:10]
    assert sorted(dist.tolist()) == want


def test_restated_typed_walk_equals_the_f32_walk_where_the_arithmetic_agrees():
    # small integers: every I32 / I64 distance of euclid and manhattan equals the F32 one, so the walks are identical
    rng = np.random.default_rng(6)
    data = rng.integers(-20, 20, (400, 10)).astype(np.float32)
    h = O.Hnsw(10, "euclidean", m=8, efc=60, seed=3)
    for v in data:
        h.insert(v)
    g = h.export()
    for metric in ("euclidean", "manhattan"):
        for vt in ("I64", "I32", "F64"):
            gt = dict(g, vectors=data.astype(R.DTYPES[vt]))
            for q in data[:4] + 1:
                a = R.search_csr(g, q, 10, 40, metric)
                b = R.search_csr(gt, q.astype(R.DTYPES[vt]), 10, 40, metric, vector_type=vt)
                assert list(a[0]) == list(b[0]) and a[1].tobytes() == b[1].tobytes() and a[2] == b[2], (metric, vt)


def test_query_conversion_rule():
    from surrealdb_b200 import SdbError
    from surrealdb_b200.hnsw import to_vector_type
    assert to_vector_type([1.9, -1.9, 0.5, -0.5], "I16").tolist() == [1, -1, 0, 0]   # truncation toward zero
    assert to_vector_type([32767, -32768], "I16").tolist() == [32767, -32768]
    assert to_vector_type([32767.9, -32768.9], "I16").tolist() == [32767, -32768]
    for bad in ([32768], [-32769], [32768.0], [float("nan")], [float("inf")]):
        with pytest.raises(SdbError, match="SDB_EINVAL"):
            to_vector_type(bad, "I16")
    big = 2 ** 53 + 1
    assert to_vector_type(np.array([big], np.int64), "I64").tolist() == [big]   # integers keep their value
    assert to_vector_type(np.array([big], object), "I64").tolist() == [big]
    with pytest.raises(SdbError, match="SDB_EINVAL"):
        to_vector_type([2.0 ** 63], "I64")
    assert to_vector_type([-(2.0 ** 63)], "I64").tolist() == [-(2 ** 63)]
    assert to_vector_type([2 ** 31 - 1, 1.5e9], "I32").tolist() == [2 ** 31 - 1, 1500000000]
    with pytest.raises(SdbError, match="SDB_EINVAL"):
        to_vector_type([2 ** 31], "I32")
    # floats: today's conversion
    assert to_vector_type([0.1], "F32").dtype == np.float32 and to_vector_type([0.1], "F32")[0] == np.float32(0.1)
    assert to_vector_type([0.1], "F64")[0] == 0.1
