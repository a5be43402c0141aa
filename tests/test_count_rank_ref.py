"""CPU checks of the count path's model (count_rank_ref): the equality keys count exactly what Number equality on the
widened elements counts, JACCARD's count identity equals the reference's set computation, and the union of per-range
top-k lists holds the global top k under any ties."""
import numpy as np
import pytest

import count_rank_ref as R
from oracle import pyoracle as O


@pytest.mark.parametrize("fdt", [np.float32, np.float64])
def test_keys_count_what_equality_counts(fdt):
    rng = np.random.default_rng(7 if fdt == np.float32 else 8)
    sub = np.finfo(fdt).smallest_subnormal
    pool = np.concatenate([R.nan_patterns(fdt), np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, sub, -sub], fdt)])
    qpool = np.concatenate([pool.astype(np.float64), R.f64_nans(), [0.1, 1e300, 1e-320, -0.0, 2.0 ** -149]])
    for _ in range(200):
        row = pool[rng.integers(0, pool.size, 12)]
        query = qpool[rng.integers(0, qpool.size, 12)]
        assert R.hamming_by_keys(row, query) == R.hamming_by_equality(row, query), (row, query)


def test_f64_elements_without_an_f32_image_match_nothing():
    for q in [0.1, 1e300, 1e-320, float(R.f64_nans()[2]), float(R.f64_nans()[3])]:
        assert R.eq_qkey_f32(q) == R.EQ_KEY_NONE
    assert all(R.eq_key_f32(x) != R.EQ_KEY_NONE for x in R.nan_patterns(np.float32))
    assert R.eq_key_f32(np.float32(-0.0)) == R.eq_key_f32(np.float32(0.0)) == R.eq_qkey_f32(-0.0) == 0


def test_count_matches_the_oracle():
    rng = np.random.default_rng(11)
    corpus = rng.integers(-2, 3, (300, 9)).astype(np.float32)
    corpus[3, 2] = np.nan
    corpus[4, 1] = -0.0
    q = rng.integers(-2, 3, 9).astype(np.float64)
    q[2] = np.nan
    d = np.array([R.hamming_by_keys(corpus[i], q) for i in range(300)], np.float64)
    r, dd = O.knn_topk(corpus, q, "hamming", 300)
    assert np.array_equal(d[r], dd)
    assert list(r) == R.full_topk(d, 300)


@pytest.mark.parametrize("data", ["all_tied", "mostly_tied", "binary", "decreasing"])
def test_union_of_range_lists_holds_the_top_k(data):
    rng = np.random.default_rng(len(data))
    n = 997
    dist = {"all_tied": np.full(n, 5.0), "mostly_tied": np.where(rng.random(n) < 0.02, 3.0, 7.0),
            "binary": rng.binomial(16, 0.5, n).astype(np.float64), "decreasing": np.arange(n, 0, -1.0)}[data]
    skip = rng.random(n) < 0.1
    for k in (1, 2, 10, 100, 256):
        for s in (1, 2, 3, 16, 64, n):
            for sk in (None, skip):
                assert R.range_union_topk(dist, k, s, sk)[:k] == R.full_topk(dist, k, sk), (data, k, s)


def test_jaccard_identity_equals_the_reference():
    rng = np.random.default_rng(21)
    pool = [0.0, -0.0, 1.0, 2.0, -3.0, float("nan"), float("inf"), 0.5]
    for dim in (1, 2, 5, 17, 40):
        for _ in range(60):
            row = [pool[i] for i in rng.integers(0, len(pool), dim)]
            query = [pool[i] for i in rng.integers(0, len(pool), dim)]
            st, ref = O.num_metric("jaccard", row, query)
            assert st == 0
            got = R.jaccard_by_counts(np.array(row), np.array(query))
            assert np.float64(ref).tobytes() == got.tobytes(), (row, query, ref, got)
