"""Pins tests/select_ref.py (the order the exact kernel's radix select and the shard merges return) on hand-picked
values and against the oracle's KnnTopK, so the GPU selection tests compare the kernels with Number::cmp and not with
a second copy of a mistake."""
import numpy as np
import pytest

import select_ref as R
from oracle import pyoracle as O

GEN_NAN = np.uint64(0xFFF8000000000000).view(np.float64)  # 0/0 on x86-64: negative, sorts first
DATA_NAN = np.uint64(0x7FF8000000000000).view(np.float64)  # f64::NAN from the data: positive, sorts last

# the PEARSON similarity of row 0 underflows to -0.0; the oracle returns it with its sign
NEG_ZERO_CORPUS = np.array([[0.0, -8.805437202403729e-162, -5.870291468269152e-162], [1, 2, 3], [0, 0, 1]])
NEG_ZERO_QUERY = np.array([5.870291468269152e-162, 8.805437202403729e-162, 2.935145734134576e-162])


def bits(a):
    return np.asarray(a, np.float64).view(np.uint64).tolist()


def test_num_key_is_the_full_order():
    ladder = [GEN_NAN, -np.inf, -1.7976931348623157e308, -1.0, -2.2250738585072014e-308, -5e-324, -0.0,
              5e-324, 2.2250738585072014e-308, 1.0, 1.7976931348623157e308, np.inf, DATA_NAN]
    keys = R.num_key(np.array(ladder)).tolist()
    zero = ladder.index(-0.0)
    assert keys[zero] == R.num_key(0.0)[0] == 1 << 63  # -0.0 and 0.0 are one key
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    # shuffled, with every value twice: the order is the ladder, each value's rows ascending, -0.0 tying with 0.0
    vals = np.array(ladder + [0.0] + ladder)
    rng = np.random.default_rng(1)
    perm = rng.permutation(vals.size)
    rows, got = R.topk(vals[perm], vals.size)
    want = sorted(range(vals.size), key=lambda i: (R.num_key(vals[perm][i])[0], i))
    assert rows.tolist() == want
    assert bits(got) == bits(vals[perm][want])  # the values come back as given: -0.0 keeps its sign
    assert bits(got[:2]) == bits([GEN_NAN, GEN_NAN]) and bits(got[-2:]) == bits([DATA_NAN, DATA_NAN])


@pytest.mark.parametrize("k", [0, 1, 3, 4, 5, 9, 50])
def test_topk_cuts_inside_tie_groups(k):
    vals = np.array([2.0, 1.0, -0.0, 1.0, 0.0, 2.0, 1.0, -0.0, 3.0])
    skip = np.array([0, 0, 0, 1, 0, 0, 0, 0, 0], np.uint8)
    rows, got = R.topk(vals, k, skip)
    want = [2, 4, 7, 1, 6, 0, 5, 8][:k]
    assert rows.tolist() == want and bits(got) == bits(vals[want])


def test_topk_large_is_linear_and_exact():
    rng = np.random.default_rng(2)
    vals = rng.integers(0, 50, 2_000_000).astype(np.float64)
    skip = (rng.random(vals.size) < 0.3).astype(np.uint8)
    for k in (1, 256, 4096):
        rows, got = R.topk(vals, k, skip)
        valid = np.nonzero(skip == 0)[0]
        want = valid[np.lexsort((valid, vals[valid]))][:k]
        assert rows.tolist() == want.tolist() and bits(got) == bits(vals[want])


@pytest.mark.parametrize("metric", ["cosine", "euclidean", "manhattan", "chebyshev", "hamming", "pearson", "jaccard"])
def test_topk_agrees_with_oracle_knn(metric):
    rng = np.random.default_rng(len(metric))
    corpus = rng.integers(-3, 4, (400, 5)).astype(np.float64)  # small alphabet: many exact ties
    corpus[[5, 77, 300]] = 0.0          # zero rows: generated NaN for cosine / pearson
    corpus[[9, 200], 1] = np.nan        # data NaN
    corpus[10:13] = NEG_ZERO_CORPUS[0].tolist() + [0.0, 0.0]
    queries = np.vstack([rng.integers(-3, 4, (4, 5)), [0.0] * 5, NEG_ZERO_QUERY.tolist() + [0.0, 0.0]])
    skip = (rng.random(400) < 0.1).astype(np.uint8)
    for q in queries:
        vals = np.array([O.f64_metric(metric, row, q) for row in corpus])
        for k in (1, 7, 64, 399, 500):
            for sk in (None, skip):
                r, d = O.knn_topk(corpus, q, metric, k, skip=sk)
                rows, got = R.topk(vals, k, sk)
                assert rows.tolist() == r.tolist(), (metric, k)
                assert bits(got) == bits(d), (metric, k)


def test_topk_keeps_the_negative_zero_pearson_similarity():
    vals = np.array([O.f64_metric("pearson", row, NEG_ZERO_QUERY) for row in NEG_ZERO_CORPUS])
    r, d = O.knn_topk(NEG_ZERO_CORPUS, NEG_ZERO_QUERY, "pearson", 3)
    rows, got = R.topk(vals, 3)
    assert r.tolist() == rows.tolist() == [2, 1, 0]
    assert bits(d)[2] == bits(got)[2] == 0x8000000000000000


def test_merge_orders_across_lists_and_truncates_counts():
    k = 4
    # two disjoint shards of one query, each sorted by (key, row); distances repeat across lists
    rows = np.array([[[3, 8, 20, 21]], [[2, 9, 10, 30]]], np.uint64)
    dist = np.array([[[-0.0, 1.0, 1.0, DATA_NAN]], [[GEN_NAN, 0.0, 1.0, np.inf]]])
    for counts, want in (([[4], [4]], [2, 3, 9, 8]), ([[1], [0]], [3]), ([[0], [0]], []), ([[9], [2]], [2, 3, 9, 8]),
                         ([[4], [1]], [2, 3, 8, 20])):
        r, d, c = R.merge(rows, dist, np.array(counts), k)
        assert c.tolist() == [len(want)] and r[0, : len(want)].tolist() == want
    r, d, c = R.merge(rows, dist, np.array([[4], [4]]), 8)
    assert r[0].tolist() == [2, 3, 9, 8, 10, 20, 30, 21]
    assert bits(d[0]) == bits([GEN_NAN, -0.0, 0.0, 1.0, 1.0, 1.0, np.inf, DATA_NAN])
