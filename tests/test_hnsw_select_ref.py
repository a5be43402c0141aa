"""CPU checks of tests/hnsw_select_ref.py, the restatement the GPU builder's selection and exact kNN are tested
against, on hand-worked cases."""
import numpy as np

import hnsw_select_ref as S
import hnsw_types_ref as R

# points on a line, euclidean F64: d(i, j) = |x_i - x_j|
LINE = np.array([[0.0], [1.0], [2.0], [3.0], [-5.0], [-1.0]])


def test_take_all_when_at_most_m_max_candidates():
    # three candidates, m_max 3: every one is taken, in list order, although 2 and 3 lie behind 1
    assert S.select("euclidean", LINE, 0, [3, 1, 2], 3, True, vector_type="F64") == [3, 1, 2]
    # m_max 2: the heuristic runs -- 3 (e_dist 3) is accepted first, 1 (e_dist 1 < d(3, 1) = 2) too
    assert S.select("euclidean", LINE, 0, [3, 1, 2], 2, True, vector_type="F64") == [3, 1]
    # nearest first: 1, then 2 (e_dist 2 > d(1, 2) = 1) and 3 (3 > 2) are rejected
    assert S.select("euclidean", LINE, 0, [1, 2, 3], 2, True, vector_type="F64") == [1]


def test_the_element_itself_is_skipped_and_not_counted():
    # four entries, one of them the element: three real candidates <= m_max 3, so all of them are taken
    assert S.select("euclidean", LINE, 0, [0, 1, 2, 3], 3, True, vector_type="F64") == [1, 2, 3]
    assert S.select("euclidean", LINE, 0, [1, 0, 2, 3], 2, False, vector_type="F64") == [1]


def test_equal_distances_keep_list_order():
    # 1 and 5 are both at distance 1 from 0 (re-sort mode): FIFO, i.e. list order decides who is visited first
    assert S.select("euclidean", LINE, 0, [5, 1, 3], 1, False, vector_type="F64") == [5]
    assert S.select("euclidean", LINE, 0, [1, 5, 3], 1, False, vector_type="F64") == [1]
    # and both are kept: d(5, 1) = 2 is not closer than e_dist 1
    assert S.select("euclidean", LINE, 0, [1, 5, 3], 2, False, vector_type="F64") == [1, 5]


def test_resort_mode_orders_by_distance_to_the_element():
    # visited 1 (1), 2 (2), 3 (3), 4 (5): 2 and 3 lie behind 1; 4 (e_dist 5 < d(1, 4) = 6) is accepted
    assert S.select("euclidean", LINE, 0, [3, 4, 2, 1], 2, False, vector_type="F64") == [1, 4]
    # the same list presorted is visited as given: 3, then 4 (5 < d(3, 4) = 8)
    assert S.select("euclidean", LINE, 0, [3, 4, 2, 1], 2, True, vector_type="F64") == [3, 4]


def test_asymmetric_jaccard_f64_uses_the_reference_argument_orders():
    X = np.array([[1.0, 1.0, 2.0], [1.0, 2.0, 3.0], [1.0, 1.0, 1.0]])
    # jaccard_f64 (vector.rs:316-327): union = distinct(a); each b_i already in it counts, else joins it; 1 - inter/union
    assert R.distance("jaccard", X[0], X[1], vector_type="F64") == 1.0 - 2.0 / 3.0
    assert R.distance("jaccard", X[1], X[0], vector_type="F64") == 0.0
    assert R.distance("jaccard", X[0], X[2], vector_type="F64") == -0.5
    assert R.distance("jaccard", X[2], X[0], vector_type="F64") == 0.0
    # re-sort mode ranks by calculate(element, candidate): 2 (-0.5) before 1 (1/3).  The swapped order would tie them
    # at 0.0 and keep list order (1 first).
    assert S.select("jaccard", X, 0, [1, 2], 1, False, vector_type="F64") == [2]
    # presorted: the list order is the visiting order, whatever the distances
    assert S.select("jaccard", X, 0, [1, 2], 1, True, vector_type="F64") == [1]
    assert S.select("jaccard", X, 0, [2, 1, 0], 1, True, vector_type="F64") == [2]


def test_knn_orders_by_key_then_id():
    X = np.array([[0.0], [2.0], [-2.0], [1.0], [np.nan], [-0.0]])
    ids, d = S.knn("euclidean", X, np.array([0.0]), 6, vector_type="F64")
    # 0 and 5 tie at 0 (the -0.0 row gives +0.0), 1 and 2 tie at 2; NaN last
    assert list(ids) == [0, 5, 3, 1, 2, 4]
    assert np.signbit(d[1]) == False and np.isnan(d[-1])
    ids, d = S.knn("euclidean", X, np.array([0.0]), 2, members=[5, 2, 1], vector_type="F64")
    assert list(ids) == [5, 1]


def test_knn_keeps_a_negative_zero_pearson_distance_before_zero():
    # F64 PEARSON underflows to -0.0 for element 1: sxy is a tiny negative subnormal, the denominator about 1e10.
    # FloatKey orders by total_cmp, so it comes before the 0.0 of elements 0 (uncorrelated) and 2 (constant)
    X = np.array([[1.0, -1.0, 0.0], [1e10, -1e10, 1e-320], [5.0, 5.0, 5.0], [1.0, 2.0, 3.0]])
    q = np.array([0.0, 0.0, -1.0])
    ids, d = S.knn("pearson", X, q, 4, vector_type="F64")
    assert list(ids) == [3, 1, 0, 2]
    assert d[0] < 0 and d[1] == 0.0 and np.signbit(d[1]) and not np.signbit(d[2]) and not np.signbit(d[3])
