"""Test reference for the GPU HNSW builder's two primitives, restated on tests/hnsw_types_ref.py's distance():

  knn(metric, X, q, k, members, order, vector_type)       TestCollection::knn (idx/trees/hnsw/mod.rs:1186-1197):
                                                          calculate(X[e], q) for every member e, the k smallest by
                                                          (total-order key, element id) -- KnnResultBuilder's order
  select(metric, X, elem, cand, m_max, presorted, ...)    Heuristic::select, standard variant
                                                          (idx/trees/hnsw/heuristic.rs:61-81,201-216)

Distances are ordered by f64::total_cmp, the order of FloatKey (idx/trees/knn.rs:129-160): -0.0 before 0.0, and each
distance is reported as computed, -0.0 included.  A NaN distance sorts after +inf here; on the GPU it ranks by the bit pattern the GPU produced (DESIGN.md section 8), so the
tests compare the non-NaN part of a ranking.
"""
import numpy as np

import hnsw_types_ref as R


def distances(metric, X, q, order=3.0, vector_type="F32"):
    """calculate(X[r], q) for every row; F32 COSINE is the oracle's (tests/hnsw_metric_ref.py does not restate it)"""
    if vector_type == "F32" and metric == "cosine":
        from oracle import pyoracle as O
        return np.array([O.vec_distance_f32("cosine", x, q) for x in np.atleast_2d(np.asarray(X, np.float32))])
    return R.distances(metric, X, q, order, vector_type)


def key(d):
    """FloatKey's total-order key of an f64 distance (f64::total_cmp: -0.0 before 0.0; NaN after +inf here)"""
    d = float(d)
    if d != d:
        return (1, 0)
    b = int(np.float64(d).view(np.int64))
    return (0, b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF))


def knn(metric, X, q, k, members=None, order=3.0, vector_type="F32"):
    """-> (element ids int64, distances f64), at most k, ordered by (key, id)"""
    ids = np.arange(X.shape[0]) if members is None else np.sort(np.asarray(members, np.int64))
    d = distances(metric, np.asarray(X)[ids], q, order, vector_type)
    rank = sorted(range(ids.size), key=lambda i: (key(d[i]), int(ids[i])))[:k]
    out = np.array([d[i] for i in rank], np.float64)
    return ids[rank].astype(np.int64), out


def select(metric, X, elem, cand, m_max, presorted, order=3.0, vector_type="F32"):
    """Heuristic::select for element `elem` over the candidate ids `cand` -> accepted ids, in acceptance order.

    presorted: cand is visited as given and e_dist = calculate(X[e], X[elem]), the distance an insertion search ranked
    it by (element first, the new element as the query); otherwise (build_priority_list, layer.rs:389-405) e_dist =
    calculate(X[elem], X[e]) and cand is visited by (key of e_dist, list position).  The element itself is skipped; when
    at most m_max other candidates remain they are all taken.  e is rejected when e_dist > calculate(X[r], X[e]) for
    an accepted r (elements.rs:133-140)."""
    cand = [int(c) for c in cand]

    def dist(a, b):
        return float(distances(metric, np.asarray(X)[a][None, :], X[b], order, vector_type)[0])

    real = [j for j, c in enumerate(cand) if c != elem]
    take_all = len(real) <= m_max
    e_dist = {}
    if not (presorted and take_all):
        for j in real:
            e_dist[j] = dist(cand[j], elem) if presorted else dist(elem, cand[j])
    visit = real if presorted else sorted(real, key=lambda j: (key(e_dist[j]), j))
    acc = []
    for j in visit:
        if len(acc) >= m_max:
            break
        e = cand[j]
        if not take_all and any(e_dist[j] > dist(r, e) for r in acc):
            continue
        acc.append(e)
    return acc
