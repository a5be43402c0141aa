"""Test reference for HNSW indexes of the vector types other than F32 (VectorType F64, I64, I32, I16;
idx/trees/vector.rs:206-451): all eight metrics, each in the type's own arithmetic, and the walk over an exported graph
in them.  F32 is delegated unchanged to tests/hnsw_metric_ref.py, whose walk (queues, visited set, counters) is reused.

  distance(metric, a, b, order, vector_type)     Distance::calculate(a, b) for two vectors of the type (JACCARD is
                                                 asymmetric in a, b)
  distances(metric, X, q, order, vector_type)    calculate(X[r], q) for every row: the walk's argument order
                                                 (hnsw/layer.rs:207,251)
  search_csr(graph, q, k, ef, metric, ..., vector_type)
                                                 hnsw_metric_ref.search_csr in the type's metric (graph "vectors" and
                                                 q hold values of the type)

Plain numpy, as in hnsw_metric_ref: every sequential fold is an `add.accumulate` in the array's dtype.  The integer
types are numpy arrays of their native dtype, so `+ - * abs` wrap as in the reference's release build (np.abs of the
minimum stays negative).
"""
import numpy as np

import hnsw_metric_ref as F32
from hnsw_metric_ref import _search_single, _seq_sum

DTYPES = {"F64": np.float64, "F32": np.float32, "I64": np.int64, "I32": np.int32, "I16": np.int16}


def nd_sum_f64(X):
    """nd_sum_f32 in f64: ArrayBase::sum of contiguous f64 rows (unrolled_fold), and the fold of ndarray's f64 dot.
    PARITY UNPINNED exactly like the f32 case (ndarray is not vendored): isolated here."""
    X = np.atleast_2d(np.asarray(X, np.float64))
    rows, dim = X.shape
    n8 = dim // 8 * 8
    if n8:
        p = _seq_sum(np.ascontiguousarray(X[:, :n8].reshape(rows, -1, 8).transpose(0, 2, 1)))  # (rows, 8)
    else:
        p = np.zeros((rows, 8), np.float64)
    s = np.zeros(rows, np.float64)
    for j in range(4):
        s = s + (p[:, j] + p[:, j + 4])
    for c in range(n8, dim):
        s = s + X[:, c]
    return s


def _wrap_sum(X):
    """a.sum() of integer rows in their own type: a wrapping sum, the same in any order"""
    return np.sum(X, axis=-1, dtype=X.dtype)


def _pearson_state(X, vector_type):
    """per row: mean (ndarray mean() in T, widened) and the sequential f64 sum of (f64(x_i) - mean)^2"""
    n = X.shape[1]
    if vector_type == "F64":
        mean = nd_sum_f64(X) / np.float64(n)
    else:
        if vector_type == "I16" and n > 32767:
            raise ValueError("A::from_usize(n) fails: the reference panics")
        sums = _wrap_sum(X).tolist()  # wrapped in T; the division in T truncates toward zero
        mean = np.array([(abs(s) // n) * (1 if s >= 0 else -1) for s in sums], X.dtype).astype(np.float64)
    d = X.astype(np.float64) - mean[:, None]
    return mean, d, _seq_sum(d * d)


def _keys(v, vector_type):
    """JACCARD keys: u64 bit patterns for F64 (jaccard_f64), the values themselves for the integers"""
    v = np.asarray(v, DTYPES[vector_type])
    return (v.view(np.uint64) if vector_type == "F64" else v).tolist()


def _jaccard(a, b, vector_type):
    """jaccard_f64 / jaccard_integers (vector.rs:316-356), literally; F64 returns 1 - inter / union"""
    union = set(_keys(a, vector_type))
    inter = 0
    for k in _keys(b, vector_type):
        if k in union:
            inter += 1
        else:
            union.add(k)
    r = float(inter) / float(len(union))
    return 1.0 - r if vector_type == "F64" else r


def distances(metric, X, q, order=3.0, vector_type="F32"):
    """calculate(X[r], q) for every row r -> f64 array"""
    if vector_type == "F32":
        return F32.distances(metric, X, q, order)
    dt = DTYPES[vector_type]
    X = np.atleast_2d(np.asarray(X, dt))
    q = np.asarray(q, dt)
    Xf, qf = X.astype(np.float64), q.astype(np.float64)
    f64, i16 = vector_type == "F64", vector_type == "I16"
    with np.errstate(all="ignore"):
        if metric == "cosine":         # 1 - dot / (na * nb); norms: 8-lane f64 sums of f64(x)^2
            if f64:
                dot = nd_sum_f64(X * q)  # unrolled_dot folds the products exactly as unrolled_fold folds values
            else:
                dot = _wrap_sum(X * q).astype(np.float64)  # wrapping products and sum in T (I16: in i16)
            na = np.sqrt(nd_sum_f64(Xf * Xf))
            nb = np.sqrt(nd_sum_f64(qf * qf)[0])
            return 1.0 - dot / (na * nb)
        if metric == "euclidean":
            if f64:                    # l2_dist: sequential f64
                d = X - q
                return np.sqrt(_seq_sum(d * d))
            if i16:                    # euclidean(): 8-lane f64 sum of exact squares
                return np.sqrt(nd_sum_f64((Xf - qf) ** 2))
            d = X - q                  # l2_dist in T, wrapping
            return np.sqrt(_seq_sum(d * d).astype(np.float64))
        if metric == "manhattan":
            if f64:
                return _seq_sum(np.abs(X - q))
            if i16:                    # (a - b) wraps in i16, then |f64|
                return _seq_sum(np.abs((X - q).astype(np.float64)))
            return _seq_sum(np.abs(X - q)).astype(np.float64)
        if metric == "chebyshev":
            if f64:                    # linf_dist: `if d > max` from 0, a NaN never wins
                return np.fmax.reduce(np.abs(X - q), axis=1, initial=0.0)
            if i16:                    # fold(0.0, f64::max)
                return np.fmax.reduce(np.abs(Xf - qf), axis=1, initial=0.0)
            return np.maximum.reduce(np.abs(X - q), axis=1, initial=0).astype(np.float64)  # abs(MIN) < 0 never wins
        if metric == "hamming":
            return (X != q).sum(axis=1).astype(np.float64)
        if metric == "minkowski":
            s = _seq_sum(np.power(np.abs(Xf - qf), float(order)))
            return np.power(s, 1.0 / float(order))
        if metric == "pearson":
            _, dx, sx2 = _pearson_state(X, vector_type)
            _, dy, sy2 = _pearson_state(q[None, :], vector_type)
            sxy = _seq_sum(dx * dy[0])
            den = np.sqrt(sx2 * sy2[0])
            return np.where(den == 0.0, 0.0, sxy / den)
        if metric == "jaccard":
            return np.array([_jaccard(x, q, vector_type) for x in X], np.float64)
    raise ValueError(f"metric {metric!r} is not restated here")


def distance(metric, a, b, order=3.0, vector_type="F32"):
    """Distance::calculate(a, b) for two vectors of the type (vector.rs:659-672)"""
    return float(distances(metric, np.asarray(a, DTYPES[vector_type])[None, :], b, order, vector_type)[0])


def search_csr(graph, q, k, ef, metric, order=3.0, truthy=None, all_docs_pending=None, vector_type="F32"):
    """-> (ids u64, dist f64, (visited, expanded)) like hnsw_metric_ref.search_csr, walked in `metric` with the
    arithmetic of `vector_type`.  all_docs_pending: unfiltered search only."""
    if vector_type == "F32":
        return F32.search_csr(graph, q, k, ef, metric, order, truthy, all_docs_pending)
    vec = np.ascontiguousarray(graph["vectors"], DTYPES[vector_type])
    q = np.asarray(q, DTYPES[vector_type])
    layers = graph["layers"]
    entry = int(graph["entry_point"])
    counters = [0, 0]
    if entry < 0 or k == 0:
        return np.zeros(0, np.uint64), np.zeros(0, np.float64), (0, 0)
    if metric == "jaccard":  # per pair, on demand
        cache = {}

        def dist(e):
            if e not in cache:
                cache[e] = _jaccard(vec[e], q, vector_type)
            return cache[e]
    else:
        all_d = distances(metric, vec, q, order, vector_type)

        def dist(e):
            return float(all_d[e])
    noexp = None if truthy is not None else all_docs_pending
    ep = entry
    ep_d = dist(ep)
    counters[0] += 1
    for l in range(len(layers) - 1, 0, -1):  # search_ep: never filtered
        w = _search_single(layers[l], dist, ep_d, ep, 1, counters, noexp)
        if len(w):
            ep_d, ep = w.first()
    w = _search_single(layers[0], dist, ep_d, ep, ef, counters, noexp, truthy)
    top = [e[2:] for e in w.e[:k]]
    return (np.array([i for _, i in top], np.uint64), np.array([d for d, _ in top], np.float64),
            (counters[0], counters[1]))
