"""Test reference for the HNSW walk in the typed F32 metrics the CPU oracle (oracle/) does not restate: MINKOWSKI,
PEARSON and JACCARD (idx/trees/vector.rs:329-451), plus EUCLIDEAN / MANHATTAN / CHEBYSHEV / HAMMING so that this module
can be checked against the oracle where both exist (tests/test_oracle_hnsw_metrics.py).

  distance(metric, a, b, order)      Distance::calculate(a, b) for two F32 vectors (JACCARD is asymmetric in a, b)
  distances(metric, X, q, order)     calculate(X[r], q) for every row: the walk's argument order (hnsw/layer.rs:207,251)
  search_csr(graph, q, k, ef, ...)   Hnsw::knn_search / knn_search_with_filter over an exported graph, restated from
                                     HnswLayer::search (layer.rs:184-223), search_with_filter / add_if_truthy (:226-306),
                                     search_single[_with_filter] (:76-149) and search_ep (mod.rs:521-548), with the
                                     DoublePriorityQueue of idx/trees/knn.rs:15-123 and the same two visit counters as
                                     oracle/pyoracle.hnsw_search_csr: (distance evaluations, expanded nodes)

Plain numpy: every sequential fold of the reference is an `add.accumulate` (numpy's cumsum is a strict left-to-right
fold in the array's dtype), never a pairwise `sum`.
"""
import bisect
import struct

import numpy as np

F64_MAX = 1.7976931348623157e308


# ---------------------------------------------------------------- typed F32 metrics (vector.rs:218-451)
def _seq_sum(t):
    """sequential fold along the last axis, in t's dtype"""
    if t.shape[-1] == 0:
        return np.zeros(t.shape[:-1], t.dtype)
    return np.cumsum(t, axis=-1, dtype=t.dtype)[..., -1]


def nd_sum_f32(X):
    """ArrayBase::sum of contiguous f32 rows: ndarray's unrolled_fold -- 8 partial sums p_j over the columns 8i+j,
    sum = 0 + (p0+p4) + (p1+p5) + (p2+p6) + (p3+p7), then the < 8 tail columns in order.  PARITY UNPINNED like the
    oracle's orc_nd_dot_f32 / orc_nd_sumsq_f32 (the crate is not vendored, DESIGN section 3): isolated here."""
    X = np.atleast_2d(np.asarray(X, np.float32))
    rows, dim = X.shape
    n8 = dim // 8 * 8
    if n8:
        p = _seq_sum(np.ascontiguousarray(X[:, :n8].reshape(rows, -1, 8).transpose(0, 2, 1)))  # (rows, 8)
    else:
        p = np.zeros((rows, 8), np.float32)
    s = np.zeros(rows, np.float32)
    for j in range(4):
        s = (s + (p[:, j] + p[:, j + 4])).astype(np.float32)
    for c in range(n8, dim):
        s = (s + X[:, c]).astype(np.float32)
    return s


def _pearson_state(X):
    """per row: mean (ndarray mean() = sum / n as f32, widened) and the sequential f64 sum of (x_i - mean)^2"""
    X = np.atleast_2d(np.asarray(X, np.float32))
    mean = (nd_sum_f32(X) / np.float32(X.shape[1])).astype(np.float32).astype(np.float64)
    d = X.astype(np.float64) - mean[:, None]
    return mean, d, _seq_sum(d * d)


def _jaccard(a, b):
    """jaccard_f32 (vector.rs:329-340), literally: union = HashSet of a's bit patterns; every b_i whose pattern is
    already in the set counts (insert returns false), the others are inserted.  count / union.len(), a similarity."""
    union = set(np.asarray(a, np.float32).view(np.uint32).tolist())
    inter = 0
    for bits in np.asarray(b, np.float32).view(np.uint32).tolist():
        if bits in union:
            inter += 1
        else:
            union.add(bits)
    return float(inter) / float(len(union))


def distances(metric, X, q, order=3.0):
    """calculate(X[r], q) for every row r -> f64 array"""
    X = np.atleast_2d(np.asarray(X, np.float32))
    q = np.asarray(q, np.float32)
    with np.errstate(all="ignore"):
        if metric == "euclidean":      # ndarray-stats l2_dist: f32 sum of squares, f64 sqrt
            d = (X - q).astype(np.float32)
            return np.sqrt(_seq_sum((d * d).astype(np.float32)).astype(np.float64))
        if metric == "manhattan":      # l1_dist: f32 sum of |a - b|, then as f64
            return _seq_sum(np.abs((X - q).astype(np.float32))).astype(np.float64)
        if metric == "chebyshev":      # linf_dist: max from 0, `if d > max` (a NaN never wins)
            return np.fmax.reduce(np.abs((X - q).astype(np.float32)), axis=1, initial=np.float32(0)).astype(np.float64)
        if metric == "hamming":        # count of a_i != b_i under f32 != (NaN != NaN, 0.0 == -0.0)
            return (X != q).sum(axis=1).astype(np.float64)
        if metric == "minkowski":      # f64 sum of |a_i - b_i|^p, then ^(1/p)
            s = _seq_sum(np.power(np.abs(X.astype(np.float64) - q.astype(np.float64)), float(order)))
            return np.power(s, 1.0 / float(order))
        if metric == "pearson":        # sxy / sqrt(sx2 * sy2), 0.0 when that is 0 (x = a, y = b)
            _, dx, sx2 = _pearson_state(X)
            _, dy, sy2 = _pearson_state(q[None, :])
            sxy = _seq_sum(dx * dy[0])
            den = np.sqrt(sx2 * sy2[0])
            return np.where(den == 0.0, 0.0, sxy / den)
        if metric == "jaccard":
            return np.array([_jaccard(x, q) for x in X], np.float64)
    raise ValueError(f"metric {metric!r} is not restated here")


def distance(metric, a, b, order=3.0):
    """Distance::calculate(a, b) for two F32 vectors (vector.rs:659-672)"""
    return float(distances(metric, np.asarray(a, np.float32)[None, :], b, order)[0])


# ---------------------------------------------------------------- the walk
def _total_key(d):
    """f64::total_cmp as a signed integer key (FloatKey of the queues)"""
    b = struct.unpack("<q", struct.pack("<d", d))[0]
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


class _Dpq:
    """DoublePriorityQueue (idx/trees/knn.rs:15-123): BTreeMap<FloatKey, VecDeque<id>>.  pop_first = smallest key,
    oldest id; pop_last = largest key, newest id."""

    def __init__(self):
        self.e, self.seq = [], 0

    def push(self, d, i):
        bisect.insort(self.e, (_total_key(d), self.seq, d, i))
        self.seq += 1

    def pop_first(self):
        return self.e.pop(0)[2:]

    def pop_last(self):
        self.e.pop()

    def last_dist(self):
        return self.e[-1][2]

    def first(self):
        return self.e[0][2:]

    def __len__(self):
        return len(self.e)


def _layer_search(adj, dist, cand, visited, w, ef, counters, noexp=None, truthy=None):
    """HnswLayer::search (truthy None) / search_with_filter + add_if_truthy"""
    rp, ci = adj
    fq = w.last_dist() if len(w) else F64_MAX
    while len(cand):
        cd, c = cand.pop_first()
        if cd > fq:
            break
        counters[1] += 1
        for e in ci[int(rp[c]):int(rp[c + 1])].tolist():
            if e in visited:
                continue
            visited.add(e)
            ed = dist(e)
            counters[0] += 1
            if ed < fq or len(w) < ef:
                if truthy is None:
                    if noexp is None or not noexp[e]:  # layer.rs:209: enters w, never expanded
                        cand.push(ed, e)
                    w.push(ed, e)
                    if len(w) > ef:
                        w.pop_last()
                    fq = w.last_dist() if len(w) else F64_MAX
                else:
                    cand.push(ed, e)
                    if truthy[e]:
                        w.push(ed, e)
                        if len(w) > ef:
                            w.pop_last()
                        fq = w.last_dist()


def _search_single(adj, dist, ep_d, ep, ef, counters, noexp=None, truthy=None):
    cand, w = _Dpq(), _Dpq()
    cand.push(ep_d, ep)
    if truthy is None or truthy[ep]:
        w.push(ep_d, ep)
    _layer_search(adj, dist, cand, {ep}, w, ef, counters, noexp, truthy)
    return w


def search_csr(graph, q, k, ef, metric, order=3.0, truthy=None, all_docs_pending=None):
    """-> (ids u64, dist f64, (visited, expanded)) like oracle/pyoracle.hnsw_search_csr, in `metric` (the graph's own
    "metric" entry is ignored: any graph can be walked in any metric).  all_docs_pending: unfiltered search only."""
    vec = np.ascontiguousarray(graph["vectors"], np.float32)
    layers = graph["layers"]
    entry = int(graph["entry_point"])
    counters = [0, 0]
    if entry < 0 or k == 0:
        return np.zeros(0, np.uint64), np.zeros(0, np.float64), (0, 0)
    if metric == "jaccard":  # per pair, on demand
        cache = {}

        def dist(e):
            if e not in cache:
                cache[e] = _jaccard(vec[e], q)
            return cache[e]
    else:
        all_d = distances(metric, vec, q, order)

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
