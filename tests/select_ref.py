"""Test reference for the last selection stages of the brute-force path, in numpy:

  num_key(d)                    dist_key (internal.cuh): Number::cmp on floats (val/number.rs:620-633) as a u64 --
                                -0.0 equals 0.0, f64::total_cmp otherwise.  A generated NaN (negative) sorts first,
                                a data NaN (positive) last.
  topk(values, k, skip)         the k smallest (num_key, row) of one query's values: what the exact kernel's radix
                                select returns (rows, and the values themselves, so -0.0 stays -0.0)
  merge(rows, dist, counts, k)  sdb_topk_merge_device: the first min(count, k) entries of every list, ordered by
                                (num_key, row), the first k of them

topk is O(n) (np.partition finds the k-th key, its ties are taken in row order), so it serves corpora of 17M rows.
"""
import numpy as np

SIGN = np.uint64(1 << 63)


def num_key(d):
    """dist_key of every element of d (float64 array or scalar) -> uint64 array"""
    b = np.atleast_1d(np.asarray(d, np.float64)).view(np.uint64).copy()
    b[(b << np.uint64(1)) == 0] = 0  # -0.0 -> 0.0
    neg = (b & SIGN) != 0
    return np.where(neg, ~b, b | SIGN)


def topk(values, k, skip=None):
    """-> (rows int64, values f64): the min(k, #valid) smallest rows by (num_key, row); skip: truthy = excluded"""
    values = np.asarray(values, np.float64)
    keys = num_key(values)
    rows = np.arange(values.size, dtype=np.int64)
    if skip is not None:
        valid = np.asarray(skip) == 0
        rows, keys = rows[valid], keys[valid]
    k = min(int(k), rows.size)
    if k == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.float64)
    kth = np.partition(keys, k - 1)[k - 1]
    below = keys < kth
    lo_rows = rows[below][np.argsort(keys[below], kind="stable")]  # rows ascend, so ties stay in row order
    ties = rows[keys == kth][: k - lo_rows.size]
    out = np.concatenate([lo_rows, ties])
    return out, values[out]


def merge(rows, dist, counts, k):
    """rows / dist: (n_lists, nq, k) per-list results, counts: (n_lists, nq) -> (rows u64 (nq, k), dist f64 (nq, k),
    count u32 (nq,)); entries past a query's count are left 0"""
    rows = np.asarray(rows, np.uint64)
    dist = np.asarray(dist, np.float64)
    counts = np.asarray(counts)
    n_lists, nq = counts.shape
    out_rows = np.zeros((nq, k), np.uint64)
    out_dist = np.zeros((nq, k), np.float64)
    out_cnt = np.zeros(nq, np.uint32)
    for q in range(nq):
        r = np.concatenate([rows[l, q, : min(int(counts[l, q]), k)] for l in range(n_lists)])
        d = np.concatenate([dist[l, q, : min(int(counts[l, q]), k)] for l in range(n_lists)])
        order = np.lexsort((r, num_key(d)))[:k]
        out_rows[q, : order.size] = r[order]
        out_dist[q, : order.size] = d[order]
        out_cnt[q] = order.size
    return out_rows, out_dist, out_cnt
