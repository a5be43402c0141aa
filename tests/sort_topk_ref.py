"""Reference of `ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k` for the GPU tests: each row's value from the CPU
oracle's Number-domain functions, ranked by a restatement of the reference's SortTopK (exec/operators/sort/topk.rs:
a heap of the `limit` best keyed rows, compare_keys then the insertion sequence, so earlier rows win ties; a row equal
to the worst of a full heap is not taken).  Number::cmp on floats is total_cmp with -0.0 == 0.0 (val/number.rs)."""
import heapq
import struct

import numpy as np

from oracle import pyoracle

# sdb_metric ids and sdb_vector_fn ids -> the oracle's Number-domain function names
FN_NAMES = {0: "chebyshev", 1: "cosine_distance", 2: "euclidean", 3: "hamming", 4: "jaccard", 5: "manhattan",
            6: "minkowski", 7: "pearson", 16: "cosine_similarity", 17: "dot", 18: "magnitude"}
FN_IDS = {"CHEBYSHEV": 0, "COSINE": 1, "EUCLIDEAN": 2, "HAMMING": 3, "JACCARD": 4, "MANHATTAN": 5, "MINKOWSKI": 6,
          "PEARSON": 7, "SIMILARITY_COSINE": 16, "DOT": 17, "MAGNITUDE": 18}


def num_key(v):
    """an integer key whose order is Number::cmp on a float: total_cmp with -0.0 folded onto 0.0"""
    b = struct.unpack("<Q", struct.pack("<d", float(v)))[0]
    if (b << 1) & 0xFFFFFFFFFFFFFFFF == 0:
        b = 0
    return (~b & 0xFFFFFFFFFFFFFFFF) if b >> 63 else (b | (1 << 63))


def key_cmp(a, b):
    ka, kb = num_key(a), num_key(b)
    return (ka > kb) - (ka < kb)


class _Entry:
    """a heap entry whose `<` means "worse": the heap's top is the worst kept row (topk.rs KeyedValue::cmp)"""
    __slots__ = ("v", "seq", "cmp", "desc")

    def __init__(self, v, seq, cmp, desc):
        self.v, self.seq, self.cmp, self.desc = v, seq, cmp, desc

    def better(self, other):  # compare_keys(self, other) == Less
        c = self.cmp(self.v, other.v)
        return (c > 0) if self.desc else (c < 0)

    def __lt__(self, other):  # self is worse than other
        if other.better(self):
            return True
        if self.better(other):
            return False
        return self.seq > other.seq


def sort_topk(values, k, desc, passes=None, cmp=pyoracle.num_cmp):
    """SortTopK over values[i] (scan position i).  passes: bool per row (None: every row).  cmp: a three-way Number
    comparison (default: the oracle's orc_num_cmp).  -> (rows, values) best first."""
    heap = []
    for i, v in enumerate(values):
        if passes is not None and not passes[i]:
            continue
        e = _Entry(v, i, cmp, desc)
        if len(heap) >= k:
            if heap and e.better(heap[0]):
                heapq.heapreplace(heap, e)
        else:
            heapq.heappush(heap, e)
    out = []
    while heap:
        out.append(heapq.heappop(heap))
    out.reverse()
    return np.array([e.seq for e in out], np.uint64), np.array([e.v for e in out], np.float64)


def sort_keyed(values, k, desc, passes=None):
    """sort_topk by a plain sort on (Number::cmp key, reversed for DESC, scan position): the same result
    (tests/test_oracle_sort_topk.py), fast enough for whole columns"""
    v = np.asarray(values, np.float64)
    idx = np.arange(v.size) if passes is None else np.flatnonzero(passes)
    keys = [num_key(x) for x in v[idx]]
    order = sorted(range(idx.size), key=lambda j: ((-keys[j]) if desc else keys[j], int(idx[j])))[:k]
    rows = idx[order].astype(np.uint64)
    return rows, v[rows.astype(np.int64)]


def row_values(fn, rows, query, minkowski_p=3.0):
    """the oracle's value of vector function fn (id) for every row (rows widened to f64 as Number::Float)"""
    name = FN_NAMES[fn]
    out = np.empty(len(rows), np.float64)
    q = [float(x) for x in query] if query is not None else None
    for i, r in enumerate(np.asarray(rows, np.float64)):
        r = [float(x) for x in r]
        if name == "magnitude":
            out[i] = pyoracle.num_magnitude(r)
        else:
            st, v = pyoracle.num_metric(name, r, q, p=minkowski_p)
            assert st == 0, (name, st)
            out[i] = v
    return out
