"""Numpy restatement of the count path (count.cu: count_hamming_kernel, count_jaccard_kernel; exactmath.cuh: the keys).

- Number equality of two elements widened to f64: same bits, or both zero (num_eq_f64).
- The keys that make it one integer compare: eq_key_f64, eq_key_f32 (f32 rows) and eq_qkey_f32 (an f64 query element
  against f32 rows; EQ_KEY_NONE when no f32 widens to it).  The widening is the host's here (payload kept, quiet bit
  set), the device's in the kernel; the keys are built so that they agree with the widening either way.
- JACCARD from counts: u_x / u_q = distinct values of the row / the query, m = values both share; inter =
  D - u_q + m, union = u_x + u_q - m (jaccard_counts; the row's distinct values through its first-occurrence bitmask).
- Selection: rows cut into contiguous ranges, each range's k smallest (count, row) pairs; their union, re-sorted by
  (count, row), starts with the global top k however many counts tie."""
import numpy as np

EQ_KEY_NONE = 0x80000000


def _bits64(x):
    return int(np.asarray(x, np.float64).view(np.uint64))


def num_eq_f64(a, b):
    return _bits64(a) == _bits64(b) or (a == 0.0 and b == 0.0)


def eq_key_f64(x):
    b = _bits64(x)
    return 0 if (b << 1) & 0xFFFFFFFFFFFFFFFF == 0 else b


def eq_key_f32(x):
    w = np.float64(np.float32(x))
    b = _bits64(w)
    if (b << 1) & 0xFFFFFFFFFFFFFFFF == 0:
        return 0
    if w != w:
        return ((b >> 32) & 0x80000000) | 0x7F800000 | ((b >> 29) & 0x7FFFFF)
    return int(np.asarray(np.float32(x)).view(np.uint32))


def eq_qkey_f32(q):
    b = _bits64(q)
    if (b << 1) & 0xFFFFFFFFFFFFFFFF == 0:
        return 0
    if q != q:
        fb = ((b >> 32) & 0x80000000) | 0x7F800000 | ((b >> 29) & 0x7FFFFF)
        f = np.asarray(np.uint32(fb)).view(np.float32)[()]
    else:
        with np.errstate(over="ignore"):
            f = np.float32(q)
    if _bits64(np.float64(f)) != b:
        return EQ_KEY_NONE
    return eq_key_f32(f)


def hamming_by_keys(row, query):
    """Mismatch count of a row (f32 or f64) against an f64 query through the keys."""
    if row.dtype == np.float64:
        return sum(eq_key_f64(x) != eq_key_f64(q) for x, q in zip(row, query))
    return sum(eq_key_f32(x) != eq_qkey_f32(q) for x, q in zip(row, query))


def hamming_by_equality(row, query):
    """The exact kernel's count: num_eq_f64 on the widened row element."""
    return sum(not num_eq_f64(np.float64(x), q) for x, q in zip(row, query))


def first_occurrence(v):
    """Bit i set when no earlier element of v equals v[i] (num_eq_f64 after the widening): finalize_jaccard_kernel."""
    keys = [eq_key_f64(np.float64(x)) for x in v]
    return [keys[i] not in keys[:i] for i in range(len(keys))]


def jaccard_by_counts(row, query):
    """(D - u_q + m) / (u_x + u_q - m) in f64, m = first-occurrence row elements whose value the query holds."""
    qset = {eq_key_f64(np.float64(x)) for x in query}
    first = first_occurrence(row)
    u_x, u_q = sum(first), len(qset)
    m = sum(1 for x, f in zip(row, first) if f and eq_key_f64(np.float64(x)) in qset)
    return np.float64(len(query) - u_q + m) / np.float64(u_x + u_q - m)


def nan_patterns(fdt):
    """NaNs of the row type with canonical, non-canonical, signalling and negative payloads, and ordinary values."""
    if fdt == np.float32:
        bits = np.array([0x7FC00000, 0xFFC00000, 0x7FC00001, 0x7F800001, 0xFF812345, 0x7FFFFFFF, 0x7FA00000,
                         0x3F800000, 0x00000000, 0x80000000], np.uint32)
        return bits.view(np.float32)
    bits = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000001, 0x7FF0000000000001,
                     0xFFF0123456789ABC, 0x7FFFFFFFFFFFFFFF, 0x7FF4000000000000, 0x3FF0000000000000, 0,
                     0x8000000000000000], np.uint64)
    return bits.view(np.float64)


def f64_nans():
    """f64 NaNs: two that widen from an f32 NaN on the host, two that no f32 widens to (low payload bits set)."""
    return np.array([0x7FF8000000000000, 0xFFF8002000000000, 0x7FF8000000000001, 0xFFF0000000000007],
                    np.uint64).view(np.float64)


def range_union_topk(dist, k, n_ranges, skip=None):
    """Per contiguous range of rows, the k smallest (dist, row) pairs; the union re-sorted by (dist, row)."""
    n = dist.size
    out = []
    for r in range(n_ranges):
        lo, hi = r * n // n_ranges, (r + 1) * n // n_ranges
        rows = [i for i in range(lo, hi) if skip is None or not skip[i]]
        rows.sort(key=lambda i: (dist[i], i))
        out += rows[:k]
    out.sort(key=lambda i: (dist[i], i))
    return out


def full_topk(dist, k, skip=None):
    rows = [i for i in range(dist.size) if skip is None or not skip[i]]
    rows.sort(key=lambda i: (dist[i], i))
    return rows[:k]
