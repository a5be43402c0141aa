"""numpy restatement of the MANHATTAN / CHEBYSHEV screen (surrealdb_b200/csrc/screen_lp.cu) and of its error bound
(cand_begin_lp_kernel in candidates.cu, DESIGN.md section 2).

  screen score   s~ = sum_i |x^_i - q^_i| (f32, any summation order) or max_i |x^_i - q^_i|, q^ / x^ the f32 copies
  reference      d = sequential f64 over the f64 values: acc + |x_i - q_i| from 0.0, or the max from f64::MIN
  bound          |s~ - d| <= beps(metric, D, max_norm, q^) for every screened row"""
import numpy as np

U = 2.0 ** -24


def f32_norm(X, metric):
    """finalize_lp_kernel's per-row norm of the f32 copy, in f64 (before the final rounding up)."""
    a = np.abs(np.asarray(X, np.float32).astype(np.float64))
    return a.sum(axis=-1) if metric == "MANHATTAN" else a.max(axis=-1)


def max_norm(X, metric):
    """the corpus figure the bound uses: the largest row norm, rounded up to f32 (f64 sums get a 2^-30 margin)."""
    v = f32_norm(X, metric).max()
    if metric == "MANHATTAN":
        v = v * (1.0 + 2.0 ** -30)
    f = np.float32(v)
    return f if np.float64(f) >= v else np.nextafter(f, np.float32(np.inf))


def beps(metric, dim, mnorm, q32):
    """per query: the bound of cand_begin_lp_kernel (before its rounding up to f32)."""
    a = np.abs(np.asarray(q32, np.float32).astype(np.float64))
    D = float(dim)
    if metric == "MANHATTAN":
        w = np.float64(mnorm) + a.sum(axis=-1) * (1.0 + 2.0 ** -30)
        return ((D + 3.0) * U * (1.0 + 2.0 * (D + 3.0) * U) + D * 2.0 ** -52) * w + D * 2.0 ** -147
    w = np.float64(mnorm) + a.max(axis=-1)
    return (3.0 * U + 2.0 ** -52) * w * (1.0 + 2.0 ** -20) + 2.0 ** -147


def terms32(Q, X):
    """[nq][n][D] f32 |x^_i - q^_i| (one correctly rounded f32 subtraction each)."""
    q = np.asarray(Q, np.float64).astype(np.float32)
    x = np.asarray(X, np.float64).astype(np.float32)
    with np.errstate(over="ignore"):
        return np.abs(x[None, :, :] - q[:, None, :])


def _pairwise(t):
    d = t.shape[-1]
    p = 1
    while p < d:
        p *= 2
    t = np.concatenate([t, np.zeros(t.shape[:-1] + (p - d,), np.float32)], axis=-1)
    while t.shape[-1] > 1:
        t = t[..., 0::2] + t[..., 1::2]
    return t[..., 0]


def _strided32(t):
    """32 lanes, lane l sums columns l, l + 32, ... sequentially, then a butterfly over the lanes."""
    d = t.shape[-1]
    pad = (-d) % 32
    t = np.concatenate([t, np.zeros(t.shape[:-1] + (pad,), np.float32)], axis=-1)
    lanes = np.cumsum(t.reshape(t.shape[:-1] + (-1, 32)), axis=-2, dtype=np.float32)[..., -1, :]
    while lanes.shape[-1] > 1:
        h = lanes.shape[-1] // 2
        lanes = lanes[..., :h] + lanes[..., h:]
    return lanes[..., 0]


def screen_sum(Q, X, metric, order):
    """[nq][n] f32 screen values s~ in one summation order: sequential, pairwise or strided32 (CHEBYSHEV: the max)."""
    t = terms32(Q, X)
    if metric == "CHEBYSHEV":
        return t.max(axis=-1)
    if order == "sequential":
        return np.cumsum(t, axis=-1, dtype=np.float32)[..., -1]
    if order == "pairwise":
        return _pairwise(t)
    return _strided32(t)


def reference(Q, X, metric):
    """[nq][n] the reference's distance: sequential f64 (Distance::compute, vector.rs)."""
    q = np.asarray(Q, np.float64)
    x = np.asarray(X, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        t = np.abs(x[None, :, :] - q[:, None, :])
    if metric == "CHEBYSHEV":
        return np.maximum(t.max(axis=-1), -np.finfo(np.float64).max)
    return np.cumsum(t, axis=-1)[..., -1]
