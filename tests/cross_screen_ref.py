"""A numpy restatement of the cross views of COSINE and EUCLIDEAN columns (DESIGN.md sections 2 and 5, "cross views"):
which score, query copy and per-row array a ranking takes (internal.cuh view_of), the cross screening norm and its
special rule (corpus.cu finalize_cross_kernel), the screens' score in exact arithmetic, the bounds beps / beps2 of
cand_begin_kernel in the view's form, and cand_final's proof bound per view."""
from dataclasses import dataclass

import numpy as np

import dot_screen_ref as D

F32_MIN_NORMAL, F32_MAX = 2.0 ** -126, 3.4028234663852886e38


@dataclass
class View:
    sc: str        # "cos" (acc / |x|), "euc" (2 acc - |x|^2) or "far" (2 acc + |x|^2)
    neg: bool      # the screen copies are those of -q
    cross: bool    # the per-row array and special list are the other metric's
    sim: bool      # a cosine view's value is the similarity (else the distance)
    desc: bool


def view(metric, fn, desc):
    """the view of (fn, order) on a column of `metric`: fn "COSINE" / "SIMILARITY_COSINE" / "EUCLIDEAN" """
    if fn == "EUCLIDEAN":
        return View("far" if desc else "euc", desc, metric != "EUCLIDEAN", False, desc)
    # cosine distance ascending and similarity descending look towards q, the other two orders towards -q
    return View("cos", (fn == "COSINE") == desc, metric != "COSINE", fn == "SIMILARITY_COSINE", desc)


def query_copies(Q, v):
    """the f32 and bf16 screen copies of q or -q, negated in f64 before any rounding"""
    return D.query_copies(Q, not v.neg)


def cross_norm(X, metric):
    """the other metric's screening norm from the exact magnitude m: fl32(fl64(m m)) on COSINE columns, fl32(1 / m) on
    EUCLIDEAN ones"""
    m = D.magnitude(X)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        return ((m * m) if metric == "COSINE" else (1.0 / m)).astype(np.float32), m


def cross_special(X, metric, f64_rows):
    """the rows the other metric's rule makes special (finalize_cross_kernel; the own special rows join them there)"""
    xn, m = cross_norm(X, metric)
    with np.errstate(over="ignore", invalid="ignore"):
        if metric == "COSINE":
            special = ~np.isfinite(m * m) | ~np.isfinite(xn)
        else:
            special = ~(m > 0) | ~np.isfinite(m)
        if f64_rows:
            mf = m.astype(np.float32).astype(np.float64)
            a = np.abs(xn.astype(np.float64))
            bad = (m < 2.0 ** -100) | ~((mf >= F32_MIN_NORMAL) & (mf <= F32_MAX)) | ~((a >= F32_MIN_NORMAL) & (a <= F32_MAX))
            special |= (m > 0) & bad
    return special


def exact_score(X, q, v):
    """what the view's screen score stands for, in f64 from exact-as-possible arithmetic: cos: x.(+-q) / |x| (similarity
    times |q|), euc: 2 x.q - |x|^2, far: |x|^2 - 2 x.q"""
    sq = np.asarray(q, np.float64) * (-1.0 if v.neg else 1.0)
    X = np.asarray(X, np.longdouble)
    dot = X @ sq.astype(np.longdouble)
    n2 = (X * X).sum(axis=1)
    if v.sc == "cos":
        return np.asarray(dot / np.sqrt(n2), np.float64)
    return np.asarray(2 * dot + (n2 if v.sc == "far" else -n2), np.float64)


def score_tolerance(v, beps, qm):
    """|screen score - exact_score| <= this: beps is in similarity units for cos, in score units otherwise"""
    return beps * qm if v.sc == "cos" else beps


def screen_score(acc, norm, v):
    """the f32 epilogue of the screens and stage B (one rounding: a product or an FMA)"""
    acc = np.asarray(acc, np.float64)
    norm = np.asarray(norm, np.float64)
    if v.sc == "cos":
        return (acc * norm).astype(np.float32).astype(np.float64)
    return (2 * acc + (norm if v.sc == "far" else -norm)).astype(np.float32).astype(np.float64)


def bounds(screen, v, Dm, qm, mn, ex=0.0, eq=0.0, f64_rows=False):
    """(beps, beps2) of cand_begin_kernel in the view's form, before the f32 rounding up: cos in similarity units
    (with the F64 rows' underflow term), euc / far in score units with max_norm mn"""
    qm = np.asarray(qm, np.float64)
    cos = v.sc == "cos"
    u_abs = Dm * 2.0 ** -26 / qm if (f64_rows and cos) else 0.0
    if screen == "TC_BF16":
        eps_rel = ex + eq + ex * eq + Dm * 4.76837158e-7 + 1e-5 + u_abs
    else:  # SIMT_F32
        eps_rel = (Dm / 16.0 + 16.0) * 1.1920929e-7
    e2_rel = (Dm + 16.0) * 5.9604645e-8 + ((5.9604644775390625e-8 + u_abs) if f64_rows else 0.0)
    if cos:
        return eps_rel + 0 * qm, e2_rel + 0 * qm
    eps = 2.0 * eps_rel * qm * mn + 4.8e-7 * (mn * mn + 2.0 * qm * mn) + 1e-30
    e2 = 2.0 * e2_rel * qm * mn + 2.4e-7 * mn * mn + 1e-30
    return eps, e2


def proof_bound(v, tau, bscale, beps, qm, Dm):
    """cand_final's bound on a non-candidate's value (the value of the ranked function): at most it (DESC) or at least
    it (ASC), one ulp outward for each directed rounding of the kernel"""
    up = lambda a: np.nextafter(np.float64(a), np.inf)  # noqa: E731
    if v.sc == "cos":
        U = up(up(up(up(np.float64(tau) * bscale) / qm) + beps) + 1e-9)
        if not v.neg:  # sim <= U, dist >= 1 - U
            return U if v.sim else np.nextafter(1.0 - U, -np.inf)
        return -U if v.sim else up(1.0 + U)  # sim >= -U, dist <= 1 + U
    if v.sc == "euc":
        L = -np.float64(tau) + qm * qm - beps
        return np.sqrt(max(L, 0.0)) * (1.0 - 1e-12)
    U = up(up(up(np.float64(tau) + beps) + up(qm * qm)) + 2.0 ** -1000)
    return up(up(np.sqrt(max(U, 0.0))) * (1.0 + (Dm + 4.0) * 2.0 ** -53))


def reference_values(fn, X, q):
    """vector::distance::cosine / ::euclidean or vector::similarity::cosine of every row, vectorised over the rows in
    the reference's sequential f64 arithmetic (dot and sums of squares left to right).  A row with a NaN element gets a
    positive NaN, a zero row's cosine the generated (negative) NaN, as the exact kernel's canon_nan."""
    X = np.asarray(X, np.float64)
    q = np.asarray(q, np.float64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if fn == "EUCLIDEAN":
            acc = np.zeros(X.shape[0])
            for i in range(X.shape[1]):
                t = X[:, i] - q[i]
                acc = acc + t * t
            v = np.sqrt(acc)
        else:
            s = D.reference_dot(X, q) / (D.magnitude(X) * D.magnitude(q[None])[0])
            v = np.array(s if fn == "SIMILARITY_COSINE" else 1.0 - s)
            nan = np.isnan(v)
            v[nan] = np.float64("nan")  # positive: a NaN element propagates
            v[nan & ~np.isnan(X).any(axis=1)] = np.frombuffer(np.uint64(0xFFF8000000000000).tobytes(), np.float64)[0]
    return v
