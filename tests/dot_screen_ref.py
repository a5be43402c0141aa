"""A numpy restatement of the vector::dot screens (DESIGN.md section 2, "vector::dot"): the screen copies of q (DESC)
or -q (ASC), the bound beps of cand_begin_dot_kernel and stage B's beps2, the reference's sequential f64 dot and
cand_final's eps_ref, plus CPU models of the bf16 and f32 screen sums."""
from fractions import Fraction

import numpy as np

F32_MAX = 3.4028234663852886e38


def bf16(a):
    """round to nearest even to bf16 (f32 or f64 input, one rounding step), returned as f64"""
    a = np.asarray(a, np.float64)
    m, e = np.frexp(a)
    quantum = np.exp2(np.maximum(e.astype(np.float64) - 8.0, -133.0))
    with np.errstate(invalid="ignore"):
        out = np.round(a / quantum) * quantum
    return np.where(np.isfinite(a), out, a)


def query_copies(Q, desc):
    """the f32 and bf16 screen copies of +q (DESC) or -q (ASC), negated in f64 before any rounding"""
    s = np.asarray(Q, np.float64) * (1.0 if desc else -1.0)
    q32 = s.astype(np.float32)
    return q32, bf16(q32).astype(np.float32)


def magnitude(Q):
    """the reference's |q|: sequential f64 sum of squares, then sqrt"""
    Q = np.atleast_2d(np.asarray(Q, np.float64))
    acc = np.zeros(Q.shape[0])
    for i in range(Q.shape[1]):
        acc = acc + Q[:, i] * Q[:, i]
    return np.sqrt(acc)


def qbferr(Q, desc):
    """|q~ - q| / |q| of the bf16 copy actually screened, rounded up as prep_queries rounds it"""
    q32, qb = query_copies(Q, desc)
    r = np.sqrt(((q32.astype(np.float64) - qb.astype(np.float64)) ** 2).sum(axis=1))
    return r / magnitude(Q) * 1.0001 + 2.4e-7


def row_residual(X):
    """e_x: the largest |x - bf16(x)| / |x| over the rows (the corpus' bf16_rel_err, before its rounding up)"""
    X = np.asarray(X, np.float64)
    r = np.sqrt(((X - bf16(X)) ** 2).sum(axis=1))
    n = np.sqrt((X * X).sum(axis=1))
    ok = n > 0
    return float((r[ok] / n[ok]).max()) if ok.any() else 0.0


def bounds(screen, D, qm, mn, ex=0.0, eq=0.0, f64_rows=False):
    """(beps, beps2) of cand_begin_dot_kernel for queries of norm qm (array) against max_norm mn, before the f32
    rounding up; inf where the kernel gives up (no bound)"""
    qm = np.asarray(qm, np.float64)
    if screen == "TC_BF16":
        e_rel = ex + eq + ex * eq + 1.01 * D * 2.0 ** -21
    else:  # SIMT_F32
        e_rel = (D / 16.0 + 16.0) * 2.0 ** -23
    e_abs = D * 2.0 ** -120 * (1.0 + qm + mn)
    eps = e_rel * qm * mn + e_abs
    e2 = ((D + 16.0) * 2.0 ** -24 + (2.0 ** -24 if f64_rows else 0.0)) * qm * mn + e_abs
    hi = qm * mn * 1.01 + eps + 1e-30
    bad = ~(qm > 0) | ~(hi <= F32_MAX) | ~(2.1 * eps <= F32_MAX)
    return np.where(bad, np.inf, eps), np.where(bad, np.inf, e2)


def eps_ref(D, mn):
    """cand_final's bound on |reference dot - x.q| per unit of |q|"""
    return (D + 2.0) * 2.0 ** -53 * mn * (1.0 + 2.0 ** -20)


def reference_dot(X, q):
    """vector::dot as the reference computes it: sequential f64, products and sums each rounded"""
    X = np.asarray(X, np.float64)
    acc = np.zeros(X.shape[0])
    for i in range(X.shape[1]):
        acc = acc + X[:, i] * float(q[i])
    return acc


def exact_dot(X, q):
    """x.q in exact rational arithmetic, rounded to f64 at the end"""
    qf = [Fraction(float(v)) for v in q]
    return np.array([float(sum(Fraction(float(a)) * b for a, b in zip(row, qf))) for row in np.asarray(X, np.float64)])


def _f32_ftz(v):
    v = np.asarray(v, np.float64).astype(np.float32).astype(np.float64)
    return np.where(np.abs(v) < 2.0 ** -126, 0.0, v)


def screen_sum(terms, order):
    """f32 sums of the per-element products (rows x D, exact in f64), with every partial sum rounded to f32 and
    flushed below 2^-126, in one of the orders a GPU reduction may take"""
    t = np.asarray(terms, np.float64)
    if order == "sequential":
        acc = np.zeros(t.shape[0])
        for i in range(t.shape[1]):
            acc = _f32_ftz(acc + t[:, i])
        return acc
    if order == "pairwise":
        while t.shape[1] > 1:
            if t.shape[1] % 2:
                t = np.concatenate([t, np.zeros((t.shape[0], 1))], axis=1)
            t = _f32_ftz(t[:, 0::2] + t[:, 1::2])
        return t[:, 0]
    # strided32: 32 lanes each summing every 32nd term, then a butterfly
    lanes = []
    for lane in range(32):
        acc = np.zeros(t.shape[0])
        for i in range(lane, t.shape[1], 32):
            acc = _f32_ftz(acc + t[:, i])
        lanes.append(acc)
    lanes = np.stack(lanes, axis=1)
    while lanes.shape[1] > 1:
        h = lanes.shape[1] // 2
        lanes = _f32_ftz(lanes[:, :h] + lanes[:, h:])
    return lanes[:, 0]


def bf16_terms(X, qb):
    """products of the bf16 screen copies (exact in f64), flushed below 2^-126 as the tensor cores may flush them"""
    p = bf16(X) * np.asarray(qb, np.float64)[None, :]
    return np.where(np.abs(p) < 2.0 ** -126, 0.0, p)


def f32_terms(X, q32):
    """products of the f32 row copies and the f32 query, flushed below 2^-126"""
    p = np.asarray(X, np.float32).astype(np.float64) * np.asarray(q32, np.float64)[None, :]
    return np.where(np.abs(p) < 2.0 ** -126, 0.0, p)


def proof_bound(tau, beps, eref, qm, desc):
    """cand_final's bound on a non-candidate's value: at most U (DESC) or at least -U (ASC),
    U = tau + beps + eps_ref |q| (the kernel rounds each step up)"""
    U = np.float64(tau) + np.float64(beps) + eref * qm
    U = np.nextafter(np.nextafter(U, np.inf), np.inf)
    return U if desc else -U
