"""The cross views' error bounds (DESIGN.md section 2) against exact arithmetic, on the CPU: for every (query, row)
pair and every view, the bf16 screen's score (stage A) and stage B's f32 score, each with the view's per-row array and
epilogue, lie within beps / beps2 of what the score stands for, for the f32 summation orders a GPU reduction may take,
on inputs chosen to stress each term of the bound; the cross screening norm |x|^2 = fl32(m m) stays inside the room
the euclidean bounds give it; and the cross special rule catches zero rows and f64 rows with a non-normal cross norm."""
from fractions import Fraction

import numpy as np
import pytest

import cross_screen_ref as X
import dot_screen_ref as D
from test_dot_screen_bound import CASES

PAIRS = [("COSINE", "COSINE", True), ("COSINE", "SIMILARITY_COSINE", False), ("COSINE", "EUCLIDEAN", False),
         ("COSINE", "EUCLIDEAN", True), ("EUCLIDEAN", "EUCLIDEAN", True), ("EUCLIDEAN", "COSINE", False),
         ("EUCLIDEAN", "SIMILARITY_COSINE", True), ("EUCLIDEAN", "COSINE", True),
         ("EUCLIDEAN", "SIMILARITY_COSINE", False)]


def _norms(X64, metric, v):
    """the per-row array the view reads: the own screening norm or the cross one"""
    m = D.magnitude(X64)
    s = np.zeros(X64.shape[0])
    for i in range(X64.shape[1]):
        s = s + X64[:, i] * X64[:, i]
    own_cos = metric == "COSINE"
    if v.cross:
        return X.cross_norm(X64, metric)[0].astype(np.float64)
    if own_cos:
        return (1.0 / m).astype(np.float32).astype(np.float64)
    return s.astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{p[0]}-{p[1]}-{'DESC' if p[2] else 'ASC'}")
@pytest.mark.parametrize("case", list(CASES))
def test_bound_covers_every_summation_order(case, pair):
    metric, fn, desc = pair
    v = X.view(metric, fn, desc)
    rng = np.random.default_rng(sum(map(ord, case + fn + metric)) + desc)
    Xr, Q = CASES[case](rng)
    f64_rows = Xr.dtype == np.float64
    X64 = np.asarray(Xr, np.float64)
    keep = ~X.cross_special(X64, metric, f64_rows) & (D.magnitude(X64) > 0)
    X64, Xr = X64[keep], Xr[keep]
    Dm = Xr.shape[1]
    mn = float(np.sqrt((X64 ** 2).sum(axis=1)).max()) * (1 + 2.0 ** -23)
    ex = D.row_residual(Xr) * (1 + 2.0 ** -20)
    qm = D.magnitude(Q)
    q32, qb = X.query_copies(Q, v)
    eq = D.qbferr(Q, not v.neg)
    be, be2 = X.bounds("TC_BF16", v, Dm, qm, mn, ex, eq, f64_rows)
    norm = _norms(X64, metric, v)
    for qi in range(Q.shape[0]):
        exact = X.exact_score(X64, Q[qi], v)
        for order in ("sequential", "pairwise", "strided32"):
            a = X.screen_score(D.screen_sum(D.bf16_terms(Xr, qb[qi]), order), norm, v)
            err = np.abs(a - exact)
            assert (err <= X.score_tolerance(v, be[qi], qm[qi])).all(), (order, float(err.max()))
            b = X.screen_score(D.screen_sum(D.f32_terms(Xr, q32[qi]), order), norm, v)
            err = np.abs(b - exact)
            assert (err <= X.score_tolerance(v, be2[qi], qm[qi])).all(), (order, float(err.max()))


@pytest.mark.parametrize("case", list(CASES))
def test_cross_square_norm_gap(case):
    """fl32(fl64(m m)), m = fl64(sqrt(s)) with s the reference's sequential f64 sum of squares, is within
    2^-24 + 4 2^-53 of the real sum of squares relatively (the (D + 2) 2^-53 of s itself aside) -- inside the 8 2^-24
    and 4 2^-24 of |x|^2 that stage A's and stage B's euclidean bounds give the screening norm.  Some rows' fl32(m m)
    differ from fl32(s)."""
    rng = np.random.default_rng(sum(map(ord, case)))
    Xr, _ = CASES[case](rng)
    X64 = np.asarray(Xr, np.float64)
    xn, m = X.cross_norm(X64, "COSINE")
    s = np.zeros(X64.shape[0])
    for i in range(X64.shape[1]):
        s = s + X64[:, i] * X64[:, i]
    ok = (m > 0) & ~X.cross_special(X64, "COSINE", Xr.dtype == np.float64)
    real = np.array([float(sum(Fraction(float(a)) ** 2 for a in row)) for row in X64[ok]])
    gap = np.abs(xn[ok].astype(np.float64) - real) / real
    Dm = X64.shape[1]
    assert (gap <= 2.0 ** -24 + (Dm + 6.0) * 2.0 ** -53).all()
    assert (gap <= 4 * 2.0 ** -24).all()


def test_square_of_the_magnitude_is_not_the_sum_of_squares():
    rng = np.random.default_rng(3)
    X64 = rng.standard_normal((4000, 33)) * np.exp2(rng.uniform(-8, 8, (4000, 1)))
    _, m = X.cross_norm(X64, "COSINE")
    s = np.zeros(X64.shape[0])
    for i in range(X64.shape[1]):
        s = s + X64[:, i] * X64[:, i]
    assert (m * m != s).mean() > 0.1  # fl64(m m) is not the stored sum: the gap test above covers those rows


def test_cross_special_rows():
    """zero rows are special for the cosine views of a EUCLIDEAN column (their cosine is a generated NaN); an f64 row
    of a COSINE column whose |x|^2 is below the normal f32 range, or beyond it, is special for its euclidean views; an
    ordinary row is neither"""
    rng = np.random.default_rng(9)
    x = rng.standard_normal((6, 20))
    x[1] = 0.0
    x[2] *= 2.0 ** -75      # |x|^2 ~ 2^-146: subnormal in f32, |x| itself normal and above 2^-100
    x[3] *= 2.0 ** 70       # |x|^2 ~ 2^142: beyond f32
    x[4, 0] = np.inf
    eu = X.cross_special(x, "EUCLIDEAN", True)
    co = X.cross_special(x, "COSINE", True)
    assert eu[1] and eu[4] and not eu[0] and not eu[2] and not eu[3]
    assert co[2] and co[3] and co[4] and not co[0]
    assert X.cross_special(x.astype(np.float32), "EUCLIDEAN", False)[1]


def test_views():
    """the (fn, order) pairs and their query sign, score and per-row array"""
    v = X.view("COSINE", "COSINE", True)
    assert (v.sc, v.neg, v.cross, v.sim) == ("cos", True, False, False)
    v = X.view("COSINE", "SIMILARITY_COSINE", False)
    assert (v.sc, v.neg, v.cross, v.sim) == ("cos", True, False, True)
    v = X.view("COSINE", "EUCLIDEAN", True)
    assert (v.sc, v.neg, v.cross) == ("far", True, True)
    v = X.view("EUCLIDEAN", "EUCLIDEAN", True)
    assert (v.sc, v.neg, v.cross) == ("far", True, False)
    v = X.view("EUCLIDEAN", "SIMILARITY_COSINE", True)
    assert (v.sc, v.neg, v.cross, v.sim) == ("cos", False, True, True)
    v = X.view("EUCLIDEAN", "COSINE", True)
    assert (v.sc, v.neg, v.cross, v.sim) == ("cos", True, True, False)


def test_farthest_first_proof_bound():
    """the EuclidFar bound: every row whose screened score is below tau has a reference distance at most the bound,
    computed from exact arithmetic on random rows"""
    rng = np.random.default_rng(21)
    Xr = rng.standard_normal((500, 64))
    q = rng.standard_normal(64)
    v = X.view("EUCLIDEAN", "EUCLIDEAN", True)
    exact = X.exact_score(Xr, q, v)                 # d^2 - |q|^2
    qm = float(D.magnitude(q[None])[0])
    tau, beps = float(np.median(exact)), 1e-3
    below = exact < tau - beps                      # a screened score below tau at most beps from the exact one
    d_ref = np.sqrt(((Xr - q) ** 2).sum(axis=1))
    assert (d_ref[below] <= X.proof_bound(v, tau, 1.0, beps, qm, 64)).all()
