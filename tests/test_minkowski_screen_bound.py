"""CPU checks of the MINKOWSKI screen's error bound (cand_begin_minkowski_kernel, DESIGN.md section 2) against a numpy
restatement of the screen's arithmetic (tests/minkowski_screen_ref.py): the launch's scale, the f32 subtraction, the
multiplication chain and its FFMA, in three summation orders, for every screened order 1 .. 8."""
import numpy as np
import pytest

import minkowski_screen_ref as R

ORDERS = list(range(1, 9))
SUMS = ["sequential", "pairwise", "strided32"]


def _case(name, rng):
    """(rows, queries) of one adversarial family"""
    if name == "uniform_d100":
        return rng.uniform(-1, 1, (40, 100)), rng.uniform(-1, 1, (3, 100))
    if name == "binades_d65":  # elements spanning 40 binades, both signs
        sg = np.where(np.arange(65) % 2, -1.0, 1.0)
        return (np.exp2(rng.uniform(-20, 20, (40, 65))) * sg, np.exp2(rng.uniform(-20, 20, (3, 65))) * sg[::-1])
    if name == "rounding_up_d1025":  # a first term of 1, then terms just above half an ulp of the sum
        return R.rounding_up_rows(6, 1025).astype(np.float64), np.zeros((2, 1025))
    if name == "underflow_d256":  # terms below 2^-126 under the scale that one row of 1 sets
        X = rng.uniform(1e-6, 1e-4, (40, 256)) * np.where(rng.random((40, 256)) < 0.5, -1.0, 1.0)
        X[0, 0] = 1.0
        return X, rng.uniform(-1e-5, 1e-5, (3, 256))
    if name == "overflow_d64":  # (2e5)^8 overflows f32 without the scale
        return rng.uniform(-2e5, 2e5, (40, 64)), rng.uniform(-2e5, 2e5, (3, 64))
    if name == "subnormal_queries_d1024":  # f64 queries 0.49 ulp off f32's subnormal grid, rows on it
        return subnormal_rows_and_queries(rng, 40, 1024)
    if name == "subnormal_f64_rows_d256":  # f64 rows off f32's subnormal grid (F64 columns round them while staging)
        X = (rng.integers(500, 520, (40, 256)) + rng.uniform(-0.49, 0.49, (40, 256))) * 2.0 ** -149
        return X, rng.integers(500, 520, (3, 256)) * 2.0 ** -149
    raise KeyError(name)


def subnormal_rows_and_queries(rng, n, dim):
    """rows q^ + k 2^-149 (k in -2 .. 2) on f32's subnormal grid, queries q = q^ + 0.49 2^-149 (f64; their f32 copy
    is q^): every element of the query moves by almost 2^-150 when it is rounded to f32, whatever the scale"""
    base = 1000 * 2.0 ** -149
    X = base + rng.integers(-2, 3, (n, dim)) * 2.0 ** -149
    Q = np.full((3, dim), base + 0.49 * 2.0 ** -149)
    Q[1] = base - 0.49 * 2.0 ** -149
    return X, Q


CASES = ["uniform_d100", "binades_d65", "rounding_up_d1025", "underflow_d256", "overflow_d64",
         "subnormal_queries_d1024", "subnormal_f64_rows_d256"]
F64_ROWS = {"subnormal_f64_rows_d256"}  # the reference reads the f64 rows, the screen their f32 copies


def _errors(X, Q, p, order, underflow=True, scale=True, subnormal_rounding=True, rows64=False):
    """(|n~ - d|, beps) per (query, row) for rows X (f32, or f64 with rows64) and f64 queries Q"""
    X32 = np.asarray(X, np.float64).astype(np.float32)
    q32 = np.asarray(Q, np.float64).astype(np.float32)
    m = R.max_abs(X32)
    e = R.batch_exponent(m, q32)
    S = R.power_sum(Q, X32, p, e, order, scale=scale)
    n = R.score_norm(S, p, e if scale else 0).astype(np.float64)
    d = R.reference(Q, np.asarray(X, np.float64) if rows64 else X32, p)
    with np.errstate(invalid="ignore"):
        err = np.abs(n - d)
    return err, R.beps(p, X32.shape[1], m, q32, e, underflow, subnormal_rounding)[:, None]


@pytest.mark.parametrize("summation", SUMS)
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("p", ORDERS)
def test_bound_holds(p, case, summation):
    rng = np.random.default_rng(1000 * p + CASES.index(case))
    X, Q = _case(case, rng)
    err, eps = _errors(X, Q, p, summation, rows64=case in F64_ROWS)
    assert np.isfinite(err).all()
    assert (err <= eps).all(), f"max err / beps = {(err / eps).max():.3g}"


def test_scale_keeps_every_term_at_most_one():
    rng = np.random.default_rng(7)
    for X, Q in (_case("overflow_d64", rng), _case("binades_d65", rng)):
        X32, q32 = X.astype(np.float32), Q.astype(np.float32)
        e = R.batch_exponent(R.max_abs(X32), q32)
        a, b = R.terms(Q, X32, 1, e)
        assert np.abs(a).max() <= 1.0


def test_rounding_up_row_rounds_up_at_every_step():
    # the p = 1 sum of the rounding-up row gains a full ulp at every step: its error is about (D - 1) u / 2 of the sum
    X = R.rounding_up_rows(1, 1025).astype(np.float64)
    Q = np.zeros((1, 1025))
    e = R.batch_exponent(R.max_abs(X.astype(np.float32)), Q.astype(np.float32))
    S = float(R.power_sum(Q, X.astype(np.float32), 1, e)[0, 0])
    exact = (1.0 + 1024 * 2.0 ** -24 * (1 + 2.0 ** -10)) * 2.0 ** -e
    assert S - exact > 1000 * 2.0 ** -25 * 2.0 ** -e


# ---- mutants: each variant of the screen or of its bound fails a case ---------------------------------------------
def test_mutant_without_the_underflow_terms_fails():
    # under the scale of a row of 1, elements of 2^-24 .. 2^-19.5 have 8th powers below 2^-149: their FFMAs add nothing
    # to the f32 power sum, a loss that only the underflow terms of the bound cover
    rng = np.random.default_rng(11)
    worst = 0.0
    for _ in range(3):
        X = np.exp2(rng.uniform(-24, -19.5, (200, 32)))
        X[0, 0] = 1.0
        Q = np.zeros((1, 32))
        err, eps = _errors(X, Q, 8, "sequential", underflow=True)
        assert (err <= eps).all()
        err, eps = _errors(X, Q, 8, "sequential", underflow=False)
        worst = max(worst, float((err / eps).max()))
    assert worst > 1.0, worst


def test_mutant_without_the_scale_overflows():
    rng = np.random.default_rng(12)
    X, Q = _case("overflow_d64", rng)
    err, eps = _errors(X, Q, 8, "sequential", scale=False)
    assert not (err <= eps).all()


@pytest.mark.parametrize("p", [1, 2, 3])
def test_mutant_without_the_subnormal_rounding_term_fails(p):
    # an f64 query 0.49 ulp off f32's subnormal grid in every element: its f32 copy is off by D^(1/p) 0.49 2^-149 in
    # p-norm, an absolute error that the scale does not shrink and that only the unscaled R 2^-149 covers
    rng = np.random.default_rng(13 + p)
    X, Q = subnormal_rows_and_queries(rng, 40, 1024)
    err, eps = _errors(X, Q, p, "sequential")
    assert (err <= eps).all()
    err, eps = _errors(X, Q, p, "sequential", subnormal_rounding=False)
    assert (err / eps).max() > 1.0, (err / eps).max()
