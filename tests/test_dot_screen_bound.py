"""The vector::dot screens' error bound (DESIGN.md section 2) against exact arithmetic, on the CPU: for every (query,
row) pair the bf16 screen's score (stage A), the f32 SIMT screen's and stage B's lie within beps / beps2 of the exact
dot with +-q, for the f32 summation orders a GPU reduction may take, on inputs chosen to stress each term of the
bound; and the reference's own f64 dot lies within eps_ref |q| of it."""
import numpy as np
import pytest

import dot_screen_ref as R


def _uniform(rng):
    return rng.standard_normal((60, 96)).astype(np.float32), rng.standard_normal((3, 96))


def _cancelling(rng):
    # pairs of nearly equal terms of opposite sign: the dot is tiny against |x||q|, the bound is relative to |x||q|
    x = rng.uniform(1, 2, (60, 128))
    x[:, 1::2] = -x[:, 0::2] * (1 + rng.uniform(-1e-6, 1e-6, (60, 64)))
    q = np.ones((3, 128)) + rng.uniform(-1e-7, 1e-7, (3, 128))
    return x.astype(np.float32), q


def _binades(rng):
    # 40 binades, alternating signs: large and small terms in one sum
    mag = np.exp2(rng.uniform(-20, 20, (60, 257))) * rng.uniform(1, 2, (60, 257))
    sign = np.where(np.arange(257) % 2 == 0, 1.0, -1.0)
    return (mag * sign).astype(np.float32), np.exp2(rng.uniform(-20, 20, (3, 257))) * sign


def _subnormal_products(rng):
    # products below 2^-126 (flushed by the tensor cores or the f32 chains) next to ordinary ones; an f32-subnormal
    # query element
    x = rng.standard_normal((60, 64)) * 2.0 ** -70
    x[:, ::3] = rng.standard_normal((60, 22))
    q = rng.standard_normal((3, 64)) * 2.0 ** -60
    q[:, 1] = 2.0 ** -140
    return x.astype(np.float32), q


def _f64_rows(rng):
    # f64 rows: their bf16 copy is rounded from f64 in one step, stage B rounds them to f32 element by element
    x = rng.standard_normal((60, 130)) * np.exp2(rng.uniform(-10, 10, (60, 1)))
    return x, rng.standard_normal((3, 130))


def _norms_16x(rng):
    # row norms spanning 16x: the bound's uniform max_norm is loose for the small rows, still valid
    x = rng.standard_normal((60, 300)) * np.exp2(rng.uniform(0, 4, (60, 1)))
    return x.astype(np.float32), rng.standard_normal((3, 300))


CASES = {"uniform": _uniform, "cancelling": _cancelling, "binades_40": _binades,
         "subnormal_products": _subnormal_products, "f64_rows": _f64_rows, "norms_16x": _norms_16x}


@pytest.mark.parametrize("desc", [True, False])
@pytest.mark.parametrize("case", list(CASES))
def test_bound_covers_every_summation_order(case, desc):
    rng = np.random.default_rng(sum(map(ord, case)) + desc)
    X, Q = CASES[case](rng)
    f64_rows = X.dtype == np.float64
    D = X.shape[1]
    mn = float(np.sqrt((np.asarray(X, np.float64) ** 2).sum(axis=1)).max()) * (1 + 2.0 ** -23)
    ex = R.row_residual(X) * (1 + 2.0 ** -20)
    qm = R.magnitude(Q)
    eq = R.qbferr(Q, desc)
    q32, qb = R.query_copies(Q, desc)
    be, be2 = R.bounds("TC_BF16", D, qm, mn, ex, eq, f64_rows)
    bs, _ = R.bounds("SIMT_F32", D, qm, mn)
    assert np.isfinite(be).all() and np.isfinite(be2).all()
    for qi in range(Q.shape[0]):
        sq = Q[qi] if desc else -Q[qi]
        exact = R.exact_dot(X, sq)
        ref = R.reference_dot(X, Q[qi])
        assert (np.abs(ref - R.exact_dot(X, Q[qi])) <= R.eps_ref(D, mn) * qm[qi]).all()
        for order in ("sequential", "pairwise", "strided32"):
            a = R.screen_sum(R.bf16_terms(X, qb[qi]), order)
            assert (np.abs(a - exact) <= be[qi]).all(), (order, float(np.abs(a - exact).max()), float(be[qi]))
            b = R.screen_sum(R.f32_terms(X, q32[qi]), order)
            assert (np.abs(b - exact) <= be2[qi]).all(), (order, float(np.abs(b - exact).max()), float(be2[qi]))
            if not f64_rows:  # the SIMT screen streams f32 rows only
                assert (np.abs(b - exact) <= bs[qi]).all()


def test_query_copies_negate_before_rounding():
    """the ASC copy is the rounding of -q: the exact negation of the DESC copy (round to nearest is symmetric), and the
    residual does not change"""
    rng = np.random.default_rng(2)
    Q = rng.standard_normal((4, 33)) * np.exp2(rng.uniform(-30, 30, (4, 33)))
    a32, ab = R.query_copies(Q, True)
    d32, db = R.query_copies(Q, False)
    assert np.array_equal(a32, -d32) and np.array_equal(ab, -db)
    assert np.array_equal(R.qbferr(Q, True), R.qbferr(Q, False))


def test_no_bound_beyond_f32_range():
    """|q| max_norm beyond f32: no finite score range, the kernel gives up (exact fallback)"""
    be, be2 = R.bounds("TC_BF16", 8, np.array([1e20, 1.0, 0.0]), 1e20)
    assert np.isinf(be[0]) and np.isinf(be2[0]) and np.isfinite(be[1]) and np.isinf(be[2])


def test_bound_is_tight_enough_to_prove():
    """on spread-out data the bound is a small fraction of the spread of the dots it has to separate (about an eighth:
    the bf16 residuals of both operands, 2^-9 each, times |q| max_norm, against a spread of |q| |x| / sqrt(D))"""
    rng = np.random.default_rng(5)
    X = rng.standard_normal((2000, 768)).astype(np.float32)
    Q = rng.standard_normal((4, 768))
    mn = float(np.sqrt((X.astype(np.float64) ** 2).sum(axis=1)).max())
    be, _ = R.bounds("TC_BF16", 768, R.magnitude(Q), mn, R.row_residual(X), R.qbferr(Q, True))
    spread = np.array([np.std(R.reference_dot(X, q)) for q in Q])
    assert (be < 0.15 * spread).all()
