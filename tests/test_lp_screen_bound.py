"""The MANHATTAN / CHEBYSHEV screen's error bound (DESIGN.md section 2) against the reference's distance, on the CPU:
|s~ - d| <= beps for every (query, row) pair, for the f32 summation orders a GPU reduction may take (sequential,
pairwise, 32 lanes strided then a butterfly), on inputs chosen to stress each term of the bound."""
import numpy as np
import pytest

import lp_screen_ref as R


def _uniform(rng):
    X = rng.uniform(-1, 1, (300, 96)).astype(np.float32)
    return X, rng.uniform(-1, 1, (6, 96))


def _binades(rng):
    # 40 binades, alternating signs: large and small terms in one sum
    mag = np.exp2(rng.uniform(-20, 20, (300, 257))) * rng.uniform(1, 2, (300, 257))
    sign = np.where(np.arange(257) % 2 == 0, 1.0, -1.0)
    X = (mag * sign).astype(np.float32)
    Q = np.exp2(rng.uniform(-20, 20, (6, 257))) * sign
    return X, Q


def _subnormal(rng):
    # f32-subnormal elements in rows and queries: the rounding of q and of f64 rows is absolute there
    X = (rng.uniform(-1, 1, (300, 64)) * 2.0 ** -130).astype(np.float64)
    X[:, ::5] = rng.uniform(-1, 1, (300, 13)) * 2.0 ** -140
    Q = rng.uniform(-1, 1, (6, 64)) * 2.0 ** -131
    return X, Q


def _near_f32_max(rng):
    # f64 rows with an element just inside the f32 range (finalize makes rows beyond it special); sums that stay
    # below f32 max (a larger W is not a finite f32: cand_begin_lp_kernel then gives up and the exact kernel ranks)
    X = rng.uniform(-1, 1, (200, 3)) * 1e30
    X[:, 0] = 3.4028234663852886e38 * rng.choice([-1.0, 1.0], 200) * rng.uniform(0.99, 0.999, 200)
    Q = rng.uniform(-1, 1, (4, 3)) * 1e30
    return X, Q


def _one_ulp(rng):
    # rows that differ from the query by one ulp (f32 and f64 ulps): d is tiny, the bound still covers it
    Q = rng.uniform(-1, 1, (4, 768))
    q32 = Q.astype(np.float32)
    X = np.concatenate([np.nextafter(q32, np.float32(np.inf)).astype(np.float64),
                        np.nextafter(Q, np.inf), Q, q32.astype(np.float64)])
    return X, Q


def _f64_rows(rng):
    X = rng.uniform(-1e3, 1e3, (300, 130))
    return X, rng.uniform(-1e3, 1e3, (6, 130))


def _rounding_up(rng):
    # one 1.0 then terms just above half an ulp of the running sum: a sequential f32 sum rounds up at every step and
    # gathers almost (D - 1) 2^-24 of error -- the accumulation term of the bound is nearly reached
    X = np.full((8, 1025), 2.0 ** -24 * (1 + 2.0 ** -10), np.float32)
    X[:, 0] = 1.0
    X[4:] *= -1
    return X, np.zeros((3, 1025))


CASES = {"rounding_up": _rounding_up, "uniform": _uniform, "binades_40": _binades, "f32_subnormal": _subnormal, "f64_near_f32_max": _near_f32_max,
         "one_ulp": _one_ulp, "f64_rows": _f64_rows}


@pytest.mark.parametrize("metric", ["MANHATTAN", "CHEBYSHEV"])
@pytest.mark.parametrize("case", list(CASES))
def test_bound_covers_every_summation_order(metric, case):
    rng = np.random.default_rng(sum(map(ord, case + metric)))
    X, Q = CASES[case](rng)
    assert np.isfinite(np.asarray(X, np.float32)).all()  # every row is screenable (not special)
    mnorm = R.max_norm(X, metric)
    eps = R.beps(metric, X.shape[1], mnorm, Q.astype(np.float32))
    assert np.isfinite(eps).all() and (eps > 0).all()
    d = R.reference(Q, X, metric)
    for order in ("sequential", "pairwise", "strided32"):
        s = R.screen_sum(Q, X, metric, order).astype(np.float64)
        assert np.isfinite(s).all(), order
        dev = np.abs(s - d)
        slack = dev - eps[:, None]
        assert (slack <= 0).all(), (order, float(slack.max()), float(dev.max()))


def test_bound_is_tight_enough_to_prove():
    """on spread-out data the bound is a small fraction of the gap it has to clear: the screen can prove answers"""
    rng = np.random.default_rng(5)
    X = rng.uniform(0, 1, (2000, 768)).astype(np.float32)
    Q = rng.uniform(0, 1, (4, 768))
    eps = R.beps("MANHATTAN", 768, R.max_norm(X, "MANHATTAN"), Q.astype(np.float32))
    d = np.sort(R.reference(Q, X, "MANHATTAN"), axis=1)
    assert (eps < 1e-3 * d[:, 0]).all()
