"""CPU checks of the PEARSON screen's restatement (tests/pearson_screen_ref.py): the reference arithmetic against the
oracle, eps_ref against exact rational cosines of the centred vectors, and why stage B centres in f64."""
from fractions import Fraction

import numpy as np
import pytest

import pearson_screen_ref as R
from oracle import pyoracle as O


def adversarial_sets(rng, D):
    base = rng.uniform(-1, 1, D)
    rows = [
        rng.uniform(-1, 1, D),
        rng.uniform(-20, 20, D),
        1000.0 + rng.uniform(-1e-3, 1e-3, D),           # offset dwarfs spread
        1e6 + rng.uniform(-1, 1, D),
        2.0 * base + 0.5,                               # affine copies of one row
        3.0 * base - 7.0,
        -base,
        np.nextafter(base, np.inf),
        np.exp2(rng.uniform(-30, 30, D)) * np.where(np.arange(D) % 2, -1.0, 1.0),  # many binades
        np.where(np.arange(D) == 0, 1.0, 1.0 + 2.0 ** -30 * rng.uniform(0, 1, D)),  # one spike on a plateau
    ]
    return np.array(rows)


def exact_cos_within(dx, dq, p, eps):
    """is cos(dx, dq), with the f64 values taken exactly, within eps of p?  (rational arithmetic, no sqrt)"""
    fx = [Fraction(float(v)) for v in dx]
    fq = [Fraction(float(v)) for v in dq]
    N = sum(a * b for a, b in zip(fx, fq))
    AB = sum(a * a for a in fx) * sum(b * b for b in fq)
    lo, hi = Fraction(float(p)) - Fraction(eps), Fraction(float(p)) + Fraction(eps)
    below_hi = (N <= 0 or N * N <= hi * hi * AB) if hi >= 0 else (N < 0 and N * N >= hi * hi * AB)
    above_lo = (N >= 0 or N * N <= lo * lo * AB) if lo <= 0 else (N > 0 and N * N >= lo * lo * AB)
    return below_hi and above_lo


@pytest.mark.parametrize("D", [1, 2, 3, 7, 33, 100])
def test_restatement_matches_the_oracle(D):
    rng = np.random.default_rng(D)
    X = adversarial_sets(rng, D)
    for q in adversarial_sets(np.random.default_rng(D + 100), D)[:5]:
        mine = R.pearson(X, q)
        for i, x in enumerate(X):
            ref = O.f64_metric("pearson", x, q)
            if D == 1:
                assert np.isnan(ref) and np.isnan(mine[i])
            else:
                assert np.float64(ref).tobytes() == mine[i].tobytes(), (i, ref, mine[i])


@pytest.mark.parametrize("D", [2, 5, 64, 257, 1000])
def test_eps_ref_covers_the_gap_to_the_exact_cosine(D):
    rng = np.random.default_rng(1000 + D)
    X = adversarial_sets(rng, D)
    Q = adversarial_sets(np.random.default_rng(2000 + D), D)
    _, _, dX = R.moments(X)
    _, _, dQ = R.moments(Q)
    eps = R.eps_ref(D)
    some_gap = False
    for qi in range(len(Q)):
        P = R.pearson(X, Q[qi])
        for i in range(len(X)):
            if R.is_special(X[i:i + 1])[0] or R.is_special(Q[qi:qi + 1])[0]:
                continue
            assert exact_cos_within(dX[i], dQ[qi], P[i], eps), (i, qi)
            some_gap |= not exact_cos_within(dX[i], dQ[qi], P[i], 0.0)
    assert some_gap  # the reference's pearson is not the exact cosine: without eps_ref the proof would be unsound


def test_stage_b_centres_in_f64():
    # offset / spread ~ 1e6: fl32(x - m1) errs by at most 2^-24 |dx_i| per element, the bound stage B carries over from
    # f64 cosine; fl32(x) - fl32(m1) errs by up to 2^-24 |m1| per element, far beyond it
    rng = np.random.default_rng(6)
    D = 256
    x = (1e6 + rng.uniform(-1, 1, D)).astype(np.float32).astype(np.float64)
    m1, _, dx = R.moments(x[None, :])
    good = dx[0].astype(np.float32).astype(np.float64)
    assert (np.abs(good - dx[0]) <= 2.0 ** -24 * np.abs(dx[0])).all()
    bad = (x.astype(np.float32) - np.float32(m1[0])).astype(np.float64)
    rel = np.linalg.norm(bad - dx[0]) / np.linalg.norm(dx[0])
    assert rel > (D + 17) * 2.0 ** -24, rel


def test_copies_and_specials():
    assert R.bf16_rn(np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -3.0 - 2.0 ** -7])).tolist() == \
        [1.0, 1.0, 1.0 + 2 * 2.0 ** -7, -3.0]  # (ties to even; the bf16 step is 2^-6 in [2, 4))
    X = np.array([[1.0, 2.0, 3.0], [5.0, 5.0, 5.0], [0.0, -0.0, 0.0], [1.0, np.nan, 2.0], [np.inf, 1.0, -np.inf],
                  [7.0, 7.0 + 2.0 ** -60, 7.0], [1e39, 0.0, 1.0]])
    assert R.is_special(X).tolist() == [False, True, True, True, True, True, True]
    q8, res = R.int8_copy(X[:1], 1.0 / 127)
    assert q8.tolist() == [[-90, 0, 90]] and res[0] < 1.0 / 127
