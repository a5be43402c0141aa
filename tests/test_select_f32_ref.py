"""CPU checks of tests/select_f32_ref.py, the op-for-op restatement of the F32 COSINE / EUCLIDEAN selection kernel
(hnsw_select_kernel) that tests/test_gpu_hnsw_build_shapes.py compares the GPU with."""
from fractions import Fraction

import numpy as np

import select_f32_ref as S

F32 = np.float32


def rn32(x):
    """the f32 nearest to the exact rational x, ties to even"""
    f = F32(float(x))  # within one step of the answer
    cands = [np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c).view(np.int32)) & 1))
    return best


def test_fmaf_is_exact_where_plain_f64_rounds_twice():
    # c = 1 and a * b just above 2^-24, half an f32 step of 1: the f64 sum lands on the midpoint 1 + 2^-24 and ties
    # to even (1.0), while the exact sum lies above it (1 + 2^-23)
    rng = np.random.default_rng(1)
    found = 0
    for _ in range(4000):
        a = F32(rng.uniform(1, 2))
        b = F32(2.0 ** -24 / float(a))
        c = F32(rng.choice([1.0, -1.0, 3.0, 1.5]))
        want = rn32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))
        naive = F32(float(a) * float(b) + float(c))
        got = S.fmaf(a, b, c)
        assert got.view(np.int32) == want.view(np.int32), (a, b, c)
        found += naive != want
    assert found >= 5, found
    # vectorised, with signs, subnormal results and specials
    a = np.array([1e-30, -3.0, np.inf, 0.0, 2.0 ** -75], F32)
    b = np.array([1e-10, 5.0, 0.0, np.nan, 1.5 * 2.0 ** -75], F32)
    c = np.array([-1e-40, 15.0, 1.0, 1.0, 0.0], F32)
    got = S.fmaf(a, b, c)
    assert got[1] == 0.0 and np.isnan(got[2]) and np.isnan(got[3])
    assert got[4] == F32(2.0 ** -149)  # 0.75 * 2^-149 rounds up to the smallest subnormal
    assert got[0].view(np.int32) == rn32(Fraction(float(a[0])) * Fraction(float(b[0])) + Fraction(float(c[0]))).view(np.int32)


def test_lane_butterfly_sum_is_not_the_sequential_sum():
    # 2^12 in column 0 and ones elsewhere: lane 0 folds 2^24 + 1, which rounds to even (2^24); lanes 1..31 fold 2 each
    # and the tree adds them without loss, while a sequential fold loses every single 1 against 2^24
    x = np.full(64, F32(1.0), F32)
    x[0] = F32(2.0 ** 12)
    lanes = S.lane_sums(x[None, :], x[None, :])
    assert lanes[0, 0] == F32(2.0 ** 24) and (lanes[0, 1:] == 2).all()
    tree = S.norms(x)[0]
    seq = F32(0)
    for v in x:
        seq = S.fmaf(v, v, seq)
    assert tree == F32(2.0 ** 24 + 62)
    assert seq == F32(2.0 ** 24)


def test_distances_match_f64_closely_and_are_symmetric():
    rng = np.random.default_rng(2)
    X = rng.normal(0, 1, (40, 77)).astype(F32)
    for cosine in (True, False):
        d = S.Dist(X[0], S.norms(X[:1])[0], X, cosine)
        x64 = X.astype(np.float64)
        if cosine:
            w = 1 - x64 @ x64[0] / np.sqrt((x64 * x64).sum(1) * (x64[0] ** 2).sum())
        else:
            w = ((x64 - x64[0]) ** 2).sum(1)
        assert np.allclose(d.vals[:, 0], w, rtol=1e-5, atol=1e-5)
        # the kernel's d(a, b) equals d(b, a) bit for bit: products commute, the norms are folded alike
        back = np.array([S.Dist(X[i], S.norms(X[i : i + 1])[0], X[:1], cosine).vals[0] for i in range(40)])
        assert back.tobytes() == d.vals.tobytes()
        if not cosine:
            assert (d.vals == d.vals[:, :1]).all()  # euclidean: exact, a single value


def test_nan_distances():
    X = np.array([[1.0, 2.0], [0.0, 0.0], [np.nan, 1.0], [np.inf, 0.0], [3.0, 4.0]], F32)
    d = S.Dist(X[0], S.norms(X[:1])[0], X, True)
    assert np.isnan(d.vals[1]).all() and np.isnan(d.vals[2]).all() and np.isnan(d.vals[3]).all()  # 1 - 0 * inf
    e = S.Dist(X[0], S.norms(X[:1])[0], X, False)
    assert np.isnan(e.vals[2]).all() and np.isinf(e.vals[3]).all()
    # a NaN distance neither rejects nor is rejected: NaN > x and x > NaN are both false
    out, ok = S.gt(d.vals[1], d.p[1], d.vals[[0, 4]], d.p[[0, 4]])
    assert not out.any() and ok.all()
    out, ok = S.gt(d.vals[4], d.p[4], d.vals[[1]], d.p[[1]])
    assert not out.any() and ok.all()


def test_rank_rule_nan():
    d = np.array([0.5, np.nan, 0.25, S.SELF_MARK, np.inf, np.nan, 0.25, -0.0, 0.0], F32)
    old = S.rank_old(d)
    # the old rule: both NaNs rank 0, no number counts them, so slot 0 collides and the last slots stay unwritten
    assert sorted(old.tolist()) != list(range(d.size)) and (old == -1).sum() == 2
    new = S.rank_fixed(d)
    assert sorted(new.tolist()) == list(range(d.size))
    # numbers by value (equal numbers, -0.0 and 0.0 included, in list order), the marker and +inf, then NaNs in order
    assert new.tolist() == [7, 8, 2, 6, 0, 3, 4, 1, 5]
    # without a NaN the two rules agree
    f = np.array([0.5, 0.25, S.SELF_MARK, 0.25, -1.0, np.inf], F32)
    assert S.rank_old(f).tolist() == S.rank_fixed(f).tolist()
    rng = np.random.default_rng(3)
    for _ in range(50):
        v = rng.integers(0, 6, 40).astype(F32)
        assert S.rank_old(v).tolist() == S.rank_fixed(v).tolist()
        v[rng.integers(0, 40, 3)] = np.nan
        assert sorted(S.rank_fixed(v).tolist()) == list(range(40))
        assert (S.rank_old(v) == -1).any()


def test_rsqrt_window_holds_the_correctly_rounded_value_and_2_ulp():
    rng = np.random.default_rng(4)
    p = rng.uniform(0.01, 1e6, 500).astype(F32)
    W = S.rsqrt_window(p)
    for i in range(p.size):
        cr = rn32(Fraction(1.0 / np.sqrt(np.float64(p[i]))))
        assert cr in W[i]
        vals = np.unique(W[i])
        assert 3 <= vals.size <= 6 and np.all(np.abs(vals.astype(np.float64) - 1 / np.sqrt(np.float64(p[i]))) <=
                                              2.01 * S.ulp32(cr)), (p[i], vals)
    assert (S.rsqrt_window(np.array([0.0, np.inf, np.nan], F32))[:, 0][:2] == [np.inf, 0.0]).all()


def test_select_hand_worked():
    # points on a line, euclidean: squared distances decide exactly as the distances do
    X = np.array([[0.0], [1.0], [2.0], [3.0], [-5.0], [-1.0]], F32)
    assert S.select(X, 0, [3, 1, 2], 3, 1, False) == ([3, 1, 2], True)  # take_all
    assert S.select(X, 0, [3, 1, 2], 2, 1, False) == ([3, 1], True)
    assert S.select(X, 0, [1, 2, 3], 2, 1, False) == ([1], True)
    assert S.select(X, 0, [3, 4, 2, 1], 2, 0, False) == ([1, 4], True)
    assert S.select(X, 0, [5, 1, 3], 1, 0, False) == ([5], True)  # equal distances: list order
    assert S.select(X, 0, [1, 0, 5, 3], 2, 0, False) == ([1, 5], True)  # the element itself is skipped
    # a NaN candidate is visited last with presorted = 0 and, never rejected, fills a free slot
    Y = np.array([[0.0], [1.0], [np.nan], [3.0]], F32)
    assert S.select(Y, 0, [2, 3, 1], 2, 0, False) == ([1, 2], True)


def test_select_f32_agrees_with_the_reference_selection_on_exact_data():
    # small integers: every f32 sum is exact, so the euclidean selection equals Heuristic::select in any arithmetic
    import hnsw_select_ref as H
    rng = np.random.default_rng(5)
    X = rng.integers(-4, 5, (60, 9)).astype(F32)
    for i in range(30):
        cand = rng.choice(60, 20, replace=False)
        for presorted in (0, 1):
            got, ok = S.select(X, i, cand, 5, presorted, False)
            assert ok
            want = H.select("euclidean", X.astype(np.float64), i, cand, 5, presorted, vector_type="F64")
            assert got == want, (i, presorted)
