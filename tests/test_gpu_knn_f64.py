"""Brute-force KNN on F64 corpora through the tensor-core screens: int8 / bf16 copies of the f64 rows, stage B on f64
rows rounded to f32, the packed f64 re-rank.  Rows, their order and the f64 distances must be IDENTICAL to the oracle
on the f64 rows, whatever the screen.

Parity runs over dimensions, screens, batch sizes and k; the special rows of F64 (elements or norms beyond f32, rows
too small for the f32 / bf16 copies) are counted; near-ties below f32 precision are repaired or fall back.  The second
half holds the proof's premises against plain references through the test-only debug ABI (as
test_gpu_screen_invariants.py does for F32): operand copies (tests/screen_ref_f64.py), residuals, |screened - exact| <=
beps, stage B within beps2 (which carries the 2^-24 term of rounding f64 rows to f32), and a proof audit.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import screen_ref as R
import screen_ref_f64 as R64
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SCREEN = {"AUTO": 0, "SIMT_F32": 1, "TC_BF16": 2, "NONE_EXACT": 3, "TC_INT8": 4}
FLT_MIN, FLT_MAX = 1.1754943508222875e-38, 3.4028234663852886e38
CAP, SPECIAL_CAP = 4096, 1024


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def column(ctx, X, metric, screen=None, skip=None):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, X.shape[1], metric, "F64" if X.dtype == np.float64 else "F32", capacity=X.shape[0])
    col.append(X)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if screen:
        col.set_screen(screen)
    return col


def check(col, X, Q, metric, k, skip=None):
    rows, dist, cnt = col.knn(Q, k)
    for q in range(Q.shape[0]):
        r, d = O.knn_topk(X, Q[q], metric.lower(), k, skip=skip)
        assert cnt[q] == r.size and list(rows[q, : cnt[q]]) == list(r), (q, rows[q, :8], r[:8])
        assert dist[q, : cnt[q]].tobytes() == d.tobytes(), q
    return col.stats()


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def expected_special(X, metric):
    """finalize_rows_kernel's special-row rule for f64 rows (skip masks aside)."""
    X = np.asarray(X, np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        s = np.zeros(X.shape[0])
        for c in range(X.shape[1]):
            s = s + X[:, c] * X[:, c]
        m = np.sqrt(s)
        amax = np.abs(X).max(axis=1)
        normal = lambda v: (np.abs(v) >= FLT_MIN) & (np.abs(v) <= FLT_MAX)  # noqa: E731
        mf = m.astype(np.float32)
        if metric == "COSINE":
            sn = (1.0 / m).astype(np.float32)
            sp = ~(m > 0) | ~np.isfinite(m)
        else:
            sn = s.astype(np.float32)
            sp = ~np.isfinite(s) | ~np.isfinite(sn)
        sp |= ~(amax <= FLT_MAX) | ((amax > 0) & ((m < 2.0**-100) | ~normal(mf) | ~normal(sn)))
    return sp


# ---------------------------------------------------------------------------------------------------------- parity
_ORACLE = {}


def _data(dim, metric):
    key = (dim, metric)
    if key not in _ORACLE:
        _ORACLE.clear()
        rng = np.random.default_rng(dim * 31 + len(metric))
        n = 20000 if dim <= 128 else 6000
        X = rng.uniform(-20, 20, (n, dim))
        Q = rng.uniform(-20, 20, (1024, dim))
        Q[1::4] = X[rng.integers(0, n, Q[1::4].shape[0])] + rng.normal(0, 0.5, Q[1::4].shape)  # queries near rows
        rows, dist = O.knn_topk_batch(X, Q, metric.lower(), 257, 16)
        _ORACLE[key] = (X, Q, rows, dist)
    return _ORACLE[key]


CASES = [(m, s) for m, screens in (("COSINE", ("TC_INT8", "TC_BF16", "AUTO")), ("EUCLIDEAN", ("TC_BF16", "AUTO")))
         for s in screens]


@pytest.mark.parametrize("dim", [7, 100, 128, 768, 1025])
@pytest.mark.parametrize("metric,screen", CASES)
def test_f64_parity(ctx, dim, metric, screen):
    X, Q, orows, odist = _data(dim, metric)
    col = column(ctx, X, metric, screen)
    for nq, k in ((1, 1), (3, 10), (11, 100), (11, 256), (1024, 10), (1024, 1), (3, 257)):
        rows, dist, cnt = col.knn(Q[:nq], k)
        assert (cnt == min(k, X.shape[0])).all()
        assert np.array_equal(rows, orows[:nq, :k]), (nq, k, np.argwhere(rows != orows[:nq, :k])[:4])
        assert dist.tobytes() == np.ascontiguousarray(odist[:nq, :k]).tobytes(), (nq, k)
        st = col.stats()
        if k > 256:
            assert st["screen_used"] == SCREEN["NONE_EXACT"]
            continue
        if screen == "AUTO":
            want = ("TC_INT8", "TC_BF16") if metric == "COSINE" else ("TC_BF16",)
            assert st["screen_used"] in [SCREEN[s] for s in want], st
        else:
            assert st["screen_used"] == SCREEN[screen], st
        assert st["n_fallback"] <= 2 + nq // 64, (nq, k, st)
    col.close()


def test_f64_simt_and_exact_requests_stay_exact(ctx):
    X, Q, orows, odist = _data(128, "COSINE")
    for screen in ("SIMT_F32", "NONE_EXACT"):
        col = column(ctx, X, "COSINE", screen)
        rows, dist, _ = col.knn(Q[:3], 10)
        assert np.array_equal(rows, orows[:3, :10]) and dist.tobytes() == np.ascontiguousarray(odist[:3, :10]).tobytes()
        st = col.stats()
        assert st["screen_used"] == SCREEN["NONE_EXACT"] and st["n_fallback"] == 3
        col.close()


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("dim", [100, 128])
def test_f32_values_stored_as_f64(ctx, metric, dim):
    rng = np.random.default_rng(dim + len(metric))
    X32 = rng.uniform(-1, 1, (20000, dim)).astype(np.float32)
    Q = rng.uniform(-1, 1, (64, dim))
    Q[::2] = X32[rng.integers(0, 20000, 32)] + rng.normal(0, 0.01, (32, dim))
    a, b = column(ctx, X32, metric), column(ctx, X32.astype(np.float64), metric)
    for k in (1, 10, 100):
        ra, da, ca = a.knn(Q, k)
        rb, db, cb = b.knn(Q, k)
        assert np.array_equal(ra, rb) and np.array_equal(ca, cb) and da.tobytes() == db.tobytes(), k
        assert b.stats()["screen_used"] in (SCREEN["TC_INT8"], SCREEN["TC_BF16"])
    check(b, X32.astype(np.float64), Q[:8], metric, 10)
    a.close()
    b.close()


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_ties_below_f32_precision(ctx, metric):
    # groups of rows that differ only below f32 precision: their f32 images (and often their f64 distances) coincide,
    # so stage B cannot order them -- the result must still be exact, by repair or by fallback
    rng = np.random.default_rng(11 + len(metric))
    n, dim = 12000, 96
    X = rng.uniform(-20, 20, (n, dim))
    base = rng.integers(0, n, 40)
    for j, r in enumerate(base):
        for t in range(1, 8):
            X[(r + 97 * t + j) % n] = X[r] * (1.0 + t * 2.0**-30)
    Q = X[base] + rng.normal(0, 1e-6, (40, dim))
    Q[::5] = X[base[::5]]
    for screen in ("AUTO", "TC_BF16"):
        col = column(ctx, X, metric, screen)
        for k in (1, 5, 10):
            st = check(col, X, Q, metric, k)
            assert st["screen_used"] != SCREEN["NONE_EXACT"]
        col.close()


def _special_corpus(rng, n, dim, binades=True):
    X = rng.uniform(-20, 20, (n, dim))
    rows = {}
    rows["elem_1e39"] = 10
    X[10, 3] = 1e39
    rows["elem_1e300"] = 20
    X[20, 0] = -1e300
    rows["norm_beyond_f32"] = 30
    X[30] = 1e38 * np.where(np.arange(dim) % 2 == 0, 1.0, -1.0)  # every element an f32, |x| is not
    rows["cos_norm_2e38"] = 35
    X[35, :4] = [2e38, -2e38, 1e38, 1e38]
    rows["tiny_1e-45"] = 40
    X[40] = 1e-45
    rows["tiny_1e-200"] = 50
    X[50] = -1e-200
    rows["subnormal"] = 60
    X[60] = 5e-324 * np.arange(1, dim + 1)
    rows["euclid_small_norm"] = 70
    X[70] = 1e-25  # a normal f32 |x|, but |x|^2 is not
    rows["zero"] = 80
    X[80] = 0.0
    if binades:
        mag = np.exp2(rng.uniform(-20, 20, (40, dim))) * rng.uniform(1, 2, (40, dim))
        X[100:140] = mag * np.where(np.arange(dim) % 2 == 0, 1.0, -1.0)  # 40 binades, alternating signs
    return X, rows


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("dim", [64, 768])
def test_special_rows(ctx, metric, dim):
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(dim + 3 * len(metric))
    n = 8000
    X, rows = _special_corpus(rng, n, dim)
    Q = rng.uniform(-20, 20, (24, dim))
    Q[:8] = X[100:108] * rng.uniform(0.9, 1.1, (8, 1))
    Q[8] = X[30] / 1e38  # along the norm-beyond-f32 row
    Q[9] = 1e-30 * np.sign(X[40])
    want = expected_special(X, metric)
    for name in ("elem_1e39", "elem_1e300", "norm_beyond_f32", "tiny_1e-45", "tiny_1e-200", "subnormal"):
        assert want[rows[name]], name
    assert want[rows["euclid_small_norm"]] == (metric == "EUCLIDEAN") and want[rows["zero"]] == (metric == "COSINE")
    for screen in ("AUTO", "TC_BF16"):
        col = column(ctx, X, metric, screen)
        u = np.zeros(5, np.uint32)
        L.check(L.lib().sdb_debug_corpus_state(col.h, None, _p(u), None, None, None, None))
        st = check(col, X, Q, metric, 10)
        assert st["screen_used"] != SCREEN["NONE_EXACT"]
        assert st["n_special_rows"] == int(want.sum()) + int(u[1]), (st["n_special_rows"], int(want.sum()), int(u[1]))
        check(col, X, Q[:3], metric, 256)
        col.close()


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_skip_remove_refinalize(ctx, metric):
    rng = np.random.default_rng(5 + len(metric))
    n, dim = 15000, 128
    X = rng.uniform(-20, 20, (n, dim))
    Q = X[rng.integers(0, n, 16)] + rng.normal(0, 0.3, (16, dim))
    skip = (rng.random(n) < 0.2).astype(np.uint8)
    col = column(ctx, X, metric, skip=skip)
    st = check(col, X, Q, metric, 10, skip=skip)
    assert st["screen_used"] != SCREEN["NONE_EXACT"]
    # tombstones after finalize, among them the current nearest rows
    r, _, _ = col.knn(Q, 3)
    dead = np.unique(np.concatenate([r[:, :2].ravel().astype(np.int64), rng.integers(0, n, 200)]))
    col.remove(dead)
    skip2 = skip.copy()
    skip2[dead] = 1
    st = check(col, X, Q, metric, 10, skip=skip2)
    assert st["screen_used"] != SCREEN["NONE_EXACT"]
    # a new skip mask and a re-finalize: removed rows stay removed
    skip3 = (rng.random(n) < 0.05).astype(np.uint8)
    col.set_skip(skip3)
    col.finalize()
    skip3[dead] = 1
    st = check(col, X, Q, metric, 10, skip=skip3)
    assert st["screen_used"] != SCREEN["NONE_EXACT"]
    col.close()


def test_device_entry_points_and_two_batches_in_flight(ctx):
    import torch
    rng = np.random.default_rng(21)
    n, dim, nq, k = 20000, 256, 96, 10
    X = rng.uniform(-20, 20, (n, dim))
    batches = [rng.uniform(-20, 20, (nq, dim)) for _ in range(3)]
    want = [O.knn_topk_batch(X, b, "cosine", k, 16) for b in batches]
    col = column(ctx, X, "COSINE")
    dev = torch.device("cuda", 0)
    qd = [torch.from_numpy(b).to(dev) for b in batches]
    outs = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
             torch.zeros((nq,), dtype=torch.int32, device=dev)) for _ in batches]
    torch.cuda.synchronize()
    col.knn_device(qd[0].data_ptr(), nq, k, 0, outs[0][0].data_ptr(), outs[0][1].data_ptr(), outs[0][2].data_ptr())
    t1 = col.submit_device(qd[1].data_ptr(), nq, k, 0, outs[1][0].data_ptr(), outs[1][1].data_ptr(), outs[1][2].data_ptr())
    t2 = col.submit_device(qd[2].data_ptr(), nq, k, 0, outs[2][0].data_ptr(), outs[2][1].data_ptr(), outs[2][2].data_ptr())
    col.wait(t1)
    col.wait(t2)
    torch.cuda.synchronize()
    for (r, d, c), (wr, wd) in zip(outs, want):
        assert (c.cpu().numpy() == k).all()
        assert np.array_equal(r.cpu().numpy().astype(np.uint64), wr) and d.cpu().numpy().tobytes() == wd.tobytes()
    assert col.stats()["screen_used"] in (SCREEN["TC_INT8"], SCREEN["TC_BF16"])
    col.close()


def test_f64_columns_release_everything(ctx):
    from surrealdb_b200 import Context
    from surrealdb_b200 import _lib as L

    def live():
        c, b = C.c_uint64(), C.c_uint64()
        L.lib().sdb_debug_live_allocations(C.byref(c), C.byref(b))
        return c.value, b.value

    rng = np.random.default_rng(2)
    X = rng.uniform(-20, 20, (5000, 100))
    gc.collect()
    before = live()
    c2 = Context(0)
    for metric in ("COSINE", "EUCLIDEAN"):
        col = column(c2, X, metric)
        check(col, X, X[:4] + 0.1, metric, 10)
        col.remove(np.arange(0, 5000, 7))
        col.knn(X[:2], 5)
        col.close()
    c2.close()
    gc.collect()
    assert live() == before


# ------------------------------------------------------------------------------------------ invariants (debug ABI)
INV_CASES = {
    # name: (n, dim, nq, k, metric, special rows)
    "d128_cos": (20000, 128, 65, 10, "COSINE", False),
    "d100_euclid": (6000, 100, 33, 100, "EUCLIDEAN", False),
    "d768_cos_special": (6000, 768, 33, 10, "COSINE", True),
    "d64_euclid_special": (8000, 64, 33, 10, "EUCLIDEAN", True),
}


class Inv:
    def __init__(self, ctx, name):
        from surrealdb_b200 import _lib as L
        n, dim, nq, k, metric, special = INV_CASES[name]
        rng = np.random.default_rng(sum(map(ord, name)))
        if special:  # (euclidean: no binade rows, whose norms would widen every query's bound past any proof)
            X, _ = _special_corpus(rng, n, dim, binades=metric == "COSINE")
        else:
            X = rng.uniform(-20, 20, (n, dim))
        Q = rng.uniform(-20, 20, (nq, dim))
        Q[1::2] = X[rng.integers(200, n, Q[1::2].shape[0])] * rng.uniform(0.5, 2.0, (Q[1::2].shape[0], 1))
        self.X, self.Q, self.n, self.dim, self.k, self.metric, self.L = X, Q, n, dim, k, metric, L
        self.col = column(ctx, X, metric)
        f, u = np.zeros(4, np.float32), np.zeros(5, np.uint32)
        L.check(L.lib().sdb_debug_corpus_state(self.col.h, _p(f), _p(u), None, None, None, None))
        self.i8_scale, self.max_rel_qerr, self.bf16_rel_err, self.max_norm = (np.float32(v) for v in f)
        self.n_special, self.n_outliers, self.dim_pad, self.dim_pad8, self.n_pad = (int(v) for v in u)
        cos = metric == "COSINE"
        self.x8 = np.zeros((self.n_pad, self.dim_pad8), np.int8) if cos else None
        self.xbf = np.zeros((self.n_pad, self.dim_pad), np.uint16)
        self.snorm = np.zeros(self.n_pad, np.float32)
        self.special = np.zeros(max(self.n_special, 1), np.uint32)
        L.check(L.lib().sdb_debug_corpus_state(self.col.h, None, None, _p(self.x8), _p(self.xbf), _p(self.snorm),
                                               _p(self.special)))
        self.special = self.special[: self.n_special]
        self.valid = ~np.isnan(self.snorm[:n])
        with np.errstate(over="ignore"):
            self.mag = R.magnitude(X)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            self.exact = R.cosine_sim(Q, X) if cos else R.euclid_score(Q, X)

    def batch(self, screen, streaming=True, score_all=False):
        nq = self.Q.shape[0]
        capq = max(CAP, self.n_pad) if score_all else CAP
        out = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
                   q8=np.zeros((nq, self.dim_pad8), np.int8), qbf=np.zeros((nq, self.dim_pad), np.uint16),
                   a=np.zeros((nq, capq, 3), np.uint32))
        if not score_all:
            out["b"] = np.zeros((nq, capq, 2), np.uint32)
            out["rr"] = np.zeros((nq, capq + SPECIAL_CAP), np.uint32)
        self.L.check(self.L.lib().sdb_debug_screen_batch(
            self.col.h, _p(self.Q), nq, self.k, SCREEN[screen], int(streaming), CAP, int(score_all),
            _p(out["qf"]), _p(out["qmag"]), _p(out["qu"]), _p(out["q8"]), _p(out["qbf"]), _p(out["a"]),
            _p(out.get("b")), _p(out.get("rr"))))
        for j, name in enumerate(("tau", "margin", "bscale", "beps", "tau2", "beps2", "q8scale", "q8err", "qbferr")):
            out[name] = out["qf"][:, j]
        for j, name in enumerate(("flags", "qflags", "gathered", "n_a", "n_b", "n_e")):
            out[name] = out["qu"][:, j].astype(np.int64)
        return out


_INV = {}


def get_inv(ctx, name):
    if name not in _INV:
        _INV.clear()
        _INV[name] = Inv(ctx, name)
    return _INV[name]


def _inv_screens(name):
    return ("TC_INT8", "TC_BF16") if INV_CASES[name][4] == "COSINE" else ("TC_BF16",)


@pytest.mark.parametrize("name", list(INV_CASES))
def test_f64_operand_copies(ctx, name):
    c = get_inv(ctx, name)
    n, dim, v = c.n, c.dim, c.valid
    special = expected_special(c.X, c.metric)
    assert not (v & special).any(), "a row the f32 / bf16 copies cannot stand for is screened"
    assert set(c.special.tolist()) == set(np.flatnonzero(~v).tolist())
    assert c.n_special == int(special.sum()) + c.n_outliers
    assert np.isnan(c.snorm[n:]).all()
    with np.errstate(divide="ignore", over="ignore"):
        want_sn = (1.0 / c.mag).astype(np.float32) if c.metric == "COSINE" else None
    if want_sn is not None:
        assert np.array_equal(c.snorm[:n][v], want_sn[v])
    # bf16 copy: one rounding of every f64 element (valid or not), zero padding
    assert np.array_equal(c.xbf[:n, :dim], R64.bf16_rne_f64(c.X))
    assert not c.xbf[:, dim:].any() and not c.xbf[n:].any()
    nz = v & (c.mag > 0)  # (an all-zero row is exact in every copy; euclidean screens it)
    assert R64.bf16_residual_f64(c.X[nz], c.xbf[:n, :dim][nz], c.mag[nz]).max() <= c.bf16_rel_err
    if c.x8 is not None:
        want8 = np.zeros((c.n_pad, c.dim_pad8), np.int8)
        want8[:n][v, :dim] = R64.quantize_rows_f64(c.X[v], c.mag[v], c.i8_scale)
        bad = np.argwhere(c.x8 != want8)
        assert bad.size == 0, f"{bad.shape[0]} int8 elements differ, first {bad[:4].tolist()}"
        res8 = R64.i8_residual_f64(c.X[v], c.x8[:n][v, :dim], c.mag[v], c.i8_scale)
        assert res8.max() <= c.max_rel_qerr, (res8.max(), c.max_rel_qerr)
        # the scale covers every screened row's largest normalised component
        assert (R64.rmax_f64(c.X[v], c.mag[v]) <= np.float32(c.i8_scale) * 127 * (1 + 2.0**-20)).all()


@pytest.mark.parametrize("name,screen", [(n, s) for n in INV_CASES for s in _inv_screens(n)])
def test_f64_screen_error_bounds(ctx, name, screen):
    c = get_inv(ctx, name)
    o = c.batch(screen, score_all=True)
    v = c.valid
    S = np.full((c.Q.shape[0], c.n), np.nan)
    for q in range(S.shape[0]):
        m = o["n_a"][q]
        rows = o["a"][q, :m, 0]
        keep = rows < c.n
        S[q, rows[keep]] = o["a"][q, :m, 1][keep].view(np.float32)
    Sv = S[:, v]
    assert not np.isnan(Sv).any(), "a valid row has no score"
    eq, ex = (o["q8err"], c.max_rel_qerr) if screen == "TC_INT8" else (o["qbferr"], c.bf16_rel_err)
    eps_rel = R.screen_eps_rel(screen, c.dim, eq.astype(np.float64), ex)
    if screen == "TC_BF16":
        eps_rel = eps_rel + _u_abs(c.metric, c.dim, o["qmag"])
    want_beps = R.screen_beps(c.metric, eps_rel, o["qmag"], c.max_norm)
    ok_q = (o["qflags"] & 1) == 0
    assert (o["beps"][ok_q] >= want_beps[ok_q] * (1 - 1e-9)).all()
    exact = c.exact[:, v]
    if c.metric == "COSINE":
        dev = np.abs(Sv * o["bscale"][:, None].astype(np.float64) / o["qmag"][:, None] - exact)
    else:
        dev = np.abs(Sv - exact)
    slack = dev[ok_q] - o["beps"][ok_q, None].astype(np.float64)
    assert (slack <= 0).all(), f"screen error above beps: {slack.max():.3g}"


def _u_abs(metric, dim, qmag):
    """cosine on f64 rows: products below 2^-126 flushed, D 2^-126 / (|q| 2^-100) in similarity units"""
    return dim * 2.0**-26 / qmag if metric == "COSINE" else 0.0


def _beps2_ref(metric, dim, qmag, max_norm):
    """cand_begin_kernel's stage-B bound for f64 rows: (D + 16) 2^-24, 2^-24 for rounding the rows to f32 and the
    underflow term."""
    e2_rel = (dim + 16.0) * 2.0**-24 + 2.0**-24 + _u_abs(metric, dim, qmag)
    if metric == "COSINE":
        return np.full(qmag.shape, e2_rel)
    mn = np.float64(max_norm)
    return 2.0 * e2_rel * qmag * mn + 2.4e-7 * mn * mn + 1e-30


@pytest.mark.parametrize("name,screen,streaming",
                         [(n, s, st) for n in INV_CASES for s in _inv_screens(n) for st in (True, False)])
def test_f64_stage_b_and_proof(ctx, name, screen, streaming):
    c = get_inv(ctx, name)
    o = c.batch(screen, streaming=streaming)
    nq, n, v = c.Q.shape[0], c.n, c.valid
    ok_q = (o["qflags"] & 1) == 0
    want_b2 = _beps2_ref(c.metric, c.dim, o["qmag"], c.max_norm)
    assert (o["beps2"][ok_q].astype(np.float64) >= want_b2[ok_q] * (1 - 1e-7)).all(), "beps2 lacks the f64 term"
    audit = []
    for q in range(nq):
        if not ok_q[q]:
            continue
        n_a = o["n_a"][q]
        rows_a = o["a"][q, :n_a, 0].astype(np.int64)
        assert (rows_a < n).all() and v[rows_a].all(), (q, "an invalid row is a candidate")
        r_a = o["a"][q, :n_a, 2].view(np.float32).astype(np.float64)
        ex = c.exact[q, rows_a]
        dev = np.abs(r_a / o["qmag"][q] - ex) if c.metric == "COSINE" else np.abs(r_a - ex)
        assert (dev <= np.float64(o["beps2"][q])).all(), (q, "stage B error above beps2", dev.max())
        tau2 = np.float32(o["tau2"][q])
        rows_b = o["b"][q, : o["n_b"][q], 0].astype(np.int64)
        assert np.array_equal(np.sort(rows_b), np.sort(rows_a[r_a.astype(np.float32) >= tau2])), (q, "stage-B set")
        rr = o["rr"][q, : o["n_e"][q]].astype(np.int64)
        assert sorted(rr.tolist()) == sorted(rows_b.tolist() + c.special.tolist()), (q, "re-ranked rows")
        tau = np.float32(o["tau"][q])
        if not (o["flags"][q] & 2) and tau > -np.inf and len(audit) < 8:
            audit.append((q, set(rows_a.tolist()), set(rr.tolist()), tau, tau2))
    assert audit, "no proven query to audit"
    qs = [a[0] for a in audit]
    rows, dist = O.knn_topk_batch(c.X, c.Q[qs], c.metric.lower(), n, 16)
    for (q, in_a, in_rr, tau, tau2), r, d in zip(audit, rows, dist):
        dq = np.full(n, np.inf)
        dq[r.astype(np.int64)] = d
        if c.metric == "COSINE":
            bound_a = R.proof_bound_cosine(tau, o["bscale"][q], o["qmag"][q], o["beps"][q])
            bound_b = R.proof_bound_cosine(tau2, 1.0, o["qmag"][q], o["beps2"][q])
        else:
            bound_a = R.proof_bound_euclid(tau, o["qmag"][q], o["beps"][q])
            bound_b = R.proof_bound_euclid(tau2, o["qmag"][q], o["beps2"][q])
        a_mask = np.zeros(n, bool)
        a_mask[list(in_a)] = True
        out = v.copy()
        out[list(in_rr)] = False
        bound = np.where(a_mask, bound_b if tau2 > -np.inf else -np.inf, bound_a)
        bad = np.flatnonzero(out & (dq < bound))
        assert bad.size == 0, (q, bad[:5].tolist(), dq[bad[:5]].tolist(), bound[bad[:5]].tolist())
