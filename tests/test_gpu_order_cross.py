"""The cross views of `ORDER BY vector::<fn>(emb, $q) ASC|DESC LIMIT k` on COSINE and EUCLIDEAN columns: cosine
distance / similarity in the order KNN does not take, euclidean distance on a COSINE column and farthest first on a
EUCLIDEAN one.  Every result byte for byte against the exact kernel (set_screen("NONE_EXACT")) and, at small sizes,
against the SortTopK reference (tests/sort_topk_ref.py); the cross special rows, tombstones and re-finalize; the
overflowing cross special list; tickets, device variants and cancellation; the remembered rung; and the screens'
invariants through sdb_debug_screen_batch_ranked against tests/cross_screen_ref.py."""
import ctypes as C

import numpy as np
import pytest

import cross_screen_ref as X
from sort_topk_ref import row_values, sort_keyed

pytestmark = pytest.mark.gpu

FN = {"COSINE": 1, "EUCLIDEAN": 2, "SIMILARITY_COSINE": 16}
SCREEN = {"SIMT_F32": 1, "TC_BF16": 2, "NONE_EXACT": 3, "TC_INT8": 4}
SPECIAL_CAP = 1024
# the (fn, order) pairs each column metric now screens; the first COSINE pairs look towards -q on the own norm (int8)
VIEWS = {"COSINE": [("COSINE", "DESC"), ("SIMILARITY_COSINE", "ASC"), ("EUCLIDEAN", "ASC"), ("EUCLIDEAN", "DESC")],
         "EUCLIDEAN": [("EUCLIDEAN", "DESC"), ("COSINE", "ASC"), ("SIMILARITY_COSINE", "DESC"), ("COSINE", "DESC"),
                       ("SIMILARITY_COSINE", "ASC")]}


def int8_view(metric, fn, order):
    return metric == "COSINE" and fn != "EUCLIDEAN"


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def make_col(ctx, x, metric, skip=None, remove=None):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, x.shape[1], metric, "F32" if x.dtype == np.float32 else "F64", capacity=x.shape[0])
    col.append(x)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if remove is not None:
        col.remove(remove)
    return col


def ordered(col, q, k, fn, order, screen, **kw):
    """the call on `screen`, its stats, and the same call on the exact kernel"""
    col.set_screen(screen)
    got = col.order_topk(q, k, fn, order, **kw)
    st = col.stats()
    col.set_screen("NONE_EXACT")
    ref = col.order_topk(q, k, fn, order, **kw)
    col.set_screen(screen)
    return got, st, ref


def same(a, b):
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()


def awkward_corpus(rng, n, d, dtype):
    """integer rows (ties that k cuts), random rows and the special rows: zero, NaN, +-inf, -0.0; for f64 an element
    beyond f32 range, a row of norm below 2^-100 and one whose |x|^2 is below the normal f32 range (a cross special
    row of COSINE columns)"""
    x = np.concatenate([rng.integers(-2, 3, size=(n // 2, d)).astype(np.float64), rng.standard_normal((n - n // 2, d))])
    rng.shuffle(x)
    x[3] = 0.0
    x[7, 2] = np.nan
    x[11, 0] = np.inf
    x[13, 1] = -np.inf
    x[17] = -0.0
    if dtype == np.float64:
        x[19, 0] = 1e39
        x[23] = rng.standard_normal(d) * 2.0 ** -110
        x[29] = rng.standard_normal(d) * 2.0 ** -75
    return x.astype(dtype)


# ---- 1. every new pair x F32/F64 x k, unfiltered and in the three filter regimes, on every screen it admits --------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_small_columns_every_regime(ctx, metric, dtype):
    from surrealdb_b200.engine import pack_row_filter
    rng = np.random.default_rng(17 + (metric == "COSINE") + 2 * (dtype == np.float64))
    n, d = 12003, 40
    x = awkward_corpus(rng, n, d, dtype)
    skip = np.zeros(n, np.uint8)
    skip[rng.choice(np.arange(40, n), 60, replace=False)] = 1
    removed = rng.choice(np.arange(40, n), 40, replace=False)
    col = make_col(ctx, x, metric, skip, removed)
    live = ~skip.astype(bool)
    live[removed] = False
    q = np.concatenate([rng.integers(-2, 3, size=(3, d)).astype(np.float64), rng.standard_normal((5, d))])
    dense = rng.random(n) < 0.8            # screened
    selective = rng.random(n) < 0.02       # the direct regime (fewer than 4096 passing rows)
    masks = np.stack([dense, selective])
    filt = pack_row_filter(masks)
    regimes = [(None, None, None), (filt, np.zeros(8, np.uint32), "dense"), (filt, np.ones(8, np.uint32), "direct"),
               (filt, (np.arange(8) % 2).astype(np.uint32), "mixed")]
    for fn, order in VIEWS[metric]:
        vals = [row_values(FN[fn], x, qq) for qq in q]
        screens = ["TC_BF16"] + (["SIMT_F32"] if dtype == np.float32 else [])
        screens += ["TC_INT8"] if int8_view(metric, fn, order) else []
        for screen in screens:
            for k in (1, 10, 256):
                for f, qf, regime in regimes:
                    kw = {} if f is None else dict(filters=f, query_filter=qf)
                    got, st, ref = ordered(col, q, k, fn, order, screen, **kw)
                    same(got, ref)
                    if regime in (None, "dense"):
                        assert st["screen_used"] == SCREEN[screen], (fn, order, screen, regime, st)
                    for qi in range(q.shape[0]):
                        ok = live if f is None else live & masks[qf[qi]]
                        er, ev = sort_keyed(vals[qi], k, order == "DESC", ok)
                        assert int(got[2][qi]) == er.size
                        assert np.array_equal(got[0][qi][: er.size], er)
                        assert got[1][qi][: er.size].tobytes() == ev.tobytes()
        if not int8_view(metric, fn, order):  # an int8 request serves the other views on bf16
            got, st, ref = ordered(col, q, 10, fn, order, "TC_INT8")
            assert st["screen_used"] == SCREEN["TC_BF16"]
            same(got, ref)
        if dtype == np.float64:  # the SIMT screen streams f32 rows: an F64 column takes the exact kernel
            got, st, ref = ordered(col, q, 10, fn, order, "SIMT_F32")
            assert st["screen_used"] == SCREEN["NONE_EXACT"]
            same(got, ref)
    col.close()


# ---- 2. zero rows of a EUCLIDEAN column: their generated-NaN cosine sorts first for similarity ASC ------------------
@pytest.mark.parametrize("fn, order", [("SIMILARITY_COSINE", "ASC"), ("COSINE", "ASC")])
def test_zero_rows_of_a_euclidean_column_come_first(ctx, fn, order):
    rng = np.random.default_rng(31)
    x = rng.standard_normal((20000, 48)).astype(np.float32)
    zeros = np.array([5, 900, 15000])
    x[zeros] = 0.0
    col = make_col(ctx, x, "EUCLIDEAN")
    q = rng.standard_normal((16, 48))
    got, st, ref = ordered(col, q, 10, fn, order, "AUTO")
    same(got, ref)
    assert st["screen_used"] == SCREEN["TC_BF16"]
    assert (np.sort(got[0][:, :3], axis=1) == zeros).all()
    assert np.isnan(got[1][:, :3]).all()
    knn = col.knn(q, 10)  # KNN screens the zero rows as ordinary ones
    assert col.stats()["screen_used"] == SCREEN["TC_BF16"]
    col.set_screen("NONE_EXACT")
    same(knn, col.knn(q, 10))
    col.close()


# ---- 3. tombstones and re-finalize ------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_remove_and_refinalize(ctx, metric):
    rng = np.random.default_rng(41)
    n, d = 30000, 64
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[[10, 20]] = 0.0  # own or cross special rows
    col = make_col(ctx, x, metric)
    q = rng.standard_normal((24, d))
    for fn, order in VIEWS[metric]:
        got, _, ref = ordered(col, q, 10, fn, order, "AUTO")
        same(got, ref)
        gone = np.unique(np.concatenate([got[0][:, :3].ravel().astype(np.int64), [10, 20]]))
        col.remove(gone)
        got2, st, ref2 = ordered(col, q, 10, fn, order, "AUTO")
        same(got2, ref2)
        assert st["screen_used"] in (SCREEN["TC_BF16"], SCREEN["TC_INT8"]), st
        assert not np.isin(got2[0], gone).any()
    skip = np.zeros(n, np.uint8)
    skip[rng.choice(n, 3000, replace=False)] = 1
    col.set_skip(skip)
    col.finalize()
    for fn, order in VIEWS[metric]:
        got, _, ref = ordered(col, q, 10, fn, order, "AUTO")
        same(got, ref)
        assert not skip[got[0].astype(np.int64)].any()
    col.close()


# ---- 4. more than SPECIAL_CAP cross special rows: the cross views take the exact kernel, KNN stays screened ----------
def test_cross_special_overflow(ctx):
    rng = np.random.default_rng(43)
    n, d = 20000, 32
    x = rng.standard_normal((n, d)).astype(np.float32)
    zeros = rng.choice(n, SPECIAL_CAP + 100, replace=False)
    x[zeros] = 0.0
    col = make_col(ctx, x, "EUCLIDEAN")
    q = rng.standard_normal((8, d))
    for fn, order in VIEWS["EUCLIDEAN"]:
        col.set_screen("AUTO")
        rows, vals, cnt = col.order_topk(q, 10, fn, order)
        st = col.stats()
        want = SCREEN["TC_BF16"] if fn == "EUCLIDEAN" else SCREEN["NONE_EXACT"]
        assert st["screen_used"] == want, (fn, order, st)
        for qi in range(q.shape[0]):
            er, ev = sort_keyed(row_values(FN[fn], x, q[qi]), 10, order == "DESC")
            assert np.array_equal(rows[qi], er) and vals[qi].tobytes() == ev.tobytes()
    col.set_screen("AUTO")
    knn = col.knn(q, 10)
    assert col.stats()["screen_used"] == SCREEN["TC_BF16"]
    col.set_screen("NONE_EXACT")
    same(knn, col.knn(q, 10))
    col.close()


# ---- 5. k = 257 stays on the exact kernel -------------------------------------------------------------------------
def test_k_257_ranks_on_the_exact_kernel(ctx):
    rng = np.random.default_rng(4)
    x = awkward_corpus(rng, 5000, 24, np.float32)
    col = make_col(ctx, x, "EUCLIDEAN")
    q = rng.standard_normal((3, 24))
    for fn, order in VIEWS["EUCLIDEAN"]:
        rows, vals, cnt = col.order_topk(q, 257, fn, order)
        assert col.stats()["screen_used"] == SCREEN["NONE_EXACT"]
        for qi in range(3):
            er, ev = sort_keyed(row_values(FN[fn], x, q[qi]), 257, order == "DESC")
            assert np.array_equal(rows[qi], er) and vals[qi].tobytes() == ev.tobytes()
    col.close()


# ---- 6. production shape: 1M x 768 F32, 1024 queries -----------------------------------------------------------------
def _big_column(ctx, metric, scaled):
    """1M x 768 clustered F32 rows and 1024 queries near the clusters.  They are drawn on the host (torch's CPU
    generator), so every machine ranks the same rows: the CUDA generator's output depends on its launch grid, so on the
    card."""
    import torch
    from surrealdb_b200 import VectorColumn
    n, d = 1_000_000, 768
    g = torch.Generator().manual_seed(13)
    centers = torch.randn(2000, d, generator=g)
    col = VectorColumn(ctx, d, metric, "F32", capacity=n)
    step = 250_000
    for i in range(0, n, step):
        idx = torch.randint(0, 2000, (step,), generator=g)
        rows = centers[idx] + 0.4 * torch.randn(step, d, generator=g)
        if scaled:  # per-row factors spanning 16x
            rows *= torch.exp2(4.0 * torch.rand(step, 1, generator=g))
        rows = rows.contiguous().cuda()
        col.append_device(rows.data_ptr(), step)
        torch.cuda.synchronize()
        del rows
    col.finalize()
    qi = torch.randint(0, 2000, (1024,), generator=g)
    q = (centers[qi] + 0.4 * torch.randn(1024, d, generator=g)).double().numpy()
    return col, q


def _knn_stats(ctx, metric, scaled, k):
    """KNN on a column of `metric` holding the same rows and queries: its stats (the same screen, score form and
    ladder as a cross view of that form)"""
    col, q = _big_column(ctx, metric, scaled)
    out = {}
    for kk in k:
        col.knn(q, kk)
        out[kk] = col.stats()
    col.close()
    return out


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_production_shape(ctx, metric, scaled):
    """every result equals the exact kernel; the repairs stay within what the same score form costs KNN.  Euclidean
    ASC on the COSINE column is KNN's euclidean screen with the cross |x|^2: it is held to EUCLIDEAN KNN on the same
    rows (at k = 256 on these clusters, about 500 rows each, the streaming screen's gathering of either can reach the
    16384-entry lists and the batch climbs the ladder).  The other views, on rows of one scale, repair at most a
    quarter of the batch."""
    col, q = _big_column(ctx, metric, scaled)
    views = [VIEWS[metric][0], VIEWS[metric][2]] if metric == "COSINE" else VIEWS[metric][:3]
    stats = {}
    for fn, order in views:
        for k in (10, 256):
            got, st, ref = ordered(col, q, k, fn, order, "AUTO")
            same(got, ref)
            assert st["screen_used"] in (SCREEN["TC_BF16"], SCREEN["TC_INT8"]), st
            print(f"\n{metric} scaled={scaled} {fn} {order} k={k}: screen {st['screen_used']}, survivors/query "
                  f"{st['n_survivors'] / 1024:.0f}, largest set {st['n_candidates']}, repaired {st['n_repaired']}, "
                  f"fallback {st['n_fallback']}")
            stats[fn, order, k] = st
    col.close()
    for (fn, order, k), st in stats.items():
        if metric == "COSINE" and fn == "EUCLIDEAN":
            continue
        if not scaled:
            assert st["n_fallback"] + st["n_repaired"] <= 1024 // 4, (fn, order, k, st)
    if metric == "COSINE":
        knn = _knn_stats(ctx, "EUCLIDEAN", scaled, (10, 256))
        for k in (10, 256):
            st, kn = stats["EUCLIDEAN", "ASC", k], knn[k]
            print(f"\nEUCLIDEAN KNN, same rows, scaled={scaled} k={k}: survivors/query {kn['n_survivors'] / 1024:.0f}, "
                  f"repaired {kn['n_repaired']}, fallback {kn['n_fallback']}")
            assert st["n_fallback"] + st["n_repaired"] <= kn["n_fallback"] + kn["n_repaired"] + 1024 // 4, (k, st, kn)


# ---- 7. a climbing cross view does not move the rung KNN starts on --------------------------------------------------
def test_cross_rung_is_kept_apart_from_knn(ctx):
    """a near-duplicate crowd larger than a 4096-slot list makes the farthest-first batches climb the ladder; KNN
    batches on the same column then run as they would have (no stats field shows a batch's first rung: the results
    and the screen are checked), and the cross batches keep answering exactly"""
    rng = np.random.default_rng(12)
    d = 96
    base = rng.standard_normal(d)
    crowd = 4.0 * base + 1e-3 * rng.standard_normal((12000, d))
    x = np.concatenate([crowd, rng.standard_normal((30000, d))]).astype(np.float32)
    col = make_col(ctx, x, "EUCLIDEAN")
    qd = np.tile(-base, (48, 1)) + 1e-2 * rng.standard_normal((48, d))
    qk = rng.standard_normal((48, d))
    col.set_screen("NONE_EXACT")
    ref_far = col.order_topk(qd, 10, "EUCLIDEAN", "DESC")
    ref_knn = col.knn(qk, 10)
    col.set_screen("AUTO")
    for _ in range(2):
        same(col.order_topk(qd, 10, "EUCLIDEAN", "DESC"), ref_far)
        assert col.stats()["screen_used"] in (SCREEN["TC_BF16"], SCREEN["SIMT_F32"])
        same(col.knn(qk, 10), ref_knn)
        assert col.stats()["screen_used"] == SCREEN["TC_BF16"]
    col.close()


# ---- 8. tickets: cross batches among KNN, cosine-DESC and dot tickets on both streams, device variants, cancel ------
def test_tickets_device_and_cancel(ctx):
    import torch
    from surrealdb_b200 import _lib
    rng = np.random.default_rng(19)
    x = rng.standard_normal((50000, 64)).astype(np.float32)
    col = make_col(ctx, x, "COSINE")
    q = rng.standard_normal((32, 64))
    k = 16
    kinds = [("EUCLIDEAN", "DESC"), None, ("SIMILARITY_COSINE", "DESC"), ("COSINE", "DESC"), ("DOT", "ASC"),
             ("EUCLIDEAN", "ASC"), ("SIMILARITY_COSINE", "ASC")]
    bufs = [(np.zeros((32, k), np.uint64), np.zeros((32, k)), np.zeros(32, np.uint32)) for _ in kinds]
    for lo in (0, 4):  # four tickets in flight at a time, alternating streams
        tickets = []
        for kind, b in zip(kinds[lo:lo + 4], bufs[lo:lo + 4]):
            ptrs = [a.ctypes.data for a in b]
            tickets.append(col.submit_host(q.ctypes.data, 32, k, *ptrs) if kind is None else
                           col.order_submit_host(q.ctypes.data, 32, k, kind[0], kind[1], *ptrs))
        for t in reversed(tickets):
            col.wait(t)
    col.set_screen("NONE_EXACT")
    for kind, b in zip(kinds, bufs):
        same(b, col.knn(q, k) if kind is None else col.order_topk(q, k, *kind))
    refs = {o: col.order_topk(q, k, "EUCLIDEAN", o) for o in ("DESC", "ASC")}
    col.set_screen("AUTO")
    dq = torch.from_numpy(q).cuda()
    dr = torch.zeros((32, k), dtype=torch.int64, device="cuda")
    dv = torch.zeros((32, k), dtype=torch.float64, device="cuda")
    dc = torch.zeros(32, dtype=torch.int32, device="cuda")
    col.order_topk_device(dq.data_ptr(), 32, k, "EUCLIDEAN", "ASC", 0, dr.data_ptr(), dv.data_ptr(), dc.data_ptr())
    assert dr.cpu().numpy().view(np.uint64).tobytes() == refs["ASC"][0].tobytes()
    assert dv.cpu().numpy().tobytes() == refs["ASC"][1].tobytes()
    t = col.order_submit_device(dq.data_ptr(), 32, k, "EUCLIDEAN", "DESC", 5, dr.data_ptr(), dv.data_ptr(),
                                dc.data_ptr())
    col.wait(t)
    assert (dr.cpu().numpy().view(np.uint64) - 5).tobytes() == refs["DESC"][0].tobytes()
    assert dv.cpu().numpy().tobytes() == refs["DESC"][1].tobytes()
    b = bufs[0]
    t = col.order_submit_host(q.ctypes.data, 32, k, "EUCLIDEAN", "DESC", *[a.ctypes.data for a in b])
    ctx.cancel()
    try:
        with pytest.raises(_lib.SdbError) as e:
            col.wait(t)
        assert e.value.status == _lib.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    same(col.order_topk(q, k, "EUCLIDEAN", "DESC"), refs["DESC"])
    col.close()


# ---- 9. screen invariants through sdb_debug_screen_batch_ranked ------------------------------------------------------
def _ranked(L, col, Q, k, screen, fn, desc, streaming, score_all, cap, n_pad):
    nq = Q.shape[0]
    capq = max(cap, n_pad) if score_all else cap
    o = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
             qbf=np.zeros((nq, (col.dim + 63) // 64 * 64), np.uint16), a=np.zeros((nq, capq, 3), np.uint32))
    if not score_all:
        o["b"] = np.zeros((nq, capq, 2), np.uint32)
        o["rr"] = np.zeros((nq, capq + SPECIAL_CAP), np.uint32)
    L.check(L.lib().sdb_debug_screen_batch_ranked(
        col.h, _p(Q), nq, k, SCREEN[screen], int(streaming), cap, int(score_all), _p(o["qf"]), _p(o["qmag"]),
        _p(o["qu"]), None, _p(o["qbf"]), _p(o["a"]), _p(o.get("b")), _p(o.get("rr")), None, 0, None, -1, FN[fn],
        1 if desc else 0))
    return o


SHAPES = [  # (d, n, nq, dtype, screen, streaming)
    (1, 300, 5, np.float32, "TC_BF16", True),
    (37, 5001, 130, np.float32, "TC_BF16", False),
    (37, 5001, 130, np.float32, "SIMT_F32", False),
    (768, 3001, 700, np.float32, "TC_BF16", True),
    (4100, 1000, 3, np.float64, "TC_BF16", True),
    (130, 20000, 40, np.float64, "TC_BF16", False),
]


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"d{s[0]}_n{s[1]}_q{s[2]}_{s[3].__name__}_{s[4]}_{s[5]}")
def test_screen_invariants(ctx, shape, metric):
    from surrealdb_b200 import _lib as L
    d, n, nq, dtype, screen, streaming = shape
    rng = np.random.default_rng(d * 7 + n + nq + (metric == "COSINE"))
    centers = rng.standard_normal((20, d))
    Xr = centers[rng.integers(0, 20, n)] + 0.3 * rng.standard_normal((n, d))
    Xr *= np.exp2(rng.uniform(0, 2, (n, 1)))
    Xr[5] = 0.0
    Xr[9, 0] = np.nan
    Xr = Xr.astype(dtype)
    col = make_col(ctx, Xr, metric)
    Q = np.ascontiguousarray(centers[rng.integers(0, 20, nq)] + 0.3 * rng.standard_normal((nq, d)))
    k, cap = min(10, n // 4), 4096
    n_pad = (n + 255) // 256 * 256
    x64 = np.asarray(Xr, np.float64)
    snorm = np.zeros(n_pad, np.float32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, None, None, None, None, _p(snorm), None))
    for fn, order in VIEWS[metric]:
        desc = order == "DESC"
        v = X.view(metric, fn, desc)
        valid = ~np.isnan(snorm[:n]) & (~X.cross_special(x64, metric, dtype == np.float64) if v.cross else True)
        o = _ranked(L, col, Q, k, screen, fn, desc, streaming, True, cap, n_pad)
        q32, qb = X.query_copies(Q, v)
        if screen == "TC_BF16":
            assert np.array_equal(o["qbf"][:, :d], qb.view(np.uint32).__rshift__(16).astype(np.uint16))
        beps, bscale = o["qf"][:, 3].astype(np.float64), o["qf"][:, 2].astype(np.float64)
        assert np.isfinite(beps).all()
        S = np.full((nq, n), np.nan)
        for q in range(nq):
            na = int(o["qu"][q, 3])
            rows = o["a"][q, :na, 0]
            sc = o["a"][q, :na, 1].view(np.float32)
            keep = (rows < n) & ~np.isnan(sc)
            S[q, rows[keep]] = sc[keep]
        assert not np.isfinite(S[:, ~valid]).any()  # own and cross special rows never reach a list
        assert np.isfinite(S[:, valid]).all()
        for q in rng.choice(nq, min(nq, 4), replace=False):
            exact = X.exact_score(x64[valid], Q[q], v)
            err = np.abs(S[q, valid] * bscale[q] - exact)
            assert (err <= X.score_tolerance(v, beps[q], o["qmag"][q])).all(), (fn, order, float(err.max()))
        # the production sequence at rung 0: proven queries have every outside row beyond the proof's bound
        o = _ranked(L, col, Q, k, screen, fn, desc, streaming, False, cap, n_pad)
        tau, tau2, beps, beps2 = (o["qf"][:, j].astype(np.float64) for j in (0, 4, 3, 5))
        bscale = o["qf"][:, 2].astype(np.float64)
        for q in rng.choice(nq, min(nq, 8), replace=False):
            na, nb, ne = (int(o["qu"][q, j]) for j in (3, 4, 5))
            if (o["qu"][q, 0] & 3) or (o["qu"][q, 1] & 1) or not np.isfinite(tau[q]):
                continue
            refv = X.reference_values(fn, x64, Q[q])
            rr = o["rr"][q, :ne].astype(np.int64)
            a_rows = o["a"][q, :na, 0].astype(np.int64)
            b_rows = o["b"][q, :nb, 0].astype(np.int64)
            out_a = valid.copy()
            out_a[a_rows] = False
            checks = [(out_a, X.proof_bound(v, tau[q], bscale[q], beps[q], o["qmag"][q], d))]
            if np.isfinite(tau2[q]):
                out_b = np.zeros(n, bool)
                out_b[np.setdiff1d(a_rows, b_rows)] = True
                checks.append((out_b, X.proof_bound(v, tau2[q], 1.0, beps2[q], o["qmag"][q], d)))
            in_rr = np.zeros(n, bool)
            in_rr[rr] = True
            vk = sort_keyed(refv, k, desc, in_rr)[1][k - 1]
            if np.isnan(vk):
                continue
            slack = 1e-12 * abs(vk)  # (refv restates the reference's arithmetic up to the order of its roundings)
            for outside, bnd in checks:
                if desc:
                    assert (refv[outside] <= bnd + slack).all() and bnd < vk + slack
                else:
                    assert (refv[outside] >= bnd - slack).all() and bnd > vk - slack
    col.close()
