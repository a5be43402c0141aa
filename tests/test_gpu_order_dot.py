"""`ORDER BY vector::dot(emb, $q) DESC|ASC LIMIT k` on the bf16 tensor-core screen of COSINE and EUCLIDEAN columns:
every result byte for byte against the exact kernel (set_screen("NONE_EXACT")) and, at small sizes, against the SortTopK
reference (tests/sort_topk_ref.py); the ladder, the remembered rung and the int8 copy; tickets; and the screen's
invariants through sdb_debug_screen_batch_ranked against tests/dot_screen_ref.py."""
import ctypes as C

import numpy as np
import pytest

import dot_screen_ref as R
from sort_topk_ref import row_values, sort_keyed

pytestmark = pytest.mark.gpu

DOT = 17
SCREEN = {"SIMT_F32": 1, "TC_BF16": 2, "NONE_EXACT": 3, "TC_INT8": 4}
SPECIAL_CAP = 1024


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def make_col(ctx, x, metric, skip=None, remove=None, screen=None):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, x.shape[1], metric, "F32" if x.dtype == np.float32 else "F64", capacity=x.shape[0])
    col.append(x)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if remove is not None:
        col.remove(remove)
    if screen:
        col.set_screen(screen)
    return col


def ordered(col, q, k, order, screen, **kw):
    """the call on `screen`, its stats, and the same call on the exact kernel"""
    col.set_screen(screen)
    got = col.order_topk(q, k, "DOT", order, **kw)
    st = col.stats()
    col.set_screen("NONE_EXACT")
    ref = col.order_topk(q, k, "DOT", order, **kw)
    col.set_screen(screen)
    return got, st, ref


def same(a, b):
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()


def awkward_corpus(rng, n, d, dtype):
    """integer rows (dot ties that k cuts), random rows and the special rows: zero, NaN, +-inf, -0.0; for f64 an
    element beyond f32 range and a row of norm below 2^-100"""
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
    return x.astype(dtype)


# ---- 1. both metrics x F32/F64 x both directions x k, unfiltered and in the three filter regimes -------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_small_columns_every_regime(ctx, metric, dtype):
    from surrealdb_b200.engine import pack_row_filter
    rng = np.random.default_rng(7 + (metric == "COSINE") + 2 * (dtype == np.float64))
    n, d = 12003, 40
    x = awkward_corpus(rng, n, d, dtype)
    skip = np.zeros(n, np.uint8)
    skip[rng.choice(n, 60, replace=False)] = 1
    removed = rng.choice(n, 40, replace=False)
    col = make_col(ctx, x, metric, skip, removed)
    live = ~skip.astype(bool)
    live[removed] = False
    q = np.concatenate([rng.integers(-2, 3, size=(3, d)).astype(np.float64), rng.standard_normal((5, d))])
    vals = [row_values(DOT, x, qq) for qq in q]
    dense = rng.random(n) < 0.8            # screened
    selective = rng.random(n) < 0.02       # the direct regime (fewer than 4096 passing rows)
    masks = np.stack([dense, selective])
    filt = pack_row_filter(masks)
    regimes = [(None, None, None), (filt, np.zeros(8, np.uint32), "dense"), (filt, np.ones(8, np.uint32), "direct"),
               (filt, (np.arange(8) % 2).astype(np.uint32), "mixed")]
    screens = ["TC_BF16"] + (["SIMT_F32"] if dtype == np.float32 else [])
    for screen in screens:
        for order in ("DESC", "ASC"):
            for k in (1, 10, 256):
                for f, qf, regime in regimes:
                    kw = {} if f is None else dict(filters=f, query_filter=qf)
                    got, st, ref = ordered(col, q, k, order, screen, **kw)
                    same(got, ref)
                    if regime in (None, "dense"):
                        assert st["screen_used"] == SCREEN[screen], (screen, regime, st)
                    for qi in range(q.shape[0]):
                        ok = live if f is None else live & masks[qf[qi]]
                        er, ev = sort_keyed(vals[qi], k, order == "DESC", ok)
                        assert int(got[2][qi]) == er.size
                        assert np.array_equal(got[0][qi][: er.size], er)
                        assert got[1][qi][: er.size].tobytes() == ev.tobytes()
    if dtype == np.float64:  # the SIMT screen streams f32 rows: an F64 column takes the exact kernel
        got, st, ref = ordered(col, q, 10, "DESC", "SIMT_F32")
        assert st["screen_used"] == SCREEN["NONE_EXACT"]
        same(got, ref)


# ---- 2. k = 257 stays on the exact kernel -------------------------------------------------------------------------
def test_k_257_ranks_on_the_exact_kernel(ctx):
    rng = np.random.default_rng(4)
    x = awkward_corpus(rng, 5000, 24, np.float32)
    col = make_col(ctx, x, "EUCLIDEAN")
    q = rng.standard_normal((3, 24))
    for order in ("DESC", "ASC"):
        rows, vals, cnt = col.order_topk(q, 257, "DOT", order)
        assert col.stats()["screen_used"] == SCREEN["NONE_EXACT"]
        for qi in range(3):
            er, ev = sort_keyed(row_values(DOT, x, q[qi]), 257, order == "DESC")
            assert np.array_equal(rows[qi], er) and vals[qi].tobytes() == ev.tobytes()


# ---- 3. production shape: 1M x 768 F32, 1024 queries -----------------------------------------------------------------
def _big_column(ctx, metric, scaled):
    import torch
    from surrealdb_b200 import VectorColumn
    n, d = 1_000_000, 768
    g = torch.Generator(device="cuda").manual_seed(11)
    centers = torch.randn(2000, d, device="cuda", generator=g)
    col = VectorColumn(ctx, d, metric, "F32", capacity=n)
    step = 250_000
    for i in range(0, n, step):
        idx = torch.randint(0, 2000, (step,), device="cuda", generator=g)
        rows = centers[idx] + 0.4 * torch.randn(step, d, device="cuda", generator=g)
        if scaled:  # per-row factors spanning 16x
            rows *= torch.exp2(4.0 * torch.rand(step, 1, device="cuda", generator=g))
        rows = rows.contiguous()
        col.append_device(rows.data_ptr(), step)
        torch.cuda.synchronize()
        del rows
    col.finalize()
    qi = torch.randint(0, 2000, (1024,), device="cuda", generator=g)
    q = (centers[qi] + 0.4 * torch.randn(1024, d, device="cuda", generator=g)).double().cpu().numpy()
    return col, q


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_production_shape(ctx, metric, scaled):
    col, q = _big_column(ctx, metric, scaled)
    for order in ("DESC", "ASC"):
        for k in (10, 256):
            got, st, ref = ordered(col, q, k, order, "AUTO")
            same(got, ref)
            assert st["screen_used"] == SCREEN["TC_BF16"], st
            print(f"\n{metric} scaled={scaled} {order} k={k}: survivors/query {st['n_survivors'] / 1024:.0f}, "
                  f"largest set {st['n_candidates']}, repaired {st['n_repaired']}, fallback {st['n_fallback']}")
            if not scaled:
                assert st["n_fallback"] + st["n_repaired"] <= 1024 // 4, st
    col.close()


# ---- 4. the int8 copy and the remembered rung ------------------------------------------------------------------------
def test_int8_request_serves_dot_on_bf16(ctx):
    rng = np.random.default_rng(8)
    x = rng.standard_normal((40000, 64)).astype(np.float32)
    col = make_col(ctx, x, "COSINE", screen="TC_INT8")
    q = rng.standard_normal((64, 64))
    got, st, ref = ordered(col, q, 10, "DESC", "TC_INT8")
    assert st["screen_used"] == SCREEN["TC_BF16"]
    same(got, ref)
    knn = col.knn(q, 10)
    assert col.stats()["screen_used"] == SCREEN["TC_INT8"]  # the KNN batch after it still takes int8
    col.set_screen("NONE_EXACT")
    same(knn, col.knn(q, 10))


@pytest.mark.parametrize("order", ["DESC", "ASC"])
def test_ladder_climb_is_kept_per_score(ctx, order):
    """a near-duplicate crowd larger than a 4096-slot list makes dot batches climb the ladder; KNN batches on the same
    column then run as they would have (no stats field shows a batch's first rung: the results are checked), and the
    dot batches keep answering exactly"""
    rng = np.random.default_rng(12)
    d = 96
    base = rng.standard_normal(d)
    crowd = base + 1e-3 * rng.standard_normal((12000, d))
    x = np.concatenate([crowd, rng.standard_normal((30000, d))]).astype(np.float32)
    col = make_col(ctx, x, "EUCLIDEAN")
    qd = np.tile(base if order == "DESC" else -base, (48, 1)) + 1e-2 * rng.standard_normal((48, d))
    qk = rng.standard_normal((48, d))
    col.set_screen("NONE_EXACT")
    ref_dot = col.order_topk(qd, 10, "DOT", order)
    ref_knn = col.knn(qk, 10)
    col.set_screen("AUTO")
    for _ in range(2):
        same(col.order_topk(qd, 10, "DOT", order), ref_dot)
        st = col.stats()
        assert st["screen_used"] in (SCREEN["TC_BF16"], SCREEN["SIMT_F32"]), st
        same(col.knn(qk, 10), ref_knn)
        assert col.stats()["screen_used"] == SCREEN["TC_BF16"]


# ---- 5. tickets: dot batches among KNN and cosine-DESC tickets, device variants, cancellation ----------------------
def test_tickets_device_and_cancel(ctx):
    import torch
    from surrealdb_b200 import _lib
    rng = np.random.default_rng(19)
    x = rng.standard_normal((50000, 64)).astype(np.float32)
    col = make_col(ctx, x, "COSINE")
    q = rng.standard_normal((32, 64))
    k = 16
    kinds = [("DOT", "DESC"), None, ("SIMILARITY_COSINE", "DESC"), ("DOT", "ASC")]
    bufs, tickets = [], []
    for kind in kinds:
        b = (np.zeros((32, k), np.uint64), np.zeros((32, k)), np.zeros(32, np.uint32))
        bufs.append(b)
        ptrs = [a.ctypes.data for a in b]
        tickets.append(col.submit_host(q.ctypes.data, 32, k, *ptrs) if kind is None else
                       col.order_submit_host(q.ctypes.data, 32, k, kind[0], kind[1], *ptrs))
    for t in (tickets[2], tickets[0], tickets[3], tickets[1]):
        col.wait(t)
    col.set_screen("NONE_EXACT")
    for kind, b in zip(kinds, bufs):
        same(b, col.knn(q, k) if kind is None else col.order_topk(q, k, *kind))
    refs = {o: col.order_topk(q, k, "DOT", o) for o in ("DESC", "ASC")}
    col.set_screen("AUTO")
    dq = torch.from_numpy(q).cuda()
    dr = torch.zeros((32, k), dtype=torch.int64, device="cuda")
    dv = torch.zeros((32, k), dtype=torch.float64, device="cuda")
    dc = torch.zeros(32, dtype=torch.int32, device="cuda")
    col.order_topk_device(dq.data_ptr(), 32, k, "DOT", "ASC", 0, dr.data_ptr(), dv.data_ptr(), dc.data_ptr())
    assert dr.cpu().numpy().view(np.uint64).tobytes() == refs["ASC"][0].tobytes()
    assert dv.cpu().numpy().tobytes() == refs["ASC"][1].tobytes()
    t = col.order_submit_device(dq.data_ptr(), 32, k, "DOT", "DESC", 5, dr.data_ptr(), dv.data_ptr(), dc.data_ptr())
    col.wait(t)
    assert (dr.cpu().numpy().view(np.uint64) - 5).tobytes() == refs["DESC"][0].tobytes()
    assert dv.cpu().numpy().tobytes() == refs["DESC"][1].tobytes()
    b = bufs[0]
    t = col.order_submit_host(q.ctypes.data, 32, k, "DOT", "DESC", *[a.ctypes.data for a in b])
    ctx.cancel()
    try:
        with pytest.raises(_lib.SdbError) as e:
            col.wait(t)
        assert e.value.status == _lib.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    same(col.order_topk(q, k, "DOT", "DESC"), refs["DESC"])


# ---- 6. screen invariants through sdb_debug_screen_batch_ranked --------------------------------------------------------
def _ranked(L, col, Q, k, screen, desc, streaming, score_all, cap, n_pad):
    nq = Q.shape[0]
    capq = max(cap, n_pad) if score_all else cap
    o = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
             qbf=np.zeros((nq, col_dim_pad(col)), np.uint16), a=np.zeros((nq, capq, 3), np.uint32))
    if not score_all:
        o["b"] = np.zeros((nq, capq, 2), np.uint32)
        o["rr"] = np.zeros((nq, capq + SPECIAL_CAP), np.uint32)
    L.check(L.lib().sdb_debug_screen_batch_ranked(
        col.h, _p(Q), nq, k, SCREEN[screen], int(streaming), cap, int(score_all), _p(o["qf"]), _p(o["qmag"]),
        _p(o["qu"]), None, _p(o["qbf"]), _p(o["a"]), _p(o.get("b")), _p(o.get("rr")), None, 0, None, -1, DOT,
        1 if desc else 0))
    return o


def col_dim_pad(col):
    return (col.dim + 63) // 64 * 64


SHAPES = [  # (d, n, nq, dtype, screen, streaming)
    (1, 300, 5, np.float32, "TC_BF16", True),
    (37, 5001, 130, np.float32, "TC_BF16", False),
    (37, 5001, 130, np.float32, "SIMT_F32", False),
    (768, 3001, 2100, np.float32, "TC_BF16", True),
    (4100, 1000, 3, np.float64, "TC_BF16", True),
    (130, 20000, 40, np.float64, "TC_BF16", False),
    (130, 20000, 40, np.float32, "TC_BF16", True),
]


@pytest.mark.parametrize("desc", [True, False])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"d{s[0]}_n{s[1]}_q{s[2]}_{s[3].__name__}_{s[4]}_{s[5]}")
def test_screen_invariants(ctx, shape, desc):
    from surrealdb_b200 import _lib as L
    d, n, nq, dtype, screen, streaming = shape
    rng = np.random.default_rng(d * 7 + n + nq + desc)
    centers = rng.standard_normal((20, d))
    X = centers[rng.integers(0, 20, n)] + 0.3 * rng.standard_normal((n, d))
    X *= np.exp2(rng.uniform(0, 2, (n, 1)))
    X[5] = 0.0
    X[9, 0] = np.nan
    X = X.astype(dtype)
    col = make_col(ctx, X, "EUCLIDEAN" if d % 2 else "COSINE")
    Q = centers[rng.integers(0, 20, nq)] + 0.3 * rng.standard_normal((nq, d))
    Q = np.ascontiguousarray(Q)
    k, cap = min(10, n // 4), 4096
    n_pad = (n + 255) // 256 * 256
    snorm = np.zeros(n_pad, np.float32)
    n_sp = np.zeros(8, np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, None, _p(n_sp), None, None, _p(snorm), None))
    valid = ~np.isnan(snorm[:n])
    # the query copies are those of +-q
    o = _ranked(L, col, Q, k, screen, desc, streaming, True, cap, n_pad)
    q32, qb = R.query_copies(Q, desc)
    if screen == "TC_BF16":
        assert np.array_equal(o["qbf"][:, :d], qb.view(np.uint32).__rshift__(16).astype(np.uint16))
        assert np.allclose(o["qf"][:, 8], R.qbferr(Q, desc), rtol=1e-4)
    beps, bscale = o["qf"][:, 3].astype(np.float64), o["qf"][:, 2]
    assert (bscale == 1).all() and np.isfinite(beps).all()
    # every pass-0 score of a valid row lies within beps of the exact dot; invalid rows never appear
    S = np.full((nq, n), np.nan)
    for q in range(nq):
        na = int(o["qu"][q, 3])
        rows = o["a"][q, :na, 0]
        sc = o["a"][q, :na, 1].view(np.float32)
        keep = (rows < n) & ~np.isnan(sc)
        S[q, rows[keep]] = sc[keep]
    assert not np.isfinite(S[:, ~valid]).any()
    assert np.isfinite(S[:, valid]).all()
    sgn = 1.0 if desc else -1.0
    sample = rng.choice(nq, min(nq, 6), replace=False)
    for q in sample:
        exact = sgn * (X.astype(np.longdouble)[valid] @ Q[q].astype(np.longdouble))
        assert (np.abs(S[q, valid] - exact) <= beps[q]).all()
    # the production sequence at rung 0
    o = _ranked(L, col, Q, k, screen, desc, streaming, False, cap, n_pad)
    tau, mg, tau2, beps2 = (o["qf"][:, j].astype(np.float64) for j in (0, 1, 4, 5))
    refv = np.stack([R.reference_dot(X, Q[q]) for q in range(nq)])
    eref = R.eps_ref(d, float(np.sqrt((np.asarray(X, np.float64)[valid] ** 2).sum(axis=1)).max()) * 1.0001)
    for q in range(nq):
        na, nb, ne = (int(o["qu"][q, j]) for j in (3, 4, 5))
        if o["qu"][q, 0] & 1:
            continue  # overflowed: re-run by the ladder
        a_rows = o["a"][q, :na, 0].astype(np.int64)
        a_sc = o["a"][q, :na, 1].view(np.float32)
        assert np.array_equal(a_sc, S[q, a_rows].astype(np.float32))  # the screen's own scores
        srt = np.sort(S[q, valid])[::-1]
        if np.isfinite(tau[q]):
            assert tau[q] <= srt[k - 1] - mg[q]  # tau <= k-th best - margin
            want = np.flatnonzero(valid & (S[q] >= tau[q]))
            assert np.array_equal(np.sort(a_rows), want)  # stage A keeps exactly the rows reaching tau
        b_rows = o["b"][q, :nb, 0].astype(np.int64)
        if np.isfinite(tau2[q]):
            r2 = o["a"][q, :na, 2].view(np.float32)
            assert np.array_equal(np.sort(b_rows), np.sort(a_rows[r2 >= tau2[q]]))  # stage B: f32 score >= tau2
        if (o["qu"][q, 0] & 2) or (o["qu"][q, 1] & 1) or not np.isfinite(tau[q]):
            continue
        # proven: every row outside the re-rank lies beyond the proof's bound, which sorts after the k-th value
        rr = o["rr"][q, :ne].astype(np.int64)
        vk = np.sort(refv[q, rr])[::-1][k - 1] if desc else np.sort(refv[q, rr])[k - 1]
        out_a = valid.copy()
        out_a[a_rows] = False
        bound_a = R.proof_bound(tau[q], beps[q], eref, o["qmag"][q], desc)
        bounds = [(out_a, bound_a)]
        if np.isfinite(tau2[q]):
            out_b = np.zeros(n, bool)
            out_b[np.setdiff1d(a_rows, b_rows)] = True
            bounds.append((out_b, R.proof_bound(tau2[q], beps2[q], eref, o["qmag"][q], desc)))
        for outside, bnd in bounds:
            if desc:
                assert (refv[q, outside] <= bnd).all() and bnd < vk
            else:
                assert (refv[q, outside] >= bnd).all() and bnd > vk
    col.close()
