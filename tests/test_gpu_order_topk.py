"""`ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k` on a cached column (sdb_corpus_order_*): every result against
the SortTopK reference over the CPU oracle's values (tests/sort_topk_ref.py), bit for bit; the KNN ranking against
sdb_knn_bruteforce[_filtered]; the screened cosine-similarity DESC against the exact kernel at production shape;
tickets, cancellation, refusals and ownership."""
import ctypes as C

import numpy as np
import pytest

from sort_topk_ref import FN_IDS, row_values, sort_keyed

pytestmark = pytest.mark.gpu

FNS = list(FN_IDS)
KS = [1, 10, 256, 257, 1000, 4096]


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_col(ctx, corpus, metric, skip=None):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if corpus.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, corpus.shape[1], metric, dt, capacity=max(1, corpus.shape[0]))
    col.append(corpus)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    return col


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def check_result(rows, vals, cnt, er, ev, k, close=False):
    """k <= 1000: rows and values bit for bit.  Above, the reference sorts unstably: the value sequence bit for bit and
    the rows of each group of equal values as sets.  close: values to 1e-12 relative (MINKOWSKI's pow())."""
    assert int(cnt) == er.size, (int(cnt), er.size)
    r, v = rows[: er.size], vals[: er.size]
    if close:
        assert np.allclose(v, ev, rtol=1e-12, atol=0, equal_nan=True)
    else:
        assert np.array_equal(_bits(v), _bits(ev)), (v, ev)
    if k <= 1000:
        assert np.array_equal(r, er), (r, er)
        return
    j = 0
    while j < er.size:
        e = j
        while e < er.size and _bits(ev[e:e + 1])[0] == _bits(ev[j:j + 1])[0]:
            e += 1
        assert set(r[j:e].tolist()) == set(er[j:e].tolist())
        j = e


def mixed_corpus(rng, n, d, dtype):
    """integer-valued rows (many duplicates: tie groups that k cuts), random rows, and the special rows: zero, NaN,
    +-inf, a row with -0.0"""
    ints = rng.integers(-2, 3, size=(n // 2, d)).astype(np.float64)
    reals = rng.standard_normal((n - n // 2, d))
    x = np.concatenate([ints, reals])
    rng.shuffle(x)
    x[3] = 0.0
    x[7, 2] = np.nan
    x[11, 0] = np.inf
    x[13, 1] = -np.inf
    x[17] = -0.0
    return x.astype(dtype)


# ---- 1. every fn x ASC/DESC x F32/F64, filtered and unfiltered, k across the heap / full-sort boundary ------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("fn", FNS)
def test_every_function_and_order(ctx, dtype, fn):
    rng = np.random.default_rng(101 + FNS.index(fn))
    n, d = 3000, 8
    x = mixed_corpus(rng, n, d, dtype)
    skip = np.zeros(n, np.uint8)
    skip[rng.choice(n, 40, replace=False)] = 1
    # the corpus metric decides the route: COSINE serves SIMILARITY_COSINE DESC on the screens, the others the exact
    # kernel; PEARSON and HAMMING corpora take their own metric's function on the KNN path
    metric = "COSINE" if fn in ("SIMILARITY_COSINE", "DOT", "MAGNITUDE") else fn
    col = make_col(ctx, x, metric, skip)
    queries = np.stack([rng.integers(-2, 3, size=d).astype(np.float64), rng.standard_normal(d)])
    code = FN_IDS[fn]
    from surrealdb_b200.engine import pack_row_filter
    masks = np.stack([rng.random(n) < 0.5, np.zeros(n, bool)])  # the second passes nothing
    masks[0, :50] = True
    filt = pack_row_filter(masks)
    vals = [row_values(code, x, q if fn != "MAGNITUDE" else None) for q in queries]
    live = ~skip.astype(bool)
    for order in ("ASC", "DESC"):
        for k in KS:
            rows, got, cnt = col.order_topk(queries, k, fn, order)
            for qi in range(2):
                er, ev = sort_keyed(vals[qi], k, order == "DESC", live)
                check_result(rows[qi], got[qi], cnt[qi], er, ev, k, close=fn == "MINKOWSKI")
            qf = np.array([0, 1], np.uint32)
            rows, got, cnt = col.order_topk(queries, k, fn, order, filters=filt, query_filter=qf)
            for qi in range(2):
                er, ev = sort_keyed(vals[qi], k, order == "DESC", live & masks[qf[qi]])
                check_result(rows[qi], got[qi], cnt[qi], er, ev, k, close=fn == "MINKOWSKI")
            assert cnt[1] == 0  # the fully filtered query


def test_small_and_empty_columns(ctx):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((5, 4)).astype(np.float32)
    col = make_col(ctx, x, "COSINE")
    q = rng.standard_normal((1, 4))
    for fn in ("SIMILARITY_COSINE", "DOT", "EUCLIDEAN"):
        for order in ("ASC", "DESC"):
            rows, got, cnt = col.order_topk(q, 10, fn, order)
            er, ev = sort_keyed(row_values(FN_IDS[fn], x, q[0]), 10, order == "DESC")
            check_result(rows[0], got[0], cnt[0], er, ev, 10)
    rows, got, cnt = col.order_topk(q, 0, "DOT", "DESC")
    assert cnt.tolist() == [0]
    # MAGNITUDE takes no query
    rows, got, cnt = col.order_topk(None, 3, "MAGNITUDE", "DESC")
    er, ev = sort_keyed(row_values(18, x, None), 3, True)
    check_result(rows[0], got[0], cnt[0], er, ev, 3)


# ---- 2. the KNN ranking: fn = the corpus metric, ASC, byte for byte the KNN calls ---------------------------------
@pytest.mark.parametrize("metric", ["CHEBYSHEV", "COSINE", "EUCLIDEAN", "HAMMING", "JACCARD", "MANHATTAN", "MINKOWSKI",
                                    "PEARSON"])
def test_metric_ascending_is_knn(ctx, metric):
    rng = np.random.default_rng(31)
    centers = rng.standard_normal((40, 32))
    x = (centers[rng.integers(0, 40, 20000)] + 0.2 * rng.standard_normal((20000, 32))).astype(np.float32)
    if metric in ("HAMMING", "JACCARD"):
        x = np.round(x).astype(np.float32)
    col = make_col(ctx, x, metric)
    q = (x[rng.choice(20000, 16)] + 0.05 * rng.standard_normal((16, 32))).astype(np.float64)
    if metric in ("HAMMING", "JACCARD"):
        q = np.round(q)
    from surrealdb_b200.engine import pack_row_filter
    filt = pack_row_filter(np.stack([rng.random(20000) < 0.3, rng.random(20000) < 0.001]))
    qf = (np.arange(16) % 2).astype(np.uint32)
    for k in (10, 300):
        a = col.order_topk(q, k, metric, "ASC")
        b = col.knn(q, k)
        for u, v in zip(a, b):
            assert u.tobytes() == v.tobytes()
        a = col.order_topk(q, k, metric, "ASC", filters=filt, query_filter=qf)
        b = col.knn(q, k, filters=filt, query_filter=qf)
        for u, v in zip(a, b):
            assert u.tobytes() == v.tobytes()


# ---- 3. near ties: fl(1 - s) merges similarities a few ulps apart; s DESC must still order them -------------------
def test_cosine_desc_near_ties(ctx):
    n = 512
    # s ~ 0.1 (ulp 1.4e-17) while 1 - s has ulp 1.1e-16: about eight similarities share each distance
    c = 0.1 + np.arange(n) * 2.0 ** -56   # one ulp apart; scan order = similarity ascending
    x = np.stack([c, np.sqrt(1.0 - c * c)], axis=1)
    col = make_col(ctx, x, "COSINE")
    q = np.array([[1.0, 0.0]])
    s = row_values(16, x, q[0])
    k = 10
    er, ev = sort_keyed(s, k, True)
    knn_rows, _, _ = col.knn(q, k)
    # the test discriminates: the KNN order (distance, then scan position) is not the similarity order here
    assert not np.array_equal(knn_rows[0], er)
    assert not np.array_equal(knn_rows[0][::-1], er)
    rows, got, cnt = col.order_topk(q, k, "SIMILARITY_COSINE", "DESC")
    check_result(rows[0], got[0], cnt[0], er, ev, k)


# ---- 4. the screens serve cosine similarity DESC and PEARSON DESC at production shape; results equal the exact
# kernel's for every query of the batch ---------------------------------------------------------------------------
@pytest.mark.parametrize("metric,fn", [("COSINE", "SIMILARITY_COSINE"), ("PEARSON", "PEARSON")])
@pytest.mark.parametrize("screen", ["TC_INT8", "TC_BF16"])
def test_desc_screened_at_scale(ctx, screen, metric, fn):
    import torch
    from surrealdb_b200 import VectorColumn
    n, d, nq = 1_000_000, 768, 1024
    g = torch.Generator(device="cuda").manual_seed(11)
    centers = torch.randn(2000, d, device="cuda", generator=g)
    col = VectorColumn(ctx, d, metric, "F32", capacity=n)
    step = 250_000
    for i in range(0, n, step):
        idx = torch.randint(0, 2000, (step,), device="cuda", generator=g)
        rows = (centers[idx] + 0.4 * torch.randn(step, d, device="cuda", generator=g)).contiguous()
        col.append_device(rows.data_ptr(), step)
        torch.cuda.synchronize()
        del rows
    col.finalize()
    qi = torch.randint(0, 2000, (nq,), device="cuda", generator=g)
    q = (centers[qi] + 0.4 * torch.randn(nq, d, device="cuda", generator=g)).double().cpu().numpy()
    for k in (10, 256):
        col.set_screen(screen)
        got = col.order_topk(q, k, fn, "DESC")
        st = col.stats()
        assert st["screen_used"] in (2, 4), st  # a tensor-core screen ranked the batch
        # most queries are proven on the first screen's candidates: neither repaired on a later rung nor re-ranked by
        # the exact kernel (either proof refusing every query shows here)
        assert st["n_fallback"] + st["n_repaired"] <= nq // 4, st
        col.set_screen("NONE_EXACT")
        ref = col.order_topk(q, k, fn, "DESC")
        for u, v in zip(got, ref):
            assert u.tobytes() == v.tobytes()


# ---- 4b. HAMMING / JACCARD in both directions on the count path: exact under ties that k cuts ---------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("metric", ["HAMMING", "JACCARD"])
def test_count_path_both_directions(ctx, metric, dtype):
    rng = np.random.default_rng(77)
    n, d, nq = 6000, 12, 4
    x = rng.integers(0, 2 if metric == "HAMMING" else 4, size=(n, d)).astype(dtype)  # few distinct values: many ties
    skip = np.zeros(n, np.uint8)
    skip[rng.choice(n, 30, replace=False)] = 1
    col = make_col(ctx, x, metric, skip)
    q = rng.integers(0, 2 if metric == "HAMMING" else 4, size=(nq, d)).astype(np.float64)
    vals = [row_values(FN_IDS[metric], x, qq) for qq in q]
    from surrealdb_b200.engine import pack_row_filter
    mask = rng.random(n) < 0.8  # more than 4096 passing rows: screened (counted), not the direct regime
    live = ~skip.astype(bool)
    for order in ("ASC", "DESC"):
        for k in (1, 37, 256):
            for filt in (None, mask):
                if filt is None:
                    rows, got, cnt = col.order_topk(q, k, metric, order)
                else:
                    rows, got, cnt = col.order_topk(q, k, metric, order, filters=pack_row_filter(filt))
                st = col.stats()
                assert st["screen_used"] == 1 and st["n_passes"] == 1, st  # the count path ranked the batch
                for qi in range(nq):
                    er, ev = sort_keyed(vals[qi], k, order == "DESC", live if filt is None else live & filt)
                    check_result(rows[qi], got[qi], cnt[qi], er, ev, k)


# ---- 5. tickets: order and KNN batches in flight together, completed in any order; cancellation -----------------
def test_tickets_mixed_with_knn_and_cancel(ctx):
    from surrealdb_b200 import _lib
    rng = np.random.default_rng(9)
    x = rng.standard_normal((30000, 64)).astype(np.float32)
    col = make_col(ctx, x, "COSINE")
    q = rng.standard_normal((32, 64))
    k = 20
    kinds = [("SIMILARITY_COSINE", "DESC"), None, ("DOT", "DESC"), ("MANHATTAN", "ASC")]
    bufs, tickets = [], []
    for kind in kinds:
        rows = np.zeros((32, k), np.uint64)
        vals = np.zeros((32, k), np.float64)
        cnt = np.zeros(32, np.uint32)
        bufs.append((rows, vals, cnt))
        if kind is None:
            t = col.submit_host(q.ctypes.data, 32, k, rows.ctypes.data, vals.ctypes.data, cnt.ctypes.data)
        else:
            t = col.order_submit_host(q.ctypes.data, 32, k, kind[0], kind[1], rows.ctypes.data, vals.ctypes.data,
                                      cnt.ctypes.data)
        tickets.append(t)
    with pytest.raises(_lib.SdbError):  # a fifth batch finds no free slot
        col.order_submit_host(q.ctypes.data, 32, k, "DOT", "ASC", bufs[0][0].ctypes.data, bufs[0][1].ctypes.data,
                              bufs[0][2].ctypes.data)
    for t in reversed(tickets):
        col.wait(t)
    for kind, (rows, vals, cnt) in zip(kinds, bufs):
        ref = col.knn(q, k) if kind is None else col.order_topk(q, k, kind[0], kind[1])
        for u, v in zip((rows, vals, cnt), ref):
            assert u.tobytes() == v.tobytes(), kind
    # device variants equal the host ones
    import torch
    dq = torch.from_numpy(q).cuda()
    dr = torch.zeros((32, k), dtype=torch.int64, device="cuda")
    dv = torch.zeros((32, k), dtype=torch.float64, device="cuda")
    dc = torch.zeros(32, dtype=torch.int32, device="cuda")
    col.order_topk_device(dq.data_ptr(), 32, k, "DOT", "DESC", 0, dr.data_ptr(), dv.data_ptr(), dc.data_ptr())
    ref = col.order_topk(q, k, "DOT", "DESC")
    assert dr.cpu().numpy().view(np.uint64).tobytes() == ref[0].tobytes()
    assert dv.cpu().numpy().tobytes() == ref[1].tobytes()
    t = col.order_submit_device(dq.data_ptr(), 32, k, "SIMILARITY_COSINE", "DESC", 7, dr.data_ptr(), dv.data_ptr(),
                                dc.data_ptr())
    col.wait(t)
    ref = col.order_topk(q, k, "SIMILARITY_COSINE", "DESC")
    assert (dr.cpu().numpy().view(np.uint64) - 7).tobytes() == ref[0].tobytes()
    assert dv.cpu().numpy().tobytes() == ref[1].tobytes()
    # a cancel raised while an exact-kernel batch is in flight surfaces from its wait
    rows, vals, cnt = bufs[0]
    t = col.order_submit_host(q.ctypes.data, 32, k, "DOT", "DESC", rows.ctypes.data, vals.ctypes.data,
                              cnt.ctypes.data)
    ctx.cancel()
    try:
        with pytest.raises(_lib.SdbError) as e:
            col.wait(t)
        assert e.value.status == _lib.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    rows2, _, _ = col.order_topk(q, k, "DOT", "DESC")  # the column keeps answering
    assert rows2.shape == (32, k)


# ---- 6. refusals and ownership ----------------------------------------------------------------------------------
def _live():
    from surrealdb_b200 import _lib
    n, b = C.c_uint64(), C.c_uint64()
    _lib.lib().sdb_debug_live_allocations(C.byref(n), C.byref(b))
    return n.value, b.value


def test_refusals_and_ownership(ctx):
    from surrealdb_b200 import _lib
    L = _lib.lib()
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2000, 16)).astype(np.float32)
    col = make_col(ctx, x, "COSINE")
    q = rng.standard_normal((4, 16))
    rows = np.zeros((4, 5000), np.uint64)
    vals = np.zeros((4, 5000), np.float64)
    cnt = np.zeros(4, np.uint32)
    out = (rows.ctypes.data, vals.ctypes.data, cnt.ctypes.data)
    assert L.sdb_corpus_order_topk(col.h, q.ctypes.data, 4, 99, 0, 5, None, 0, None, *out) == _lib.SDB_EINVAL
    assert L.sdb_corpus_order_topk(col.h, q.ctypes.data, 4, 17, 2, 5, None, 0, None, *out) == _lib.SDB_EINVAL
    assert L.sdb_corpus_order_topk(col.h, None, 4, 17, 0, 5, None, 0, None, *out) == _lib.SDB_EINVAL
    assert L.sdb_corpus_order_topk(col.h, q.ctypes.data, 4, 17, 1, 4097, None, 0, None, *out) == \
        _lib.SDB_EUNSUPPORTED
    for fn in ("SIMILARITY_COSINE", "DOT", "COSINE"):  # warm every scratch buffer the calls grow
        col.order_topk(q, 300, fn, "DESC")
        col.order_topk(q, 10, fn, "DESC", filters=col_filter(x.shape[0]))
    before = _live()
    for fn in ("SIMILARITY_COSINE", "DOT", "COSINE"):
        col.order_topk(q, 300, fn, "DESC")
        col.order_topk(q, 10, fn, "DESC", filters=col_filter(x.shape[0]))
    assert _live() == before


def col_filter(n):
    from surrealdb_b200.engine import pack_row_filter
    return pack_row_filter(np.arange(n) % 3 == 0)


# ---- 7. the operator mirror: Compute + SortTopK over a (filtered) table scan --------------------------------------
def test_sort_topk_operator(ctx):
    from surrealdb_b200 import Filter, SdbError, SortTopK, TableScan
    rng = np.random.default_rng(21)
    x = rng.standard_normal((500, 8)).astype(np.float32)
    recs = [{"id": i, "emb": [float(v) for v in x[i]], "lang": "en" if i % 3 else "fr"} for i in range(500)]
    q = list(rng.standard_normal(8))
    op = SortTopK(TableScan("doc", recs, 1), "emb", "vector::similarity::cosine", q, 7, "DESC", alias="score",
                  ctx=ctx)
    assert op.name() == "SortTopK"
    assert op.attrs() == [("order_by", "vector::similarity::cosine(emb, $q) DESC"), ("limit", "7")]
    out = op.execute()
    er, ev = sort_keyed(row_values(16, x, q), 7, True)
    assert [r["id"] for r in out] == er.tolist()
    assert _bits([r["score"] for r in out]).tolist() == _bits(ev).tolist()
    flt = Filter(TableScan("doc", recs, 1), lambda r: r["lang"] == "fr")
    out = SortTopK(flt, "emb", "vector::dot", q, 4, "ASC", ctx=ctx).execute()
    passes = np.array([r["lang"] == "fr" for r in recs])
    er, _ = sort_keyed(row_values(17, x, q), 4, False, passes)
    assert [r["id"] for r in out] == er.tolist()
    out = SortTopK(TableScan("doc", recs, 1), "emb", "vector::magnitude", None, 3, "DESC", dim=8, ctx=ctx).execute()
    er, _ = sort_keyed(row_values(18, x, None), 3, True)
    assert [r["id"] for r in out] == er.tolist()
    with pytest.raises(SdbError):  # a ranked row without a vector: the reference raises, the GPU does not rank it
        SortTopK(TableScan("doc", recs + [{"id": 500}], 2), "emb", "vector::dot", q, 3, "DESC", ctx=ctx).execute()
