"""Filtered brute-force KNN (sdb_knn_*_filtered): per-query row bitmaps through the screens, the proof and the exact
kernel.  Every result is compared bit for bit (rows, distances, counts) with the CPU oracle run on the rows the query
may rank: oracle.knn_topk(corpus, q, metric, k, skip=skip | ~filter)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle import pyoracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_col(ctx, corpus, metric, skip=None, screen=None, streaming=True):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if corpus.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, corpus.shape[1], metric, dt, capacity=max(1, corpus.shape[0]))
    col.append(corpus)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if screen:
        col.set_screen(screen)
    col.set_schedule(streaming)
    return col


def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return pack_row_filter(np.asarray(masks, bool))


def oracle_check(corpus, queries, metric, k, masks, qf, rows, dist, cnt, skip=None, qs=None):
    n = corpus.shape[0]
    base = np.zeros(n, bool) if skip is None else np.asarray(skip, bool)
    for q in (range(queries.shape[0]) if qs is None else qs):
        sk = (base | ~masks[qf[q]]).astype(np.uint8)
        r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=sk)
        assert cnt[q] == r.size, (q, int(cnt[q]), r.size)
        assert list(rows[q, : cnt[q]]) == list(r), (q, rows[q, : cnt[q]], r)
        assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, dist[q, : cnt[q]], d)


def random_masks(rng, n, densities):
    return np.stack([rng.random(n) < p for p in densities])


# ---- 1. parity matrix: every screen, both schedules, F32 / F64, the screened metrics and the exact-only ones ----
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("screen", ["AUTO", "TC_BF16", "SIMT_F32", "NONE_EXACT"])
@pytest.mark.parametrize("streaming", [True, False])
def test_parity_matrix(ctx, dtype, metric, screen, streaming):
    rng = np.random.default_rng(zlib.crc32(f"{dtype}{metric}{screen}{streaming}".encode()))
    n, dim = 9000 + 37, 48  # not a multiple of 32 or 256
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    queries = rng.uniform(-1, 1, (5, dim))
    masks = random_masks(rng, n, [1.0, 0.5, 0.1, 0.01, 0.3])
    qf = np.array([0, 1, 2, 3, 4], np.uint32)
    col = make_col(ctx, corpus, metric, screen=screen, streaming=streaming)
    for k in (1, 10, 256, 257):
        rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
        oracle_check(corpus, queries, metric, k, masks, qf, rows, dist, cnt)


@pytest.mark.parametrize("metric", ["MANHATTAN", "CHEBYSHEV", "HAMMING", "JACCARD", "MINKOWSKI", "PEARSON"])
def test_exact_only_metrics(ctx, metric):
    rng = np.random.default_rng(len(metric))
    n, dim = 3000 + 5, 16
    corpus = rng.integers(-3, 4, (n, dim)).astype(np.float32)  # repeated values: Hamming / Jaccard see ties
    queries = rng.integers(-3, 4, (3, dim)).astype(np.float64)
    masks = random_masks(rng, n, [0.5, 0.05])
    qf = np.array([0, 1, 0], np.uint32)
    col = make_col(ctx, corpus, metric)
    rows, dist, cnt = col.knn(queries, 10, filters=pack(masks), query_filter=qf)
    if metric != "MINKOWSKI":
        oracle_check(corpus, queries, metric, 10, masks, qf, rows, dist, cnt)
        return
    for q in range(3):  # pow(): CUDA's libm and the host's differ by an ulp per term (tests/test_gpu_knn.py)
        r, d = O.knn_topk(corpus, queries[q], "minkowski", 10, skip=(~masks[qf[q]]).astype(np.uint8))
        assert cnt[q] == r.size and list(rows[q, : cnt[q]]) == list(r)
        np.testing.assert_allclose(dist[q, : cnt[q]], d, rtol=1e-12)


def test_k4096_and_chunked_batches(ctx):
    rng = np.random.default_rng(4096)
    n, dim = 20000 + 3, 32
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    masks = random_masks(rng, n, [0.5, 0.02, 0.3])
    col = make_col(ctx, corpus, "COSINE")
    q1 = rng.uniform(-1, 1, (2, dim))
    rows, dist, cnt = col.knn(q1, 4096, filters=pack(masks), query_filter=np.array([0, 1], np.uint32))
    oracle_check(corpus, q1, "COSINE", 4096, masks, [0, 1], rows, dist, cnt)
    for nq in (1025, 2100):  # query-chunked screen launches: the filter index follows the query's offset
        qs = rng.uniform(-1, 1, (nq, dim))
        qf = rng.integers(0, 3, nq).astype(np.uint32)
        for screen in ("TC_INT8", "TC_BF16"):
            col.set_screen(screen)
            rows, dist, cnt = col.knn(qs, 10, filters=pack(masks), query_filter=qf)
            oracle_check(corpus, qs, "COSINE", 10, masks, qf, rows, dist, cnt,
                         qs=list(range(0, nq, 37)) + [nq - 1, 1023, 1024])


# ---- 2. densities, the repair bar, an adversarial filter ----
def test_densities(ctx):
    rng = np.random.default_rng(11)
    n, dim, nq, k = 60000 + 17, 64, 64, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    col = make_col(ctx, corpus, "COSINE")
    for p in (1.0, 0.5, 0.1, 0.01):
        masks = random_masks(rng, n, [p])
        qf = np.zeros(nq, np.uint32)
        rows, dist, cnt = col.knn(queries, k, filters=pack(masks))
        st = col.stats()
        assert st["n_fallback"] + st["n_repaired"] <= 2 + nq // 64, (p, st)  # the unfiltered call's bar
        oracle_check(corpus, queries, "COSINE", k, masks, qf, rows, dist, cnt, qs=range(0, nq, 5))
    # exactly k rows, one row, none
    for n_pass in (k, 1, 0):
        m = np.zeros((1, n), bool)
        m[0, rng.choice(n, n_pass, replace=False)] = True
        rows, dist, cnt = col.knn(queries[:4], k, filters=pack(m))
        assert list(cnt) == [n_pass] * 4
        oracle_check(corpus, queries[:4], "COSINE", k, m, [0] * 4, rows, dist, cnt)


def test_adversarial_filter_removes_each_querys_top100(ctx):
    rng = np.random.default_rng(12)
    n, dim, nq, k = 40000 + 1, 64, 16, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    for screen in ("TC_INT8", "TC_BF16"):
        col = make_col(ctx, corpus, "COSINE", screen=screen)
        r100, _, _ = col.knn(queries, 100)
        masks = np.ones((nq, n), bool)
        for q in range(nq):
            masks[q, r100[q].astype(np.int64)] = False
        qf = np.arange(nq, dtype=np.uint32)
        rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
        oracle_check(corpus, queries, "COSINE", k, masks, qf, rows, dist, cnt)
        st = col.stats()
        assert st["n_fallback"] + st["n_repaired"] <= 2 + nq // 64, st


# ---- 3. mixed batches: 64 filters over 1024 queries, on both sides of the direct regime's bound ----
DIRECT_MAX_ROWS = 4096  # csrc/internal.cuh


def exact_count_masks(rng, n, counts):
    m = np.zeros((len(counts), n), bool)
    for i, c in enumerate(counts):
        m[i, rng.choice(n, int(c), replace=False)] = True
    return m


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_mixed_filters_match_single_query_calls(ctx, metric):
    rng = np.random.default_rng(13)
    n, dim, nq, k = 30000 + 9, 32, 1024, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    counts = np.unique(np.geomspace(n, 20, 60).astype(np.int64)).tolist()
    counts += [DIRECT_MAX_ROWS - 1, DIRECT_MAX_ROWS, DIRECT_MAX_ROWS + 1, k]
    counts = counts[:64] + [1] * (64 - len(counts[:64]))
    masks = exact_count_masks(rng, n, counts)
    qf = rng.integers(0, 64, nq).astype(np.uint32)
    col = make_col(ctx, corpus, metric)
    f = pack(masks)
    rows, dist, cnt = col.knn(queries, k, filters=f, query_filter=qf)
    st = col.stats()
    assert st["screen_used"] != 3 and st["n_passes"] > 0, st  # the screened sub-batch ran
    oracle_check(corpus, queries, metric, k, masks, qf, rows, dist, cnt, qs=range(0, nq, 7))
    # every filter once as a batch of its own: at most DIRECT_MAX_ROWS rows -> no screen, else screened
    for fi in range(64):
        q = int(np.nonzero(qf == fi)[0][0]) if (qf == fi).any() else fi
        r1, d1, c1 = col.knn(queries[q : q + 1], k, filters=f, query_filter=[fi])
        st = col.stats()
        assert (st["n_passes"] == 0 and st["screen_used"] == 3) == (counts[fi] <= DIRECT_MAX_ROWS), (fi, counts[fi], st)
        assert st["n_fallback"] == 0, st
        if qf[q] == fi:
            c = cnt[q]
            assert c1[0] == c and r1[0, :c].tobytes() == rows[q, :c].tobytes() and d1[0, :c].tobytes() == dist[q, :c].tobytes()
        oracle_check(corpus, queries[q : q + 1], metric, k, masks, [fi], r1, d1, c1)


def test_direct_regime_batches(ctx):
    """all-direct batches: no screen launch, the same answers as the screened path through set_skip"""
    rng = np.random.default_rng(18)
    n, dim, nq, k = 50000 + 3, 48, 300, 20
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    corpus[10] = 0.0  # a special row (zero norm) that passes
    queries = rng.uniform(-1, 1, (nq, dim))
    masks = exact_count_masks(rng, n, [DIRECT_MAX_ROWS, 500, 3])
    masks[1, 10] = True
    skip = np.zeros(n, np.uint8)
    skip[np.nonzero(masks[0])[0][:100]] = 1  # skipped rows with a set bit stay out
    col = make_col(ctx, corpus, "COSINE", skip=skip)
    removed = np.nonzero(masks[1])[0][-50:]  # (row 10, the special row, stays)
    col.remove(removed)
    skip_all = skip.astype(bool)
    skip_all[removed] = True
    qf = (np.arange(nq) % 3).astype(np.uint32)
    launches0 = ctx.kernel_launches()
    rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
    st = col.stats()
    assert st["screen_used"] == 3 and st["n_passes"] == 0 and st["n_fallback"] == 0, st
    assert ctx.kernel_launches() - launches0 < 20  # a handful of tail kernels, no screen passes
    oracle_check(corpus, queries, "COSINE", k, masks, qf, rows, dist, cnt, skip=skip_all)
    assert list(cnt[2::3]) == [3] * (nq // 3)
    for fi in range(3):  # the screened path on a corpus whose skip mask carries the filter
        sel = np.nonzero(qf == fi)[0]
        ref = make_col(ctx, corpus, "COSINE", skip=(skip_all | ~masks[fi]).astype(np.uint8))
        r2, d2, c2 = ref.knn(queries[sel], k)
        assert (c2 == cnt[sel]).all()
        for i, q in enumerate(sel):  # entries past the count are not part of the result
            assert r2[i, : c2[i]].tobytes() == rows[q, : cnt[q]].tobytes()
            assert d2[i, : c2[i]].tobytes() == dist[q, : cnt[q]].tobytes()
        ref.close()


# ---- 4. skip mask, tombstones, special rows; filtered == set_skip(~f) + finalize ----
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_corpus_state_interplay(ctx, metric):
    rng = np.random.default_rng(14)
    n, dim, nq, k = 12000 + 11, 64, 8, 20
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    corpus[5] = 0.0  # zero norm
    corpus[6, 3] = np.nan  # non-finite
    corpus[7, 2] = np.inf
    corpus[8] = 0.0
    corpus[8, 0] = 50.0  # one dominant component: an int8 outlier row
    queries = rng.uniform(-1, 1, (nq, dim))
    queries[1] = corpus[8].astype(np.float64) * 0.02
    skip = np.zeros(n, np.uint8)
    skip[rng.choice(n, 500, replace=False)] = 1
    skip[9] = 1
    col = make_col(ctx, corpus, metric, skip=skip)
    removed = rng.choice(n, 300, replace=False)
    col.remove(removed)
    skip_all = skip.astype(bool)
    skip_all[removed] = True
    masks = random_masks(rng, n, [0.7, 0.2])
    masks[0, [5, 6, 7, 8, 9]] = True  # special rows pass filter 0 (and skipped row 9: stays skipped)
    masks[0, removed[:50]] = True  # a set bit never brings a removed row back
    masks[1, [5, 6, 7, 8]] = False
    qf = np.array([0, 0, 1, 1, 0, 1, 0, 1], np.uint32)
    rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
    oracle_check(corpus, queries, metric, k, masks, qf, rows, dist, cnt, skip=skip_all)
    for q in range(nq):
        got = set(rows[q, : cnt[q]].tolist())
        assert not got & set(removed.tolist()) and 9 not in got
    # the same answers from a corpus whose skip mask carries the filter
    for fi in (0, 1):
        sel = np.nonzero(qf == fi)[0]
        ref = make_col(ctx, corpus, metric, skip=(skip_all | ~masks[fi]).astype(np.uint8))
        r2, d2, c2 = ref.knn(queries[sel], k)
        assert (c2 == cnt[sel]).all()
        for i, q in enumerate(sel):  # entries past the count are not part of the result
            assert r2[i, : c2[i]].tobytes() == rows[q, : cnt[q]].tobytes()
            assert d2[i, : c2[i]].tobytes() == dist[q, : cnt[q]].tobytes()
        ref.close()


# ---- 5. the repair ladder keeps every query's own filter ----
def test_repair_ladder_remaps_filters(ctx):
    rng = np.random.default_rng(77)
    n, dim, nq, k = 80000, 128, 256, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    center = rng.uniform(-1, 1, dim)
    corpus[1000:7000] = (center[None, :] + rng.normal(0, 2e-3, (6000, dim))).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    crowd = [5, 77, 130, 200, 201, 254]
    for q in crowd:
        queries[q] = center + rng.normal(0, 1e-3, dim)
    # every crowd query loses a different sixth of the cluster (5000 near-duplicates remain: more than the first
    # rung's lists hold), so a swapped filter changes its answer
    masks = np.ones((len(crowd) + 1, n), bool)
    for i in range(len(crowd)):
        masks[i + 1, 1000 + i * 1000 : 1000 + (i + 1) * 1000] = False
    qf = np.zeros(nq, np.uint32)
    for i, q in enumerate(crowd):
        qf[q] = i + 1
    col = make_col(ctx, corpus, "COSINE", screen="TC_INT8")
    rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
    st = col.stats()
    assert st["n_repaired"] > 0, st  # the crowd went through the repair sub-batch, with its remapped filters
    oracle_check(corpus, queries, "COSINE", k, masks, qf, rows, dist, cnt, qs=crowd + [0, 100, 255])
    for i, q in enumerate(crowd):
        r = rows[q].astype(np.int64)
        assert ((r >= 1000) & (r < 7000)).all() and not ((r - 1000) // 1000 == i).any(), (q, rows[q])


# ---- 7. the operator: KnnTopK(Filter(source)) ----
def test_language_filter_tests_through_operator(ctx):
    from surrealdb_b200 import Distance, KnnContext, KnnTopK
    from surrealdb_b200.operators import Filter, TableScan, Union
    KnnTopK.clear_column_cache()
    active = lambda r: r.get("active") is True  # noqa: E731
    # language-tests/tests/language/indexes/knn/bruteforce_knn_with_filter_new_executor.surql
    pts = TableScan("pts", [{"id": f"pts:{i+1}", "point": p, "active": a} for i, (p, a) in enumerate(
        [([10, 0], True), ([2, 0], False), ([3, 0], True), ([100, 0], True), ([50, 0], False)])], version=1)
    kc = KnnContext()
    op = KnnTopK(Filter(pts, active), "point", [1, 0], 2, Distance.Euclidean, ctx=ctx).with_knn_context(kc)
    out = op.execute()
    assert [r["id"] for r in out] == ["pts:3", "pts:1"] and kc == {"pts:3": 2.0, "pts:1": 9.0}
    assert op.name() == "KnnTopK"
    assert op.attrs() == [("field", "point"), ("k", "2"), ("distance", "Euclidean"), ("dimension", "2")]
    # bruteforce_knn_multisource_filter_new_executor.surql: Filter over Union(TableScan, TableScan)
    pts_a = TableScan("pts", [{"id": "pts:1", "point": [10, 0], "active": True},
                              {"id": "pts:2", "point": [2, 0], "active": False},
                              {"id": "pts:3", "point": [3, 0], "active": True}], version=7)
    pts_b = TableScan("pts2", [{"id": "pts2:1", "point": [1.5, 0], "active": False},
                               {"id": "pts2:2", "point": [4, 0], "active": True}], version=3)
    kc = KnnContext()
    out = KnnTopK(Filter(Union(pts_a, pts_b), active), "point", [1, 0], 2, Distance.Euclidean,
                  ctx=ctx).with_knn_context(kc).execute()
    assert [r["id"] for r in out] == ["pts:3", "pts2:2"] and kc == {"pts:3": 2.0, "pts2:2": 3.0}
    # three statements with different predicates stage the column once; a new table version stages it again
    ops = [KnnTopK(Filter(pts, pred), "point", [1, 0], 2, Distance.Euclidean, ctx=ctx)
           for pred in (active, lambda r: not r["active"], lambda r: r["point"][0] > 5)]
    outs = [[r["id"] for r in o.execute()] for o in ops]
    assert outs == [["pts:3", "pts:1"], ["pts:2", "pts:5"], ["pts:1", "pts:5"]]
    assert ops[0]._column is op._column and ops[1]._column is op._column and ops[2]._column is op._column
    pts.version = 2
    again = KnnTopK(Filter(pts, active), "point", [1, 0], 2, Distance.Euclidean, ctx=ctx)
    assert [r["id"] for r in again.execute()] == ["pts:3", "pts:1"] and again._column is not op._column
    KnnTopK.clear_column_cache()


# ---- 6. asynchrony, ownership, errors ----
def test_tickets_mixed_filtered_and_unfiltered(ctx):
    rng = np.random.default_rng(15)
    n, dim, nq, k = 20000 + 7, 64, 128, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    col = make_col(ctx, corpus, "COSINE")
    masks = random_masks(rng, n, [0.3, 0.05])
    f = np.ascontiguousarray(pack(masks))
    qs = [np.ascontiguousarray(rng.uniform(-1, 1, (nq, dim))) for _ in range(4)]
    qfs = [rng.integers(0, 2, nq).astype(np.uint32) for _ in range(4)]
    outs = [(np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32)) for _ in range(4)]
    tickets = []
    for i in range(4):  # slots 0..3 alternate the two streams
        o = outs[i]
        if i % 2 == 0:
            tickets.append(col.submit_host_filtered(qs[i].ctypes.data, nq, k, f.ctypes.data, 2, qfs[i], o[0].ctypes.data,
                                                    o[1].ctypes.data, o[2].ctypes.data))
        else:
            tickets.append(col.submit_host(qs[i].ctypes.data, nq, k, o[0].ctypes.data, o[1].ctypes.data,
                                           o[2].ctypes.data))
    for t in tickets[::-1]:
        col.wait(t)
    for i in range(4):
        if i % 2 == 0:
            r, d, c = col.knn(qs[i], k, filters=f, query_filter=qfs[i])
        else:
            r, d, c = col.knn(qs[i], k)
        assert (c == outs[i][2]).all()
        for q in range(nq):  # entries past the count are not part of the result
            assert r[q, : c[q]].tobytes() == outs[i][0][q, : c[q]].tobytes()
            assert d[q, : c[q]].tobytes() == outs[i][1][q, : c[q]].tobytes()
    oracle_check(corpus, qs[0], "COSINE", k, masks, qfs[0], outs[0][0], outs[0][1], outs[0][2], qs=range(0, nq, 9))


def test_device_entry_point(ctx):
    import torch
    rng = np.random.default_rng(16)
    n, dim, nq, k = 10000 + 5, 32, 9, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    col = make_col(ctx, corpus, "EUCLIDEAN")
    masks = random_masks(rng, n, [0.5, 0.01, 0.2])
    qf = (np.arange(nq) % 3).astype(np.uint32)
    queries = rng.uniform(-1, 1, (nq, dim))
    dq = torch.from_numpy(queries).cuda()
    df = torch.from_numpy(pack(masks).view(np.int32)).cuda()
    rows = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    dist = torch.zeros((nq, k), dtype=torch.float64, device="cuda")
    cnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
    col.knn_device_filtered(dq.data_ptr(), nq, k, df.data_ptr(), 3, qf, 1000, rows.data_ptr(), dist.data_ptr(),
                            cnt.data_ptr())
    r, d, c = rows.cpu().numpy().astype(np.uint64), dist.cpu().numpy(), cnt.cpu().numpy().astype(np.uint32)
    assert (r[c > 0, 0] >= 1000).all()
    for q in range(nq):
        r[q, : c[q]] -= 1000
    oracle_check(corpus, queries, "EUCLIDEAN", k, masks, qf, r, d, c)


def test_errors_cancellation_and_ownership():
    from surrealdb_b200 import Context, SdbError
    from surrealdb_b200 import _lib as L
    live0 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live0[0]), C.byref(live0[1]))
    ctx = Context(0)  # its own context: everything this test allocates is released by the two closes below
    rng = np.random.default_rng(17)
    n, dim = 5000, 16
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    col = make_col(ctx, corpus, "COSINE")
    q = rng.uniform(-1, 1, (3, dim))
    f = pack(random_masks(rng, n, [0.5, 0.5]))
    with pytest.raises(SdbError) as e:
        col.knn(q, 5, filters=f, query_filter=np.array([0, 2, 1], np.uint32))
    assert e.value.status == L.SDB_EINVAL
    with pytest.raises(SdbError) as e:  # packed for another row count
        col.knn(q, 5, filters=pack(random_masks(rng, n + 40, [0.5])))
    assert e.value.status == L.SDB_EINVAL
    rows = np.zeros((3, 5), np.uint64)
    dist = np.zeros((3, 5), np.float64)
    cnt = np.zeros(3, np.uint32)
    qa = np.ascontiguousarray(q)
    p = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    assert L.lib().sdb_knn_bruteforce_filtered(col.h, p(qa), 3, 5, p(f), 0, None, p(rows), p(dist), p(cnt),
                                               None) == L.SDB_EINVAL
    assert L.lib().sdb_knn_bruteforce_filtered(col.h, p(qa), 3, 5, None, 2, None, p(rows), p(dist), p(cnt),
                                               None) == L.SDB_EINVAL
    flag = np.ones(1, np.int32)
    assert L.lib().sdb_knn_bruteforce_filtered(col.h, p(qa), 3, 5, p(f), 2, None, p(rows), p(dist), p(cnt),
                                               p(flag)) == L.SDB_ECANCELLED
    ctx.cancel()
    try:
        with pytest.raises(SdbError) as e:
            col.knn(q, 5, filters=f)
        assert e.value.status == L.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    col.knn(q, 5, filters=f)
    col.close()
    ctx.close()
    live1 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live1[0]), C.byref(live1[1]))
    assert (live1[0].value, live1[1].value) == (live0[0].value, live0[1].value)
