"""Parity of the CUDA brute-force KNN path (through the C ABI) with the CPU oracle: returned rows,
their order and the f64 distances must be IDENTICAL (bit-exact), for every screen."""
import numpy as np
import pytest

from oracle import pyoracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_col(ctx, corpus, metric, skip=None, screen=None):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if corpus.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, corpus.shape[1], metric, dt, capacity=max(1, corpus.shape[0]))
    if corpus.shape[0]:
        col.append(corpus)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if screen:
        col.set_screen(screen)
    return col


def check(col, corpus, queries, metric, k, skip=None):
    rows, dist, cnt = col.knn(queries, k)
    for q in range(queries.shape[0]):
        r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=skip)
        assert cnt[q] == r.size, (q, cnt[q], r.size)
        assert list(rows[q, : cnt[q]]) == list(r), (q, rows[q], r)
        assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, dist[q], d)  # bit-exact incl. NaN sign


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("dim", [7, 100, 128, 768])
@pytest.mark.parametrize("screen", ["SIMT_F32", "TC_BF16", "TC_INT8", "NONE_EXACT"])
def test_random_parity(ctx, metric, dim, screen):
    rng = np.random.default_rng(dim * 7 + len(metric))
    n = 20000 if dim <= 128 else 6000
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (11, dim))
    col = make_col(ctx, corpus, metric, screen=screen)
    nqs = (1, 3, 11) if screen != "NONE_EXACT" else (2,)
    for nq in nqs:
        for k in (1, 10, 100):
            check(col, corpus, queries[:nq], metric, k)
    st = col.stats()
    if screen == "NONE_EXACT":
        assert st["n_fallback"] == 2


def test_c1_f64_single_query(ctx):
    # BASELINE config 0: 100k x 128, values uniform(-20,20) as f64 (reference generator range), 1 query, k=10
    rng = np.random.default_rng(0x5DB00000)
    corpus = rng.uniform(-20, 20, (100_000, 128))
    q = rng.uniform(-20, 20, (1, 128))
    for metric in ("COSINE", "EUCLIDEAN"):
        col = make_col(ctx, corpus, metric)
        check(col, corpus, q, metric, 10)


def test_language_test_vectors_through_operator(ctx):
    # language-tests/tests/language/indexes/knn/bruteforce_knn_new_executor.surql
    from surrealdb_b200 import Distance, KnnContext, KnnTopK
    pts = [{"id": f"pts:{i+1}", "point": p} for i, p in enumerate([[10, 0], [2, 0], [3, 0], [100, 0], [50, 0]])]
    kc = KnnContext()
    op = KnnTopK(pts, "point", [1, 0], 2, Distance.Euclidean, ctx=ctx).with_knn_context(kc)
    out = op.execute()
    assert [r["id"] for r in out] == ["pts:2", "pts:3"]
    assert kc == {"pts:2": 1.0, "pts:3": 2.0}
    assert op.name() == "KnnTopK"
    assert op.attrs() == [("field", "point"), ("k", "2"), ("distance", "Euclidean"), ("dimension", "2")]
    # hnsw_knn_new_executor.surql brute-force leg: pts:3 has no `point` at first -> skipped
    pts = [{"id": "pts:1", "point": [1, 2, 3, 4]}, {"id": "pts:2", "point": [4, 5, 6, 7]}, {"id": "pts:3"}]
    kc = KnnContext()
    out = KnnTopK(pts, "point", [2, 3, 4, 5], 2, Distance.Euclidean, ctx=ctx).with_knn_context(kc).execute()
    assert [r["id"] for r in out] == ["pts:1", "pts:2"] and kc == {"pts:1": 2.0, "pts:2": 4.0}
    # rows with a wrong dimension / non-numeric element are skipped, never an error (knn_topk.rs:199-210)
    pts = [{"id": "a", "v": [1.0, 1.0]}, {"id": "b", "v": [1.0]}, {"id": "c", "v": ["x", 1.0]}, {"id": "d", "v": []},
           {"id": "e", "v": [0.5, 0.0]}]
    out = KnnTopK(pts, "v", [0.0, 0.0], 5, Distance.Euclidean, ctx=ctx).execute()
    assert [r["id"] for r in out] == ["e", "a"]


def test_edge_cases(ctx):
    rng = np.random.default_rng(4)
    dim = 16
    corpus = rng.uniform(-1, 1, (300, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (3, dim))
    for metric in ("COSINE", "EUCLIDEAN"):
        col = make_col(ctx, corpus, metric)
        check(col, corpus, queries, metric, 1000)  # k > n
        rows, dist, cnt = col.knn(queries, 0)      # k == 0
        assert list(cnt) == [0, 0, 0]
        skip = (rng.uniform(0, 1, 300) < 0.5).astype(np.uint8)
        col = make_col(ctx, corpus, metric, skip=skip)
        check(col, corpus, queries, metric, 20, skip=skip)
        col = make_col(ctx, corpus, metric, skip=np.ones(300, np.uint8))  # everything skipped
        rows, dist, cnt = col.knn(queries, 5)
        assert list(cnt) == [0, 0, 0]
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, dim, "COSINE", "F32", capacity=8)  # empty corpus
    col.finalize()
    rows, dist, cnt = col.knn(queries, 5)
    assert list(cnt) == [0, 0, 0]


def test_ties_resolved_by_scan_order(ctx):
    rng = np.random.default_rng(5)
    base = rng.uniform(-1, 1, (50, 32)).astype(np.float32)
    corpus = np.concatenate([base, base, base[::-1], base])  # exact duplicates => exact distance ties
    queries = rng.uniform(-1, 1, (9, 32))
    for metric in ("COSINE", "EUCLIDEAN"):
        for screen in ("SIMT_F32", "TC_BF16", "TC_INT8"):
            col = make_col(ctx, corpus, metric, screen=screen)
            check(col, corpus, queries, metric, 10)
            check(col, corpus, queries[:2], metric, 57)


def test_zero_and_nan_rows_and_queries(ctx):
    rng = np.random.default_rng(6)
    corpus = rng.uniform(-1, 1, (500, 24)).astype(np.float32)
    corpus[7] = 0.0          # zero vector: cosine distance = generated NaN (negative on x86-64) -> sorts first
    corpus[100] = 0.0
    corpus[33, 5] = np.nan   # data NaN (positive) -> sorts last
    corpus[44, 0] = np.inf
    queries = rng.uniform(-1, 1, (4, 24))
    queries[1] = 0.0         # zero query: every cosine distance is NaN -> first k rows in scan order
    queries[2, 3] = np.nan
    for metric in ("COSINE", "EUCLIDEAN"):
        for screen in ("SIMT_F32", "TC_BF16", "TC_INT8"):
            col = make_col(ctx, corpus, metric, screen=screen)
            check(col, corpus, queries, metric, 10)
            check(col, corpus, queries, metric, 499)


def test_adversarial_cluster_forces_exact_fallback(ctx):
    # near-duplicate rows: the bf16/f32 screens cannot separate them, the proof fails and the exact kernel
    # must take over -- results still identical to the oracle.
    rng = np.random.default_rng(8)
    center = rng.uniform(-1, 1, 64).astype(np.float32)
    corpus = (center[None, :] + rng.normal(0, 1e-6, (30000, 64))).astype(np.float32)
    queries = (center[None, :] + rng.normal(0, 1e-3, (12, 64))).astype(np.float64)
    for screen in ("SIMT_F32", "TC_BF16", "TC_INT8"):
        col = make_col(ctx, corpus, "COSINE", screen=screen)
        check(col, corpus, queries, "COSINE", 10)
    col = make_col(ctx, corpus, "EUCLIDEAN", screen="TC_BF16")
    check(col, corpus, queries, "EUCLIDEAN", 10)


def test_synthetic_generator_matches_oracle(ctx):
    from surrealdb_b200 import VectorColumn
    n, dim = 5000, 96
    col = VectorColumn(ctx, dim, "COSINE", "F32", capacity=n)
    col.append_synthetic(seed=77, first_row=1000, n=n)  # rows 1000.. of the global synthetic corpus
    col.finalize()
    corpus = O.gen_f32(77, 1000 * dim, n * dim).reshape(n, dim)
    queries = O.gen_f32(78, 0, 5 * dim).reshape(5, dim).astype(np.float64)
    check(col, corpus, queries, "COSINE", 10)


def test_full_size_c2_sample_queries(ctx):
    # BASELINE config 1 shape (1M x 768 f32, batch cosine k=10): full-size corpus on the GPU; the oracle
    # checks a sample of the batch (one query costs it ~2 s), every query is checked for the
    # size-independent properties (sorted, unique rows, count == k).
    from surrealdb_b200 import VectorColumn
    n, dim, nq, k = 1_000_000, 768, 64, 10
    col = VectorColumn(ctx, dim, "COSINE", "F32", capacity=n)
    col.append_synthetic(seed=0x5DB00001, first_row=0, n=n)
    col.finalize()
    queries = O.gen_f32(0x5DB0FFFF, 0, nq * dim).reshape(nq, dim).astype(np.float64)
    rows, dist, cnt = col.knn(queries, k)
    assert (cnt == k).all()
    assert (np.diff(dist, axis=1) >= 0).all()
    assert all(len(set(r)) == k for r in rows.tolist())
    corpus = O.gen_f32(0x5DB00001, 0, n * dim).reshape(n, dim)
    for q in (0, 31, 63):
        r, d = O.knn_topk(corpus, queries[q], "cosine", k)
        assert list(rows[q]) == list(r) and dist[q].tobytes() == d.tobytes()
    for screen in ("SIMT_F32", "TC_BF16", "TC_INT8"):  # every screen gives the same bits on the same corpus
        col.set_screen(screen)
        rows1, dist1, _ = col.knn(queries[:9], k)
        assert rows1.tobytes() == rows[:9].tobytes() and dist1.tobytes() == dist[:9].tobytes(), screen
        assert col.stats()["screen_used"] == {"SIMT_F32": 1, "TC_BF16": 2, "TC_INT8": 4}[screen]


def test_large_batches_are_chunked_correctly(ctx):
    # batches above 2048 queries are split over several tensor-core screen launches (private sub-list slots per chunk)
    rng = np.random.default_rng(21)
    corpus = rng.uniform(-1, 1, (9000, 64)).astype(np.float32)
    queries = rng.uniform(-1, 1, (4500, 64))
    for screen, metric in (("TC_BF16", "EUCLIDEAN"), ("TC_INT8", "COSINE"), ("TC_BF16", "COSINE")):
        col = make_col(ctx, corpus, metric, screen=screen)
        rows, dist, cnt = col.knn(queries, 65)
        assert col.stats()["n_fallback"] <= 45
        for q in list(range(0, 4500, 97)) + [2047, 2048, 4095, 4096, 4499]:
            r, d = O.knn_topk(corpus, queries[q], metric.lower(), 65)
            assert list(rows[q]) == list(r) and dist[q].tobytes() == d.tobytes(), (screen, metric, q)


def test_approximate_mode_skips_the_fallback_but_stays_accurate(ctx):
    rng = np.random.default_rng(8)
    center = rng.uniform(-1, 1, 64).astype(np.float32)
    corpus = (center[None, :] + rng.normal(0, 1e-6, (30000, 64))).astype(np.float32)  # proof cannot succeed here
    queries = (center[None, :] + rng.normal(0, 1e-3, (12, 64))).astype(np.float64)
    col = make_col(ctx, corpus, "COSINE", screen="TC_BF16")
    col.set_exact(False)
    rows, dist, cnt = col.knn(queries, 10)
    assert col.stats()["n_fallback"] == 0 and (cnt == 10).all()
    assert (np.diff(dist, axis=1) >= 0).all()
    col.set_exact(True)
    rows2, dist2, _ = col.knn(queries, 10)
    assert col.stats()["n_fallback"] > 0
    for q in range(12):
        r, d = O.knn_topk(corpus, queries[q], "cosine", 10)
        assert list(rows2[q]) == list(r)


@pytest.mark.parametrize("metric", ["MANHATTAN", "CHEBYSHEV", "HAMMING", "PEARSON"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_other_distance_metrics_through_the_exact_kernel(ctx, metric, dtype):
    # Distance::compute catalog/schema/index.rs:287-303 -- the metrics without a screen are ranked by the exact kernel
    rng = np.random.default_rng(len(metric) + (dtype == np.float64))
    for dim in (1, 5, 33, 1100):
        n = 3000
        corpus = rng.integers(-3, 4, (n, dim)).astype(dtype) if metric == "HAMMING" else \
            rng.uniform(-20, 20, (n, dim)).astype(dtype)
        queries = rng.integers(-3, 4, (2, dim)).astype(np.float64) if metric == "HAMMING" else \
            rng.uniform(-20, 20, (2, dim))
        if dim >= 5:
            corpus[7] = 0.0           # constant row: pearson 0/0 -> generated (negative) NaN sorts first
            corpus[11, 0] = np.nan    # data NaN
            corpus[13, 1] = -0.0
        skip = np.zeros(n, np.uint8)
        skip[5] = 1
        col = make_col(ctx, corpus, metric, skip=skip)
        for k in (1, 10, 300):
            check(col, corpus, queries, metric, k, skip=skip)
        assert col.stats()["n_fallback"] == 2


def test_minkowski_and_jaccard_through_the_exact_kernel(ctx):
    # the last two catalog::Distance variants (fnc/util/math/vector.rs:120-130,163-174)
    import ctypes as C
    rng = np.random.default_rng(46)
    for dim in (3, 17, 96):
        n = 2500
        # Jaccard: set semantics over the VALUES -> small integer alphabets give non-trivial sets and many ties
        corpus = rng.integers(0, 12, (n, dim)).astype(np.float32)
        corpus[3, 0] = -0.0
        queries = rng.integers(0, 12, (3, dim)).astype(np.float64)
        col = make_col(ctx, corpus, "JACCARD")
        for k in (1, 10, 200):
            check(col, corpus, queries, "JACCARD", k)   # bit-exact, ties by scan order
        # Minkowski of order p: pow() differs by an ulp or two between CUDA's and the host's libm -> same rows
        # (no near-ties in random data), distances equal to 1e-12 relative
        corpus = rng.uniform(-20, 20, (n, dim)).astype(np.float32)
        queries = rng.uniform(-20, 20, (3, dim))
        for order in (3.0, 1.5):
            O.lib().orc_set_minkowski_order(C.c_double(order))
            col = make_col(ctx, corpus, "MINKOWSKI")
            col.set_minkowski_order(order)
            rows, dist, cnt = col.knn(queries, 10)
            for q in range(3):
                r, d = O.knn_topk(corpus, queries[q], "minkowski", 10)
                assert list(rows[q]) == list(r), (dim, order, q)
                assert np.allclose(dist[q], d, rtol=1e-12, atol=0.0)
        O.lib().orc_set_minkowski_order(C.c_double(3.0))
    # the reference's own KATs (surrealdb/core/tests/function.rs:3585-3593) through the column projection
    col = make_col(ctx, np.array([[1.1, 2.2, 3.0], [1.0, 2.0, 3.0]], np.float64), "MINKOWSKI")
    col.set_minkowski_order(3)
    assert abs(col.project("MINKOWSKI", np.array([4.0, 5.5, 6.6]))[0] - 4.747193170917638) < 1e-14
    assert abs(col.project("MINKOWSKI", np.array([4.0, 5.0, 6.0]))[1] - 4.3267487109222245) < 1e-14
    col = make_col(ctx, np.array([[10, 20, 15, 10, 5]], np.float64), "MINKOWSKI")
    col.set_minkowski_order(2)
    assert abs(col.project("MINKOWSKI", np.array([12.0, 24, 18, 8, 7]))[0] - 6.082762530298219) < 1e-14
    from surrealdb_b200 import VectorColumn
    with pytest.raises(Exception):
        VectorColumn(ctx, 4, "NOT_A_METRIC", "F32", capacity=4)


def test_legacy_two_pass_bruteforce_returns_table_order(ctx):
    # QueryExecutor::knn + KnnPriorityList (idx/planner/executor.rs:283-311, idx/planner/knn.rs:11-106)
    from surrealdb_b200 import KnnBruteForceLegacy, KnnContext
    rng = np.random.default_rng(8)
    pts = rng.integers(-3, 4, (300, 4)).astype(np.float64)          # many exact ties
    recs = [{"id": f"pts:{i}", "point": list(map(float, p))} for i, p in enumerate(pts)]
    recs[5] = {"id": "pts:5", "point": "not a vector"}
    q = [0.5, 0.0, 1.0, -1.0]
    for k in (1, 7, 40):
        kc = KnnContext()
        out = KnnBruteForceLegacy(recs, "point", q, k, "Euclidean", ctx=ctx).with_knn_context(kc).execute()
        d = [None if i == 5 else O.f64_euclidean(pts[i], np.asarray(q)) for i in range(len(recs))]
        must, tie, left = O.knn_priority_list(d, k)
        got = [int(r["id"].split(":")[1]) for r in out]
        assert got == sorted(got) and len(got) == len(must) + left                  # table order, k rows
        assert set(must) <= set(got) and set(got) - set(must) <= set(tie)
        assert all(kc[f"pts:{r}"] == d[r] for r in got)                             # vector::distance::knn()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_projected_vector_functions_match_the_reference_arithmetic(ctx, dtype):
    # SELECT vector::<fn>(emb, $q) FROM t  (fnc/vector.rs) as one columnar pass
    rng = np.random.default_rng(21)
    for dim in (3, 64, 257):
        n = 700
        corpus = rng.uniform(-20, 20, (n, dim)).astype(dtype)
        corpus[3] = 0.0
        corpus[4, 1] = np.nan
        q = rng.uniform(-20, 20, dim)
        skip = np.zeros(n, np.uint8)
        skip[9] = 1
        col = make_col(ctx, corpus, "COSINE", skip=skip)
        c64 = corpus.astype(np.float64)
        for fn in ("COSINE", "EUCLIDEAN", "MANHATTAN", "CHEBYSHEV", "HAMMING", "PEARSON"):
            got = col.project(fn, q)
            want = np.array([O.f64_metric(fn.lower(), c64[r], q) for r in range(n)])
            want[9] = np.nan
            assert got.tobytes() == want.tobytes(), fn
        got = col.project("SIMILARITY_COSINE", q)
        for r in (0, 1, 2, 3, 4, 50, n - 1):
            st, v = O.num_metric("cosine_similarity", list(c64[r]), list(q))
            assert np.float64(v).tobytes() == got[r].tobytes() or (np.isnan(v) and np.isnan(got[r])), r
        got = col.project("DOT", q)
        for r in (0, 1, 2, 3, 50, n - 1):
            st, v = O.num_metric("dot", list(c64[r]), list(q))
            assert float(v) == got[r], r
        got = col.project("MAGNITUDE")
        for r in (0, 1, 3, 50, n - 1):
            assert O.num_magnitude(list(c64[r])) == got[r], r
    with pytest.raises(Exception, match="same dimension"):
        col.project("DOT", np.zeros(5))


def test_slack_ladder_rescues_high_dimensional_large_k_batches(ctx):
    # BASELINE config 4 shape (1536 dims, k=100) at a reduced row count: similarities are packed so tightly that the
    # default slack cannot prove exactness; the ladder must widen k' (not send hundreds of queries to the exact kernel),
    # remember the rung, and the answers must still be the oracle's bit for bit.
    rng = np.random.default_rng(1536)
    n, dim, nq, k = 200_000, 1536, 256, 100
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    col = make_col(ctx, corpus, "COSINE")
    rows, dist, cnt = col.knn(queries, k)
    st1 = col.stats()
    assert st1["n_fallback"] <= 2 + nq // 64, st1
    for q in (0, 100, 255):
        r, d = O.knn_topk(corpus, queries[q], "cosine", k)
        assert list(rows[q, : cnt[q]]) == list(r) and dist[q, : cnt[q]].tobytes() == d.tobytes()
    rows2, dist2, cnt2 = col.knn(queries, k)
    st2 = col.stats()
    assert st2["n_passes"] <= st1["n_passes"] and st2["n_fallback"] <= 2 + nq // 64   # starts on the remembered rung
    assert rows2.tobytes() == rows.tobytes() and dist2.tobytes() == dist.tobytes()


def test_language_test_filtered_bruteforce_through_operator(ctx):
    # bruteforce_knn_with_filter_new_executor.surql / bruteforce_knn_multisource_filter_new_executor.surql:
    # TableScan [predicate: active = true] (or Union + Filter) feeds KnnTopK, which ranks the surviving rows
    from surrealdb_b200 import KnnContext, KnnTopK
    recs = [{"id": "pts:1", "point": [10, 0], "active": True}, {"id": "pts:2", "point": [2, 0], "active": False},
            {"id": "pts:3", "point": [3, 0], "active": True}, {"id": "pts:4", "point": [100, 0], "active": True},
            {"id": "pts:5", "point": [50, 0], "active": False}]
    kc = KnnContext()
    op = KnnTopK([r for r in recs if r["active"]], "point", [1, 0], 2, "Euclidean", ctx=ctx).with_knn_context(kc)
    assert op.attrs() == [("field", "point"), ("k", "2"), ("distance", "Euclidean"), ("dimension", "2")]
    out = op.execute()
    assert [r["id"] for r in out] == ["pts:3", "pts:1"] and [kc[r["id"]] for r in out] == [2.0, 9.0]
    multi = [{"id": "pts:1", "point": [10, 0], "active": True}, {"id": "pts:2", "point": [2, 0], "active": False},
             {"id": "pts:3", "point": [3, 0], "active": True}, {"id": "pts2:1", "point": [1.5, 0], "active": False},
             {"id": "pts2:2", "point": [4, 0], "active": True}]
    kc = KnnContext()
    out = KnnTopK([r for r in multi if r["active"]], "point", [1, 0], 2, "Euclidean", ctx=ctx).with_knn_context(kc).execute()
    assert [r["id"] for r in out] == ["pts:3", "pts2:2"] and [kc[r["id"]] for r in out] == [2.0, 3.0]
