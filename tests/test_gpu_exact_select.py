"""The exact kernel (exact.cu: one f64 pass, then a 12-pass radix select over the 96-bit (dist_key, row) pair) against the
oracle's KnnTopK, bit for bit, where selection goes wrong: ties that only the row's upper bytes separate (more than 2^24
rows), k from 256 to the 4096 limit and past it, queries wider than one 1024-column chunk, the 1024-row SPECIAL_CAP
boundary, and a -0.0 distance.  As a second check, tests/select_ref.topk over col.project(metric, q) -- the same
distance kernel, selected in numpy -- must return the same rows and values, which separates the selection from the
distance arithmetic."""
import ctypes as C

import numpy as np
import pytest

import select_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

METRICS = ["CHEBYSHEV", "COSINE", "EUCLIDEAN", "HAMMING", "JACCARD", "MANHATTAN", "MINKOWSKI", "PEARSON"]


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def bits(a):
    return np.asarray(a, np.float64).view(np.uint64).tolist()


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


def check(col, corpus, queries, metric, ks, skip=None):
    """knn at every k against the oracle (MINKOWSKI: same rows, distances within 1e-12: CUDA's pow) and against
    topk over the column's projection (bit for bit for every metric: the same GPU arithmetic)"""
    for qi, q in enumerate(queries):
        vals = col.project(metric, q)
        for k in ks:
            rows, dist, cnt = col.knn(q[None, :], k)
            n = int(cnt[0])
            r, d = O.knn_topk(corpus, q, metric.lower(), k, skip=skip)
            assert n == r.size, (metric, k, qi, n, r.size)
            assert rows[0, :n].tolist() == r.tolist(), (metric, k, qi)
            if metric == "MINKOWSKI":
                assert np.allclose(dist[0, :n], d, rtol=1e-12, atol=0.0), (k, qi)
            else:
                assert bits(dist[0, :n]) == bits(d), (metric, k, qi)
            pr, pd = R.topk(vals, k, skip)
            assert rows[0, :n].tolist() == pr.tolist() and bits(dist[0, :n]) == bits(pd), (metric, k, qi)


# ---- ties across 2^24: radix passes 8-11 pick among equal keys by the row's bytes, most significant first ----------
N_TIES = (1 << 24) + (1 << 20)
# the rows at distance 0: their ids differ in every byte, so every row pass has to choose a nonzero digit somewhere
PLANTED = [3, (1 << 8) + 1, (1 << 16) + 5, (1 << 24) - 1, 1 << 24, (1 << 24) + (1 << 16) + 3, N_TIES - 1]
TIE_KS = [1, 2, 3, 4, 5, 6, 7, 8, 256, 257, 4096]


@pytest.fixture(scope="module")
def tie_corpus():
    """dim 2, small integers: every other row is at least (2, 2) from the query (0, 0); PLANTED rows are (0, 0); a
    group of 4200 rows at (1, 1), 300 of them above 2^24, so k = 256 and 257 cut it among the low rows and k = 4096
    above 2^24"""
    rng = np.random.default_rng(24)
    x = rng.integers(2, 10, (N_TIES, 2)).astype(np.float32)
    x[PLANTED] = 0.0
    free = np.ones(N_TIES, bool)
    free[PLANTED] = False
    ids = np.arange(N_TIES)
    ones = np.concatenate([rng.choice(ids[free & (ids < 1 << 24)], 3900, replace=False),
                           rng.choice(ids[free & (ids >= 1 << 24)], 300, replace=False)])
    x[ones] = 1.0
    return x, np.sort(ones)


@pytest.mark.parametrize("metric", ["MANHATTAN", "EUCLIDEAN"])
def test_ties_across_two_to_the_24_rows(ctx, tie_corpus, metric):
    x, ones = tie_corpus
    q = np.zeros(2)
    col = make_col(ctx, x, metric, screen="NONE_EXACT")
    rng = np.random.default_rng(7)
    skip = (rng.random(N_TIES) < 0.1).astype(np.uint8)
    skip[ones] = 0  # the tie group stays larger than 4096, so k = 4096 still ends inside it
    skip[[PLANTED[1], PLANTED[4]]] = 1  # the rest of the planted group stays, whatever the random mask drew
    skip[[PLANTED[i] for i in (0, 2, 3, 5, 6)]] = 0
    removed = np.array([PLANTED[3], PLANTED[6]] + ones[::97].tolist(), np.uint64)
    for state in ("all rows", "skip mask", "skip mask and removed rows"):
        if state == "skip mask":
            col.set_skip(skip)
            col.finalize()
        eff = None
        if state != "all rows":
            eff = skip.copy()
        if state == "skip mask and removed rows":
            col.remove(removed)
            eff[removed.astype(np.int64)] = 1
        # (key, row) is a total order, so the answer at each k is a prefix of the answer at 4096
        r, d = O.knn_topk(x, q, metric.lower(), 4096, skip=eff)
        pr, pd = R.topk(col.project(metric, q), 4096, eff)
        assert r.tolist() == pr.tolist() and bits(d) == bits(pd), state
        assert int(r[4095]) >= 1 << 24, state  # k = 4096 ends inside the tie group, above 2^24
        for k in TIE_KS:
            rows, dist, cnt = col.knn(q[None, :], k)
            assert int(cnt[0]) == k, (state, k)
            assert rows[0].tolist() == r[:k].tolist(), (state, k)
            assert bits(dist[0]) == bits(d[:k]), (state, k)
        assert col.stats()["n_fallback"] == 1


# ---- k at the limits ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_k_256_screened_and_257_4096_exact(ctx, metric):
    rng = np.random.default_rng(256 + len(metric))
    corpus = rng.uniform(-1, 1, (6000, 64)).astype(np.float32)
    corpus[4000:4100] = corpus[100:200]  # exact ties across the k = 256 / 4096 cuts
    queries = rng.uniform(-1, 1, (3, 64))
    col = make_col(ctx, corpus, metric)
    for k, exact in ((256, False), (257, True), (4096, True)):
        rows, dist, cnt = col.knn(queries, k)
        st = col.stats()
        if exact:
            assert st["n_fallback"] == 3, (k, st)
        else:
            assert st["screen_used"] != 3 and st["n_fallback"] < 3, (k, st)  # 3: SDB_SCREEN_NONE_EXACT
        for qi in range(3):
            r, d = O.knn_topk(corpus, queries[qi], metric.lower(), k)
            assert cnt[qi] == k and rows[qi].tolist() == r.tolist() and bits(dist[qi]) == bits(d), (k, qi)


def test_k_4096_on_small_and_fully_skipped_corpora(ctx):
    rng = np.random.default_rng(4096)
    for n in (1, 1000, 4095):
        corpus = rng.integers(-2, 3, (n, 16)).astype(np.float32)
        queries = rng.integers(-2, 3, (2, 16)).astype(np.float64)
        skip = (rng.random(n) < 0.2).astype(np.uint8)
        for metric in ("EUCLIDEAN", "MANHATTAN"):
            check(make_col(ctx, corpus, metric, screen="NONE_EXACT"), corpus, queries, metric, [4096])
            check(make_col(ctx, corpus, metric, skip, "NONE_EXACT"), corpus, queries, metric, [4096], skip)
            col = make_col(ctx, corpus, metric, np.ones(n, np.uint8), "NONE_EXACT")
            rows, dist, cnt = col.knn(queries, 4096)
            assert cnt.tolist() == [0, 0]


def test_k_above_4096_is_refused_and_the_column_still_answers(ctx):
    from surrealdb_b200._lib import SDB_EUNSUPPORTED, SdbError
    rng = np.random.default_rng(4097)
    corpus = rng.uniform(-1, 1, (5000, 24)).astype(np.float32)
    queries = rng.uniform(-1, 1, (4, 24))
    for metric in ("COSINE", "MANHATTAN"):
        col = make_col(ctx, corpus, metric)
        with pytest.raises(SdbError) as e:
            col.knn(queries, 4097)
        assert e.value.status == SDB_EUNSUPPORTED
        check(col, corpus, queries, metric, [10])


# ---- queries wider than one EX_QCHUNK (1024 columns) ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("dim", [1023, 1024, 1025, 2049])
@pytest.mark.parametrize("metric", METRICS)
def test_query_column_chunks(ctx, metric, dim, dtype):
    rng = np.random.default_rng(dim * 8 + METRICS.index(metric))
    n = 700
    npdt = np.float32 if dtype == "F32" else np.float64
    if metric in ("HAMMING", "JACCARD"):  # a small alphabet: equal elements, and Jaccard's sets stay small
        corpus = rng.integers(0, 5, (n, dim)).astype(npdt)
        queries = rng.integers(0, 5, (2, dim)).astype(np.float64)
    else:
        corpus = rng.uniform(-1, 1, (n, dim)).astype(npdt)
        queries = rng.uniform(-1, 1, (2, dim))
        # the columns on each side of a chunk boundary decide the ranking
        for c in sorted({1022, 1023, 1024, dim - 1} & set(range(dim))):
            corpus[:, c] *= 40
            queries[:, c] *= 40
    corpus[[3, 400]] = corpus[[9, 11]]  # exact ties
    O.lib().orc_set_minkowski_order(C.c_double(3.0))
    col = make_col(ctx, corpus, metric, screen="NONE_EXACT")
    check(col, corpus, queries, metric, [1, 10, 300])


# ---- the SPECIAL_CAP boundary: 1024 special rows are screened, 1025 send every query to the exact kernel ------------
@pytest.mark.parametrize("n_special", [1024, 1025])
def test_special_row_cap(ctx, n_special):
    rng = np.random.default_rng(n_special)
    n, dim = 4000, 32
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    n_zero = n_special - 3  # special rows: zero norm, and the three rows with a non-finite norm
    zero = np.sort(rng.choice(n, n_zero, replace=False))
    corpus[zero] = 0.0  # cosine distance: a generated NaN, negative, sorts first
    data_nan = np.setdiff1d(np.arange(n), zero)[[5, 1500, 2900]]
    corpus[data_nan, 7] = np.nan  # a data NaN: positive, sorts last
    queries = rng.uniform(-1, 1, (3, dim))
    col = make_col(ctx, corpus, "COSINE")
    for k in (1, 10, 256, 1000, n):  # cuts inside the NaN group; k = n ends with the data NaNs
        rows, dist, cnt = col.knn(queries, k)
        st = col.stats()
        if n_special == 1024 and k <= 256:
            assert st["n_special_rows"] == 1024 and st["n_fallback"] == 0, (k, st)
        else:
            assert st["n_fallback"] == 3, (k, st)
        for qi in range(3):
            r, d = O.knn_topk(corpus, queries[qi], "cosine", k)
            assert cnt[qi] == r.size and rows[qi, : r.size].tolist() == r.tolist(), (k, qi)
            assert bits(dist[qi, : r.size]) == bits(d), (k, qi)
            assert rows[qi, : min(k, n_zero)].tolist() == zero[:k].tolist()
        if k == n:
            assert set(rows[:, -3:].ravel().tolist()) == set(data_nan.tolist())


# ---- -0.0: dist_key ties it with 0.0, but the result carries the value the kernel computed ---------------------------
def test_negative_zero_distance_keeps_its_sign(ctx):
    corpus = np.array([[0.0, -8.805437202403729e-162, -5.870291468269152e-162], [1, 2, 3], [0, 0, 1]])
    q = np.array([5.870291468269152e-162, 8.805437202403729e-162, 2.935145734134576e-162])
    r, d = O.knn_topk(corpus, q, "pearson", 3)
    assert r.tolist() == [2, 1, 0] and bits(d)[2] == 0x8000000000000000
    big = np.concatenate([np.tile(corpus, (200, 1)), [[0.0, 0.0, 0.0]]])  # -0.0 ties with -0.0, and the NaN row
    col = make_col(ctx, corpus, "PEARSON")
    check(col, corpus, q[None, :], "PEARSON", [1, 3])
    col = make_col(ctx, big, "PEARSON")
    check(col, big, q[None, :], "PEARSON", [1, 200, 450, 601])
