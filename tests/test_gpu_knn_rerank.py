"""Every exact re-rank kernel of brute-force KNN (candidates.cu), driven cell by cell and compared bit for bit with the
CPU oracle (rows, order, f64 distance bytes, counts) and with the same queries under NONE_EXACT, the exact kernel.
MINKOWSKI's distances come from pow(), which is CUDA's libm on the GPU and the host's in the oracle: against the
oracle they agree to 1e-12, against NONE_EXACT bit for bit.  Each cell also asserts the screen that ran and that the
re-rank served the answer (screen passes, re-ranked entries, fewer fallbacks than queries), so it provably takes its
path:
  packed  <float/double, cos/euc>   COSINE / EUCLIDEAN under TC_BF16 / TC_INT8 (stage B runs)
  v4 / staged <float>               F32 COSINE / EUCLIDEAN under SIMT_F32 and in the direct regime, dim % 4 == 0 / != 0
  staged <double>                   F64 COSINE / EUCLIDEAN in the direct regime
  per-entry <T, metric>             MANHATTAN, CHEBYSHEV, MINKOWSKI (orders 1, 3, 8) screened and direct; HAMMING and
                                    JACCARD direct; PEARSON under the tensor-core screens and direct
The corpora hold what the finishing rules exist for: a data NaN (positive, sorts last), a row of +inf and -inf (a
generated NaN, sorts first, where the metric makes one), a zero row and a constant row (special rows, re-ranked by
every unfiltered query), -0.0 elements and dim == 1.  (PEARSON's one -0.0 distance, an underflowed covariance, needs a
query whose centred norm is below 2^-100; the exact kernel ranks such queries, test_gpu_exact_select covers it.)"""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SIMT_F32, TC_BF16, NONE_EXACT, TC_INT8 = 1, 2, 3, 4
N, NQ = 3000, 8


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


@pytest.fixture
def oracle_order():
    def set_order(p):
        O.lib().orc_set_minkowski_order(C.c_double(float(p)))
    yield set_order
    set_order(3.0)


def make_data(metric, dtype, dim, n=N):
    rng = np.random.default_rng(zlib.crc32(f"rerank{metric}{dtype}{dim}{n}".encode()))
    fdt = np.float32 if dtype == "F32" else np.float64
    if metric in ("HAMMING", "JACCARD"):  # a small alphabet: distances spread instead of all tying at dim
        x, q = rng.integers(0, 4, (n, dim)).astype(fdt), rng.integers(0, 4, (NQ, dim)).astype(np.float64)
    else:
        x, q = rng.uniform(-1, 1, (n, dim)).astype(fdt), rng.uniform(-1, 1, (NQ, dim))
    x[5, dim // 2] = np.nan  # data NaN: a positive NaN, sorts last
    x[6, 0] = np.inf         # +inf and -inf: inf - inf, a generated NaN, for the metrics that form one
    x[6, dim - 1] = -np.inf if dim > 1 else np.inf
    x[7] = 0.0               # zero row: |x| = 0
    x[8] = 2.5               # constant row: PEARSON's zero deviation
    x[9, 0] = -0.0
    return x, q


def make_col(ctx, metric, x, order=None):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, x.shape[1], metric, "F32" if x.dtype == np.float32 else "F64", capacity=x.shape[0])
    col.append(x)
    col.finalize()
    if order is not None:
        col.set_minkowski_order(order)
    return col


def same(got, want, cell):
    (r, d, c), (r2, d2, c2) = got, want
    assert c.tolist() == c2.tolist(), cell
    for q in range(c.size):
        n = int(c[q])
        assert r[q, :n].tolist() == r2[q, :n].tolist(), (cell, q)
        assert d[q, :n].tobytes() == d2[q, :n].tobytes(), (cell, q)


def check(col, metric, x, queries, k, cell, order=None, filters=None, query_filter=None):
    """the answer under the column's current screen equals NONE_EXACT's and the oracle's; returns its stats"""
    kw = {} if filters is None else dict(filters=filters[1], query_filter=query_filter)
    got = col.knn(queries, k, **kw)
    st = col.stats()
    screen = st["screen_used"]
    col.set_screen("NONE_EXACT")
    want = col.knn(queries, k, **kw)
    assert col.stats()["screen_used"] == NONE_EXACT
    same(got, want, cell)
    rows, dist, cnt = got
    for q in range(queries.shape[0]):
        skip = None if filters is None else (~filters[0][query_filter[q]]).astype(np.uint8)
        r, d = O.knn_topk(x, queries[q], metric.lower(), k, skip=skip)
        n = int(cnt[q])
        assert n == r.size, (cell, q)
        if order is None:
            assert rows[q, :n].tolist() == r.tolist() and dist[q, :n].tobytes() == d.tobytes(), (cell, q)
        else:
            assert np.allclose(dist[q, :n], d, rtol=1e-12, atol=0.0, equal_nan=True), (cell, q)
            for i in np.flatnonzero(rows[q, :n] != r):
                assert abs(dist[q, i] - d[i]) <= 1e-12 * abs(d[i]) and np.isin(rows[q, i], r), (cell, q, i)
    st["screen_used"] = screen
    return st


def assert_reranked(st, screen, cell, specials=True):
    assert st["screen_used"] == screen and st["n_passes"] > 0, (cell, st)
    assert st["n_fallback"] < NQ and st["n_reranked"] > 0, (cell, st)
    if specials:
        assert st["n_special_rows"] > 0, (cell, st)


# ---- packed <T, cos/euc>: stage B after the tensor-core screens ------------------------------------------------------
@pytest.mark.parametrize("screen", ["TC_BF16", "TC_INT8"])
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("dim", [33, 64])  # odd / even f64 rows, scalar / float4 f32 rows
def test_packed(ctx, dim, dtype, metric, screen):
    x, q = make_data(metric, dtype, dim)
    col = make_col(ctx, metric, x)
    for k in (10, 100):
        cell = (metric, dtype, dim, screen, k)
        col.set_screen(screen)
        st = check(col, metric, x, q, k, cell)
        assert_reranked(st, TC_INT8 if screen == "TC_INT8" and metric == "COSINE" else TC_BF16, cell)
    col.close()


# ---- v4 (dim % 4 == 0) and staged <float> (dim % 4 != 0): the f32 SIMT screen -----------------------------------------
@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
@pytest.mark.parametrize("dim", [7, 64, 1025])
def test_simt(ctx, dim, metric):
    x, q = make_data(metric, "F32", dim)
    col = make_col(ctx, metric, x)
    for k in (10, 100):
        cell = (metric, dim, k)
        col.set_screen("SIMT_F32")
        assert_reranked(check(col, metric, x, q, k, cell), SIMT_F32, cell)
    col.close()


# ---- per-entry <T, MANHATTAN / CHEBYSHEV / MINKOWSKI>: the f32 Lp screen ----------------------------------------------
LP = [("MANHATTAN", None), ("CHEBYSHEV", None), ("MINKOWSKI", 1), ("MINKOWSKI", 3), ("MINKOWSKI", 8)]
LP_IDS = [m if o is None else f"{m}{o}" for m, o in LP]


@pytest.mark.parametrize("metric,order", LP, ids=LP_IDS)
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("dim", [1, 7, 64])
def test_lp(ctx, oracle_order, dim, dtype, metric, order):
    if order is not None:
        oracle_order(order)
    x, q = make_data(metric, dtype, dim)
    col = make_col(ctx, metric, x, order)
    for k in (10, 100):
        cell = (metric, order, dtype, dim, k)
        col.set_screen("SIMT_F32")
        assert_reranked(check(col, metric, x, q, k, cell, order), SIMT_F32, cell)
    col.close()


# ---- per-entry <T, PEARSON>: the tensor-core screens on the centred rows ----------------------------------------------
@pytest.mark.parametrize("screen", ["TC_BF16", "TC_INT8"])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("dim", [7, 64])
def test_pearson(ctx, dim, dtype, screen):
    x, q = make_data("PEARSON", dtype, dim)
    col = make_col(ctx, "PEARSON", x)
    for k in (10, 100):
        cell = (dtype, dim, screen, k)
        col.set_screen(screen)
        st = check(col, "PEARSON", x, q, k, cell)
        assert_reranked(st, TC_INT8 if screen == "TC_INT8" else TC_BF16, cell)
    col.close()


# ---- the direct regime: filters passing at most 4096 rows skip the screen, the re-rank ranks the passing rows --------
DIRECT = [("COSINE", None), ("EUCLIDEAN", None), ("PEARSON", None), ("HAMMING", None), ("JACCARD", None)] + LP


def direct_filters(metric, dtype, dim):
    """two filters, both passing the rows of make_data's special values: ~30 % of the rows, and ~40 rows (k = 64 then
    shows every passing row, the data NaN last)"""
    from surrealdb_b200.engine import pack_row_filter
    rng = np.random.default_rng(zlib.crc32(f"direct{metric}{dtype}{dim}".encode()))
    masks = np.stack([rng.random(N) < 0.3, rng.random(N) < 0.013])
    masks[:, 5:10] = True
    return masks, pack_row_filter(masks)


@pytest.mark.parametrize("metric,order", DIRECT, ids=[m if o is None else f"{m}{o}" for m, o in DIRECT])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("dim", [1, 7, 64])
def test_direct(ctx, oracle_order, dim, dtype, metric, order):
    if order is not None:
        oracle_order(order)
    x, q = make_data(metric, dtype, dim)
    col = make_col(ctx, metric, x, order)
    filters = direct_filters(metric, dtype, dim)
    qf = (np.arange(NQ) % 2).astype(np.uint32)
    for k in (10, 64):
        cell = (metric, order, dtype, dim, k)
        col.set_screen("AUTO")
        st = check(col, metric, x, q, k, cell, order, filters, qf)
        # a PEARSON query of one element is constant: the exact kernel ranks it (the re-rank still runs)
        fallback = NQ if metric == "PEARSON" and dim == 1 else 0
        assert st["screen_used"] == NONE_EXACT and st["n_passes"] == 0 and st["n_fallback"] == fallback, (cell, st)
        assert st["n_reranked"] >= NQ * 5, (cell, st)
    col.close()
