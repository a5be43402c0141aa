"""The brute-force KNN routing policy that include/sdbgpu.h documents next to sdb_screen, pinned cell by cell: for every
metric (MINKOWSKI of orders 2, 2.5 and 9), row type, screen request, k in {10, 257} and batch size in {1, 8}, the screen
that sdb_knn_last_stats reports and whether any screen pass ran.  Every answer is also compared bit for bit (rows, order,
f64 distances, counts) with the same queries under NONE_EXACT, the exact kernel."""
import ctypes as C
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

AUTO, SIMT_F32, TC_BF16, NONE_EXACT, TC_INT8 = 0, 1, 2, 3, 4
SCREENS = ["AUTO", "SIMT_F32", "TC_BF16", "NONE_EXACT", "TC_INT8"]
N, DIM = 3000, 64

# (metric, MINKOWSKI order) of every column
COLUMNS = [("COSINE", None), ("EUCLIDEAN", None), ("PEARSON", None), ("MANHATTAN", None), ("CHEBYSHEV", None),
           ("MINKOWSKI", 2.0), ("MINKOWSKI", 2.5), ("MINKOWSKI", 9.0), ("HAMMING", None), ("JACCARD", None)]


def expected(metric, order, dtype, screen, k, nq, int8_auto):
    """(screen_used, whether a screen pass runs) as the header states them, for columns whose screen copies, moments
    and first-occurrence state all fit (these small ones do) and that have no special rows.  int8_auto: the column's
    normalised rows quantise well enough for AUTO to start on the int8 screen."""
    exact = (NONE_EXACT, False)
    if screen == "NONE_EXACT" or k > 256:
        return exact
    if metric in ("HAMMING", "JACCARD"):
        # the count path, reported as one SIMT_F32 pass; AUTO ranks a single HAMMING query on the exact kernel
        if metric == "HAMMING" and screen == "AUTO" and nq == 1:
            return exact
        return SIMT_F32, True
    if metric == "MINKOWSKI" and order not in (1, 2, 3, 4, 5, 6, 7, 8):
        return exact
    if metric in ("MANHATTAN", "CHEBYSHEV", "MINKOWSKI"):
        # the f32 Lp screen for AUTO and every other request; AUTO ranks a single MANHATTAN / CHEBYSHEV query exactly
        if metric != "MINKOWSKI" and screen == "AUTO" and nq == 1:
            return exact
        return SIMT_F32, True
    int8_ok = metric in ("COSINE", "PEARSON")
    if screen == "AUTO":
        return (TC_INT8 if int8_ok and int8_auto else TC_BF16), True
    if screen == "TC_INT8":
        return (TC_INT8 if int8_ok else TC_BF16), True
    if screen == "TC_BF16":
        return TC_BF16, True
    # SIMT_F32: the f32 stream of f32 COSINE / EUCLIDEAN rows; F64 rows and PEARSON mean the exact kernel
    return (SIMT_F32, True) if dtype == "F32" and metric != "PEARSON" else exact


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_data(metric, order, dtype):
    rng = np.random.default_rng(zlib.crc32(f"route{metric}{order}{dtype}".encode()))
    fdt = np.float32 if dtype == "F32" else np.float64
    if metric in ("HAMMING", "JACCARD"):  # a small alphabet: distances spread instead of all tying at DIM
        return rng.integers(0, 4, (N, DIM)).astype(fdt), rng.integers(0, 4, (8, DIM)).astype(np.float64)
    return rng.uniform(-1, 1, (N, DIM)).astype(fdt), rng.uniform(-1, 1, (8, DIM))


def make_col(ctx, metric, order, dtype, corpus):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, DIM, metric, dtype, capacity=N)
    col.append(corpus)
    col.finalize()
    if order is not None:
        col.set_minkowski_order(order)
    return col


def int8_auto(col):
    """max_rel_qerr <= 0.02: the header's condition for AUTO to start a COSINE / PEARSON column on the int8 screen"""
    from surrealdb_b200 import _lib as L
    if col.metric not in ("COSINE", "PEARSON"):
        return False
    f = np.zeros(4, np.float32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, f.ctypes.data_as(C.c_void_p), None, None, None, None, None))
    return bool(f[1] <= 0.02)


def run(col, screen, queries, k, **kw):
    col.set_screen(screen)
    rows, dist, cnt = col.knn(queries, k, **kw)
    return rows, dist, cnt, col.stats()


def assert_same(got, want, cell):
    rows, dist, cnt = got[:3]
    r2, d2, c2 = want[:3]
    assert cnt.tolist() == c2.tolist(), cell
    for q in range(cnt.size):
        assert rows[q, : cnt[q]].tolist() == r2[q, : cnt[q]].tolist(), (cell, q)
        assert dist[q, : cnt[q]].tobytes() == d2[q, : cnt[q]].tobytes(), (cell, q)


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric,order", COLUMNS, ids=[m if o is None else f"{m}{o:g}" for m, o in COLUMNS])
def test_routing_matrix(ctx, metric, order, dtype):
    corpus, queries = make_data(metric, order, dtype)
    col = make_col(ctx, metric, order, dtype, corpus)
    auto8 = int8_auto(col)
    for k in (10, 257):
        for nq in (1, 8):
            ref = run(col, "NONE_EXACT", queries[:nq], k)
            for screen in SCREENS:
                cell = (metric, order, dtype, screen, k, nq)
                got = run(col, screen, queries[:nq], k)
                st = got[3]
                want_screen, passes = expected(metric, order, dtype, screen, k, nq, auto8)
                assert st["screen_used"] == want_screen, (cell, st)
                assert (st["n_passes"] > 0) == passes, (cell, st)
                if not passes:  # every query of an exact-only batch is ranked by the exact kernel
                    assert st["n_fallback"] == nq, (cell, st)
                assert_same(got, ref, cell)
    col.close()


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric,order", COLUMNS, ids=[m if o is None else f"{m}{o:g}" for m, o in COLUMNS])
def test_routing_direct_regime(ctx, metric, order, dtype):
    # a filter passing fewer than DIRECT_MAX_ROWS (4096) rows: the screened families skip the screen and rank each
    # query's passing rows by the exact re-rank; MINKOWSKI of an unscreened order stays on the exact kernel
    from surrealdb_b200.engine import pack_row_filter
    corpus, queries = make_data(metric, order, dtype)
    col = make_col(ctx, metric, order, dtype, corpus)
    rng = np.random.default_rng(zlib.crc32(f"direct{metric}{order}{dtype}".encode()))
    kw = dict(filters=pack_row_filter(rng.random((1, N)) < 0.3), query_filter=np.zeros(8, np.uint32))
    ref = run(col, "NONE_EXACT", queries, 10, **kw)
    got = run(col, "AUTO", queries, 10, **kw)
    st = got[3]
    direct = not (metric == "MINKOWSKI" and order != 2.0)
    assert st["screen_used"] == NONE_EXACT and st["n_passes"] == 0, st
    assert st["n_fallback"] == (0 if direct else 8), st
    assert_same(got, ref, (metric, order, dtype))
    col.close()
