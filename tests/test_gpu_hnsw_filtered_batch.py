"""Batch-filtered HNSW search (sdb_hnsw_search_filtered_batch[_device]): one element bitmap per query, any selectivity.
Every query must equal Hnsw::knn_search_with_filter with truthy[e] = bit e of its bitmap -- the CPU oracle
(oracle/pyoracle.hnsw_search_csr) for F32 EUCLIDEAN and COSINE, tests/hnsw_metric_ref.py and tests/hnsw_types_ref.py for
the other metrics and types: ids, f64 distances and both visit counters bit-equal (NaN by NaN-ness, Minkowski within
1e-12).  Selective filters make queries outgrow the on-chip candidate window; those are finished by the spill tier,
which the handle's spill count (sdb_hnsw_last_spilled) and the single-mask call's SDB_EOVERFLOW on the same batch show."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as O
from test_gpu_hnsw_walk_shapes import (METRICS, TYPES, chain_graph, dev, elements, gen, hub_layers, index,
                                       random_lists, ref_search, status)
from test_gpu_hnsw_types import same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def masks_of(rng, n, sels):
    """one bool mask per selectivity: a fraction, or "one" (a single truthy element)"""
    out = []
    for s in sels:
        if s == "one":
            m = np.zeros(n, bool)
            m[rng.integers(0, n)] = True
        else:
            m = rng.random(n) < s
        out.append(m)
    return np.stack(out)


def same_answer(a, b):
    """two (ids, dist, cnt[, ctr]) results are equal: counts, counters and each row's first cnt entries (the rest of a
    row is not written by the search)"""
    if a[2].tobytes() != b[2].tobytes() or (len(a) > 3 and a[3].tobytes() != b[3].tobytes()):
        return False
    return all(a[0][q, :c].tobytes() == b[0][q, :c].tobytes() and a[1][q, :c].tobytes() == b[1][q, :c].tobytes()
               for q, c in enumerate(a[2].tolist()))


def check_filtered(idx, g, queries, k, ef, metric, vt, masks, qf=None):
    """the batch call against the reference, query by query; returns its outputs"""
    ids, dist, cnt, ctr = idx.search_graph_filtered(queries, k, ef, masks, query_filter=qf, counters=True)
    m2 = np.atleast_2d(masks)
    for q in range(queries.shape[0]):
        t = m2[0 if qf is None else qf[q]].astype(np.uint8)
        oi, od, oc = ref_search(g, queries[q], k, ef, metric, vt, truthy=t)
        assert cnt[q] == oi.size, (vt, metric, k, ef, q)
        assert list(ids[q, : cnt[q]]) == list(oi), (vt, metric, k, ef, q)
        assert (int(ctr[q, 0]), int(ctr[q, 1])) == oc, (vt, metric, k, ef, q)
        assert all(same(metric, a, b) for a, b in zip(dist[q, : cnt[q]], od)), (vt, metric, k, ef, q)
    return ids, dist, cnt, ctr


def oracle_graph(rng, metric, n=3000, dim=24):
    data = rng.uniform(-20, 20, (n, dim)).astype(np.float32)
    h = O.Hnsw(dim, metric, m=8, efc=60, seed=1)
    for v in data:
        h.insert(v)
    return h.export()


def chain(rng, metric, n=20000, dim=64):
    x, lists = chain_graph(rng, n, dim)
    x = x.astype(np.float32)
    return dict(vectors=x, layers=hub_layers(lists), entry_point=0, metric=metric)


# ---------------------------------------------------------------- 1. every selectivity, F32 euclidean and cosine
SELS = [1.0, 0.5, 0.05, 0.01, 0.001, "one", 0.0]


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("shape", ["chain", "oracle"])
def test_every_selectivity(ctx, metric, shape):
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(7000 + len(metric) + len(shape))
    g = chain(rng, metric) if shape == "chain" else oracle_graph(rng, metric)
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, metric, "F32")
    queries = (x[rng.integers(0, n, 40)] + rng.normal(0, 0.5, (40, dim))).astype(np.float32)
    spilled = {}
    for s, m in zip(SELS, masks_of(rng, n, SELS)):
        for k, ef in ((10, 10), (10, 40)):
            ids, _, cnt, _ = check_filtered(idx, g, queries, k, ef, metric, "F32", m)
            assert all(m[int(e)] for q in range(queries.shape[0]) for e in ids[q, : cnt[q]])
            spilled[(s, ef)] = idx.last_spilled()
            if spilled[(s, ef)]:  # the single-mask call cannot serve this batch
                st = status(lambda: idx.search_graph(queries, k, ef, truthy=m.astype(np.uint8)))
                assert st == L.SDB_EOVERFLOW, (s, ef, st)
    assert spilled[(1.0, 10)] == 0 and spilled[(0.5, 40)] == 0
    assert spilled[(0.0, 10)] == queries.shape[0] and spilled[(0.001, 10)] > 0, spilled
    idx.close()


# ---------------------------------------------------------------- 2. every metric x vector type, spilled and on chip
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vt", TYPES)
def test_every_metric_and_type(ctx, vt, metric):
    rng = np.random.default_rng(7100 + TYPES.index(vt) * 8 + METRICS.index(metric))
    n, dim = 3000, 20
    x = elements(rng, metric, vt, n, dim)
    g = dict(vectors=x, layers=hub_layers(random_lists(rng, n)), entry_point=0)
    idx = index(ctx, x, g, metric, vt)
    queries = gen(rng, metric, vt, (12, dim))
    masks = np.stack([rng.random(n) < 0.5, rng.random(n) < 0.002])
    qf = np.array([0, 1] * 6, np.uint32)
    check_filtered(idx, g, queries, 10, 10, metric, vt, masks, qf)
    assert 0 < idx.last_spilled() < queries.shape[0], idx.last_spilled()
    idx.close()


# ---------------------------------------------------------------- 3. one bitmap per query
def test_per_query_filters(ctx):
    rng = np.random.default_rng(7200)
    g = chain(rng, "euclidean")
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, "euclidean", "F32")
    nq = 192
    queries = (x[rng.integers(0, n, nq)] + rng.normal(0, 0.5, (nq, dim))).astype(np.float32)
    masks = rng.random((64, n)) < 0.1
    qf = rng.permutation(np.arange(nq) % 64).astype(np.uint32)
    words = idx.filter_words(masks)
    got = check_filtered(idx, g, queries, 10, 40, "euclidean", "F32", masks, qf)
    packed = idx.search_graph_filtered(queries, 10, 40, words, query_filter=qf, counters=True)
    assert same_answer(got, packed)
    for f in range(0, 64, 9):  # a query answers the same in a batch of one filter
        sel = np.nonzero(qf == f)[0]
        one = idx.search_graph_filtered(queries[sel], 10, 40, masks[f], counters=True)
        assert same_answer(one, [b[sel] for b in got]), f
    # query_filter = None: every query uses filter 0
    a = idx.search_graph_filtered(queries, 10, 40, masks, counters=True)
    b = idx.search_graph_filtered(queries, 10, 40, masks[0], counters=True)
    assert same_answer(a, b)
    idx.close()


# ---------------------------------------------------------------- 4. agreement with the single-mask call
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_agrees_with_the_single_mask_call(ctx, metric):
    rng = np.random.default_rng(7300 + len(metric))
    g = oracle_graph(rng, metric)
    x = g["vectors"]
    idx = index(ctx, x, g, metric, "F32")
    queries = rng.uniform(-20, 20, (64, x.shape[1])).astype(np.float32)
    served = 0
    for s in (1.0, 0.5, 0.2, 0.08, 0.02):
        m = rng.random(x.shape[0]) < s
        for k, ef in ((10, 40), (3, 8), (10, 10)):
            try:
                old = idx.search_graph(queries, k, ef, counters=True, truthy=m.astype(np.uint8))
            except Exception as e:
                assert "SDB_EOVERFLOW" in str(e), str(e)
                continue
            new = idx.search_graph_filtered(queries, k, ef, m, counters=True)
            assert same_answer(old, new), (s, k, ef)
            served += 1
    assert served >= 6
    ones = np.ones(x.shape[0], bool)
    a = idx.search_graph_filtered(queries, 10, 40, ones, counters=True)
    b = idx.search_graph(queries, 10, 40, counters=True)
    assert same_answer(a, b)
    idx.close()


# ---------------------------------------------------------------- 5. the visited table of the unfiltered walk overflows
def test_visited_table_overflow_is_served(ctx):
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(5000)
    n, dim = 9500, 16
    x = gen(rng, "euclidean", "F32", (n, dim))
    queries = gen(rng, "euclidean", "F32", (24, dim))
    g = dict(vectors=x, layers=hub_layers(random_lists(rng, n, hub=9000, deg=(2, 10))), entry_point=0)
    ones = np.ones(n, bool)
    for metric in ("euclidean", "cosine"):
        idx = index(ctx, x, g, metric, "F32")
        for ef in (16, 32):
            assert status(lambda: idx.search_graph(queries, 10, ef)) == L.SDB_EOVERFLOW
            ids, dist, cnt, ctr = idx.search_graph_filtered(queries, 10, ef, ones, counters=True)
            for q in range(queries.shape[0]):
                oi, od, oc = O.hnsw_search_csr(dict(g, metric=metric), queries[q], 10, ef)
                assert list(ids[q, : cnt[q]]) == list(oi) and dist[q, : cnt[q]].tobytes() == od.tobytes(), (ef, q)
                assert (int(ctr[q, 0]), int(ctr[q, 1])) == oc, (ef, q)
        idx.close()


# ---------------------------------------------------------------- 6. device variant
def test_device_variant_stays_in_its_rows(ctx):
    import torch
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(7500)
    g = chain(rng, "cosine", n=8000)
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, "cosine", "F32")
    nq, k, ef, pad = 96, 7, 20, 64
    queries = (x[rng.integers(0, n, nq)] + rng.normal(0, 0.5, (nq, dim))).astype(np.float32)
    masks = np.stack([rng.random(n) < 0.3, rng.random(n) < 0.0005, np.zeros(n, bool)])
    qf = (np.arange(nq) % 3).astype(np.uint32)
    words = idx.filter_words(masks)
    q, f = dev(queries), dev(words)
    ids = torch.full((nq * k + pad,), -7, dtype=torch.int64, device="cuda")
    dist = torch.full((nq * k + pad,), -7.0, dtype=torch.float64, device="cuda")
    cnt = torch.full((nq + pad,), -7, dtype=torch.int32, device="cuda")
    ctr = torch.full((2 * nq + pad,), -7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    p = lambda t: C.c_void_p(t.data_ptr())
    L.check(L.lib().sdb_hnsw_search_filtered_batch_device(idx.h, p(q), nq, k, ef, p(f), 3, C.c_void_p(qf.ctypes.data),
                                                          p(ids), p(dist), p(cnt), p(ctr)))
    assert idx.last_spilled() > 0
    ids, dist, cnt, ctr = ids.cpu().numpy(), dist.cpu().numpy(), cnt.cpu().numpy(), ctr.cpu().numpy()
    assert (cnt[nq:] == -7).all() and (ids[nq * k:] == -7).all() and (dist[nq * k:] == -7.0).all()
    assert (ctr[2 * nq:] == -7).all()
    hi, hd, hc, hctr = check_filtered(idx, g, queries, k, ef, "cosine", "F32", masks, qf)
    assert cnt[:nq].view(np.uint32).tobytes() == hc.tobytes() and ctr[: 2 * nq].view(np.uint64).tobytes() == hctr.tobytes()
    for r in range(nq):  # the rows' entries past the count are not compared (neither call defines them)
        c = int(hc[r])
        assert ids[r * k: r * k + c].view(np.uint64).tobytes() == hi[r, :c].tobytes()
        assert dist[r * k: r * k + c].tobytes() == hd[r, :c].tobytes()
    idx.close()


# ---------------------------------------------------------------- 7. edge cases
def test_edge_cases_errors_cancellation_and_allocations():
    from surrealdb_b200 import Context, SdbError
    from surrealdb_b200 import _lib as L
    live0 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live0[0]), C.byref(live0[1]))
    ctx = Context(0)  # its own context: everything the test allocates is released by the closes below
    rng = np.random.default_rng(7600)
    g = chain(rng, "euclidean", n=5001, dim=32)  # 5001 elements: the last word holds 9 elements' bits
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, "euclidean", "F32")
    queries = (x[rng.integers(0, n, 16)] + rng.normal(0, 0.5, (16, dim))).astype(np.float32)
    m = rng.random(n) < 0.002
    words = idx.filter_words(m)
    base = idx.search_graph_filtered(queries, 10, 10, words, counters=True)
    assert idx.last_spilled() > 0
    junk = words.copy()
    junk[0, -1] |= np.uint32(0xFFFFFE00)  # the bits of elements 5001 .. 5023
    again = idx.search_graph_filtered(queries, 10, 10, junk, counters=True)
    assert same_answer(base, again)
    # refusals
    out = [np.zeros((16, 10), np.uint64), np.zeros((16, 10), np.float64), np.zeros(16, np.uint32)]
    p = lambda a: C.c_void_p(a.ctypes.data)
    call = lambda f, nf, qf: L.lib().sdb_hnsw_search_filtered_batch(idx.h, p(queries), 16, 10, 10, f, nf, qf, p(out[0]),
                                                                    p(out[1]), p(out[2]), None)
    assert call(p(words), 0, None) == L.SDB_EINVAL
    assert call(None, 1, None) == L.SDB_EINVAL
    bad = np.zeros(16, np.uint32)
    bad[5] = 1
    assert call(p(words), 1, p(bad)) == L.SDB_EINVAL
    assert L.lib().sdb_hnsw_search_filtered_batch(idx.h, p(queries), 0, 10, 10, p(words), 0, None, p(out[0]), p(out[1]),
                                                  p(out[2]), None) == L.SDB_OK
    # cancellation before the call, then the same handle answers
    ctx.cancel()
    try:
        with pytest.raises(SdbError) as e:
            idx.search_graph_filtered(queries, 10, 10, words)
        assert e.value.status == L.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    after = idx.search_graph_filtered(queries, 10, 10, words, counters=True)
    assert same_answer(base, after)
    idx.close()
    ctx.close()
    live1 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live1[0]), C.byref(live1[1]))
    assert (live1[0].value, live1[1].value) == (live0[0].value, live0[1].value)


# ---------------------------------------------------------------- 8. the operator mirror
def test_knn_scan_with_a_selective_residual_condition(ctx):
    from surrealdb_b200.hnsw import HnswIndex
    from surrealdb_b200.operators import KnnScan
    rng = np.random.default_rng(7700)
    g = chain(rng, "euclidean", n=20000, dim=32)
    x = g["vectors"]
    n = x.shape[0]
    idx = HnswIndex(ctx, x, g["layers"], g["entry_point"], "EUCLIDEAN")
    records = {i: {"id": f"pts:{i}", "cat": i % 1000} for i in range(n)}  # cat == 7: 0.1 % of the records
    cond = lambda rec: rec["cat"] == 7
    truthy = (np.arange(n) % 1000 == 7).astype(np.uint8)
    for q in (x[rng.integers(0, n, 3)] + rng.normal(0, 0.5, (3, 32))).astype(np.float32):
        out = KnnScan(idx, q, 10, 40, "pts", records, residual_cond=cond).execute()
        oi, od, _ = O.hnsw_search_csr(g, q, 10, 40, truthy=truthy)
        assert [r["id"] for r in out] == [f"pts:{int(e)}" for e in oi]
        assert [d for _, d in idx.knn_search(q, 10, 40, truthy_docs={v for v, r in records.items() if cond(r)})] == \
            [float(d) for d in od]
    idx.close()
