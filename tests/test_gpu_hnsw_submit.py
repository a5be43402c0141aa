"""Asynchronous HNSW search (sdb_hnsw_submit[_device], sdb_hnsw_submit_filtered[_device], sdb_hnsw_wait).  A ticket's
outputs after its wait must be byte for byte what the matching blocking call writes on the same handle: ids, f64
distance bit patterns, counts and both visit counters, for every metric and vector type, with a pending mask, with
per-query bitmaps of any selectivity (spilled queries included) and on device buffers.  Up to 4 tickets are in flight,
completed in any order around blocking calls; the errors a blocking call finds after its walk come from the wait."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_hnsw_filtered_batch import chain, masks_of, same_answer
from test_gpu_hnsw_walk_shapes import METRICS, TYPES, dev, elements, gen, hub_layers, index, random_lists, status

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def p(a):
    return C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr())


def live():
    from surrealdb_b200 import _lib as L
    n, b = C.c_uint64(), C.c_uint64()
    L.lib().sdb_debug_live_allocations(C.byref(n), C.byref(b))
    return n.value, b.value


# ---------------------------------------------------------------- 1. every metric x vector type: plain, pending, filtered
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vt", TYPES)
def test_equals_the_blocking_calls(ctx, vt, metric):
    rng = np.random.default_rng(9100 + TYPES.index(vt) * 8 + METRICS.index(metric))
    n, dim = 3000, 20
    x = elements(rng, metric, vt, n, dim)
    g = dict(vectors=x, layers=hub_layers(random_lists(rng, n)), entry_point=0)
    idx = index(ctx, x, g, metric, vt)
    queries = gen(rng, metric, vt, (12, dim))
    pending = (rng.random(n) < 0.2).astype(np.uint8)
    masks = np.stack([rng.random(n) < 0.5, rng.random(n) < 0.002])
    qf = np.array([0, 1] * 6, np.uint32)
    for k, ef in ((10, 10), (5, 40)):
        t_plain = idx.submit_graph(queries, k, ef, counters=True)
        t_pend = idx.submit_graph(queries, k, ef, counters=True, all_docs_pending=pending)
        t_filt = idx.submit_graph_filtered(queries, k, ef, masks, query_filter=qf, counters=True)
        if metric == "minkowski":  # a ticket keeps the order it was submitted with
            L_order(idx, 2.5)
        got_filt = idx.wait(t_filt)
        spilled = idx.last_spilled()
        got_pend, got_plain = idx.wait(t_pend), idx.wait(t_plain)
        if metric == "minkowski":
            L_order(idx, 3.0)
        assert same_answer(got_plain, idx.search_graph(queries, k, ef, counters=True)), (k, ef)
        assert same_answer(got_pend, idx.search_graph(queries, k, ef, counters=True, all_docs_pending=pending)), (k, ef)
        assert same_answer(got_filt, idx.search_graph_filtered(queries, k, ef, masks, query_filter=qf, counters=True))
        assert spilled == idx.last_spilled() and 0 < spilled < queries.shape[0], spilled
    # without counters, the wrapper returns what search_graph returns
    a = idx.wait(idx.submit_graph(queries, 10, 10))
    assert len(a) == 3 and same_answer(a, idx.search_graph(queries, 10, 10))
    idx.close()


def L_order(idx, order):
    from surrealdb_b200 import _lib as L
    L.check(L.lib().sdb_hnsw_set_minkowski_order(idx.h, float(order)))


# ---------------------------------------------------------------- 2. selectivities, spills, 64 shuffled filters
def test_selectivities_and_many_filters(ctx):
    rng = np.random.default_rng(9200)
    g = chain(rng, "euclidean")
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, "euclidean", "F32")
    queries = (x[rng.integers(0, n, 40)] + rng.normal(0, 0.5, (40, dim))).astype(np.float32)
    sels = [1.0, 0.1, 0.01, 0.0]
    spilled = {}
    for s, m in zip(sels, masks_of(rng, n, sels)):
        got = idx.wait(idx.submit_graph_filtered(queries, 10, 10, m, counters=True))
        spilled[s] = idx.last_spilled()
        assert same_answer(got, idx.search_graph_filtered(queries, 10, 10, m, counters=True)), s
        assert idx.last_spilled() == spilled[s]
    assert spilled[1.0] == 0 and spilled[0.0] == queries.shape[0] and spilled[0.01] > 0, spilled
    nq = 192
    queries = (x[rng.integers(0, n, nq)] + rng.normal(0, 0.5, (nq, dim))).astype(np.float32)
    masks = rng.random((64, n)) < 0.1
    qf = rng.permutation(np.arange(nq) % 64).astype(np.uint32)
    got = idx.wait(idx.submit_graph_filtered(queries, 10, 40, masks, query_filter=qf, counters=True))
    assert same_answer(got, idx.search_graph_filtered(queries, 10, 40, masks, query_filter=qf, counters=True))
    idx.close()


# ---------------------------------------------------------------- 3. device variants write only their rows
def test_device_variants_stay_in_their_rows(ctx):
    import torch
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(9300)
    g = chain(rng, "cosine", n=8000)
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, "cosine", "F32")
    nq, k, ef, pad = 96, 7, 20, 64
    queries = (x[rng.integers(0, n, nq)] + rng.normal(0, 0.5, (nq, dim))).astype(np.float32)
    masks = np.stack([rng.random(n) < 0.3, rng.random(n) < 0.0005, np.zeros(n, bool)])
    qf = (np.arange(nq) % 3).astype(np.uint32)
    q, f = dev(queries), dev(idx.filter_words(masks))

    def outputs():
        return [torch.full((nq * k + pad,), -7, dtype=torch.int64, device="cuda"),
                torch.full((nq * k + pad,), -7.0, dtype=torch.float64, device="cuda"),
                torch.full((nq + pad,), -7, dtype=torch.int32, device="cuda"),
                torch.full((2 * nq + pad,), -7, dtype=torch.int64, device="cuda")]

    def host(o):
        return [t.cpu().numpy() for t in o]

    for filtered in (False, True):
        blocking, ticket = outputs(), outputs()
        torch.cuda.synchronize()
        if filtered:
            L.check(L.lib().sdb_hnsw_search_filtered_batch_device(idx.h, p(q), nq, k, ef, p(f), 3, p(qf), *map(p, blocking)))
            t = idx.submit_filtered_device(q.data_ptr(), nq, k, ef, f.data_ptr(), 3, qf, *[o.data_ptr() for o in ticket])
            assert idx.wait(t) is None and idx.last_spilled() > 0
        else:
            L.check(L.lib().sdb_hnsw_search_device(idx.h, p(q), nq, k, ef, *map(p, blocking[:3])))
            t = idx.submit_device(q.data_ptr(), nq, k, ef, *[o.data_ptr() for o in ticket[:3]])
            assert idx.wait(t) is None
        b, a = host(blocking), host(ticket)
        assert (a[2][nq:] == -7).all() and (a[0][nq * k:] == -7).all() and (a[1][nq * k:] == -7.0).all()
        assert (a[3][2 * nq:] == -7).all()
        rows = lambda r: [r[0][: nq * k].reshape(nq, k), r[1][: nq * k].reshape(nq, k), r[2][:nq], r[3][: 2 * nq]]
        a, b = rows(a), rows(b)
        if not filtered:  # sdb_hnsw_search_device has no counters: the ticket left its counter words alone
            assert (a[3] == -7).all()
            a, b = a[:3], b[:3]
        assert same_answer(a, b), filtered
    # the device counters equal the host variant's
    t = idx.submit_device(q.data_ptr(), nq, k, ef, *[o.data_ptr() for o in ticket])
    idx.wait(t)
    _, _, _, hctr = idx.search_graph(queries, k, ef, counters=True)
    assert ticket[3][: 2 * nq].cpu().numpy().view(np.uint64).tobytes() == hctr.tobytes()
    idx.close()


# ---------------------------------------------------------------- 4. four tickets in flight
def test_four_tickets_in_flight(ctx):
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(9400)
    g = chain(rng, "euclidean", n=20000, dim=32)
    x = g["vectors"]
    n, dim = x.shape
    idx = index(ctx, x, g, "euclidean", "F32")
    queries = (x[rng.integers(0, n, 300)] + rng.normal(0, 0.5, (300, dim))).astype(np.float32)
    masks = np.stack([rng.random(n) < 0.3, rng.random(n) < 0.01])
    qf = rng.integers(0, 2, 300).astype(np.uint32)
    # slots 0 and 2 share the first stream's visited tables, 1 and 3 the second's: the later submits of each pair need
    # larger tables (larger ef) while the earlier ticket is still queued
    jobs = [("plain", 10), ("filtered", 10), ("plain", 200), ("filtered", 120)]

    def submit(kind, ef):
        if kind == "plain":
            return idx.submit_graph(queries, 10, ef, counters=True)
        return idx.submit_graph_filtered(queries, 10, ef, masks, query_filter=qf, counters=True)

    def blocking(kind, ef):
        if kind == "plain":
            return idx.search_graph(queries, 10, ef, counters=True)
        return idx.search_graph_filtered(queries, 10, ef, masks, query_filter=qf, counters=True)

    want = [blocking(kind, ef) for kind, ef in jobs]
    between = idx.search_graph(queries[:50], 10, 64, counters=True)
    for order in ("reverse", "shuffled"):
        tickets = []
        for kind, ef in jobs:
            tickets.append(submit(kind, ef))
            assert same_answer(idx.search_graph(queries[:50], 10, 64, counters=True), between)  # a blocking call between
        assert len(set(tickets)) == 4
        assert status(lambda: submit("plain", 10)) == L.SDB_EOVERFLOW  # a fifth
        assert same_answer(idx.search_graph(queries[:50], 10, 64, counters=True), between)  # the handle keeps answering
        seq = list(range(4))[::-1] if order == "reverse" else list(rng.permutation(4))
        for i in seq:
            assert same_answer(idx.wait(tickets[i]), want[i]), (order, i)
        for i in seq:
            assert L.lib().sdb_hnsw_wait(idx.h, tickets[i]) == L.SDB_EINVAL  # already completed
    assert L.lib().sdb_hnsw_wait(idx.h, 123456) == L.SDB_EINVAL  # never issued
    idx.close()


# ---------------------------------------------------------------- 5. errors the wait reports, cancellation
def test_errors_come_from_the_wait(ctx):
    from surrealdb_b200 import SdbError
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(5000)
    n, dim = 9500, 16
    x = gen(rng, "euclidean", "F32", (n, dim))
    queries = gen(rng, "euclidean", "F32", (24, dim))
    g = dict(vectors=x, layers=hub_layers(random_lists(rng, n, hub=9000, deg=(2, 10))), entry_point=0)
    idx = index(ctx, x, g, "euclidean", "F32")
    assert status(lambda: idx.search_graph(queries, 10, 16)) == L.SDB_EOVERFLOW
    t = idx.submit_graph(queries, 10, 16)  # accepted: the overflow is found by the walk
    assert status(lambda: idx.wait(t)) == L.SDB_EOVERFLOW
    # refusals raised by submit
    assert status(lambda: idx.submit_graph(queries, 10, 5000)) == L.SDB_EUNSUPPORTED
    assert status(lambda: idx.submit_graph_filtered(queries, 10, 10, np.ones((1, n), bool),
                                                    query_filter=np.full(24, 1, np.uint32))) == L.SDB_EINVAL
    out = [np.zeros((24, 10), np.uint64), np.zeros((24, 10), np.float64), np.zeros(24, np.uint32)]
    tk = C.c_uint32()
    words = idx.filter_words(np.ones(n, bool))
    assert L.lib().sdb_hnsw_submit_filtered(idx.h, p(queries), 24, 10, 10, p(words), 0, None, *map(p, out), None,
                                            C.byref(tk)) == L.SDB_EINVAL
    assert L.lib().sdb_hnsw_submit(idx.h, p(queries), 24, 10, 10, None, *map(p, out), None, None) == L.SDB_EINVAL
    # empty batches get a ticket; their wait leaves zero counts
    cnt = np.full(24, 7, np.uint32)
    for nq, k, ef in ((0, 10, 10), (24, 0, 10), (24, 10, 0)):
        cnt[:] = 7
        assert L.lib().sdb_hnsw_submit(idx.h, p(queries), nq, k, ef, None, p(out[0]), p(out[1]), p(cnt), None,
                                       C.byref(tk)) == L.SDB_OK
        assert L.lib().sdb_hnsw_wait(idx.h, tk.value) == L.SDB_OK
        assert (cnt[:nq] == 0).all() and (cnt[nq:] == 7).all(), (nq, k, ef)
    idx.close()
    # a 0 % filter spills every query: cancelled in flight, its wait reports it and runs no spill tier
    g = chain(rng, "euclidean", n=20000, dim=32)
    x = g["vectors"]
    idx = index(ctx, x, g, "euclidean", "F32")
    queries = (x[rng.integers(0, x.shape[0], 64)] + rng.normal(0, 0.5, (64, 32))).astype(np.float32)
    none = np.zeros(x.shape[0], bool)
    want = idx.search_graph_filtered(queries, 10, 10, none, counters=True)
    assert idx.last_spilled() == queries.shape[0]
    t = idx.submit_graph_filtered(queries, 10, 10, none, counters=True)
    launches = ctx.kernel_launches()
    ctx.cancel()
    try:
        with pytest.raises(SdbError) as e:
            idx.wait(t)
        assert e.value.status == L.SDB_ECANCELLED
        assert ctx.kernel_launches() == launches  # no spill tier
        with pytest.raises(SdbError) as e:  # the flag up at submit: no ticket
            idx.submit_graph(queries, 10, 10)
        assert e.value.status == L.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    assert same_answer(idx.wait(idx.submit_graph_filtered(queries, 10, 10, none, counters=True)), want)
    idx.close()


# ---------------------------------------------------------------- 6. buffer lifetimes, handle operations, allocations
def test_lifetimes_and_handle_operations():
    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.hnsw import HnswIndex
    live0 = live()
    ctx = Context(0)  # its own context: everything the test allocates is released by the closes below
    rng = np.random.default_rng(9600)
    g = chain(rng, "euclidean", n=6000, dim=32)
    x = g["vectors"]
    n, dim = x.shape
    nq, k, ef = 64, 10, 20
    queries = (x[rng.integers(0, n, nq)] + rng.normal(0, 0.5, (nq, dim))).astype(np.float32)
    masks = np.stack([rng.random(n) < 0.5, rng.random(n) < 0.002, np.ones(n, bool)])
    qf = (np.arange(nq) % 3).astype(np.uint32)
    layers = [(torch.from_numpy(rp.astype(np.int64)).cuda(),
               torch.from_numpy(ci.astype(np.int32) if ci.size else np.zeros(1, np.int32)).cuda())
              for rp, ci in g["layers"]]
    idx = HnswIndex.from_device(ctx, torch.from_numpy(x).cuda(), layers, 0, "EUCLIDEAN")
    words = idx.filter_words(masks)
    want = idx.search_graph_filtered(queries, k, ef, words, query_filter=qf, counters=True)
    # query_filter is copied by submit: overwriting it at once changes nothing
    out = [np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32),
           np.zeros((nq, 2), np.uint64)]
    mine = qf.copy()
    tk = C.c_uint32()
    for rnd in range(2):  # the second round reuses the slots: the live allocations are then at their baseline
        L.check(L.lib().sdb_hnsw_submit_filtered(idx.h, p(queries), nq, k, ef, p(words), 3, p(mine), *map(p, out),
                                                 C.byref(tk)))
        mine[:] = 2 - mine
        L.check(L.lib().sdb_hnsw_wait(idx.h, tk.value))
        assert same_answer(out, want)
        mine[:] = qf
        t = idx.submit_graph(queries, k, ef)
        idx.wait(t)
        if rnd == 0:
            base = live()
    assert live() == base
    # set_layers_device is refused while a ticket is in flight, accepted after its wait
    RP = (C.c_void_p * len(layers))(*[t[0].data_ptr() for t in layers])
    CI = (C.c_void_p * len(layers))(*[t[1].data_ptr() for t in layers])
    t = idx.submit_graph_filtered(queries, k, ef, words, query_filter=qf, counters=True)
    assert L.lib().sdb_hnsw_set_layers_device(idx.h, len(layers), RP, CI, 0) == L.SDB_EINVAL
    assert same_answer(idx.wait(t), want)
    assert L.lib().sdb_hnsw_set_layers_device(idx.h, len(layers), RP, CI, 0) == L.SDB_OK
    assert same_answer(idx.search_graph_filtered(queries, k, ef, words, query_filter=qf, counters=True), want)
    # destroy with tickets in flight returns, and frees them
    for ef_i in (10, 20, 40):
        idx.submit_graph_filtered(queries, k, ef_i, words, query_filter=qf)
    idx.submit_graph(queries, k, ef)
    idx.close()
    ctx.close()
    assert live() == live0
