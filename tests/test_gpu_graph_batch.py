"""Batches of documents through one graph call (sdb_graph_expand_batch[_device], sdb_graph_collect_batch): every
document's segment of the output against the oracle applied to that document alone, the flat calls, the reference's
multi-row language tests, shard handles, refusals and buffer hygiene."""
import contextlib
import ctypes as C
import gc
import json
import os
import re

import numpy as np
import pytest

import graph_filter_ref as R
from oracle import pyoracle as O
from test_graph_filter_ref import store

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
G = json.load(open(os.path.join(HERE, "golden", "graph_relations.json")))
F = json.load(open(os.path.join(HERE, "golden", "graph_filters.json")))
P = json.load(open(os.path.join(HERE, "golden", "graph_path_collect.json")))


def rmat_with_hub(n_log2, n_edges, hub_edges, seed, cyclic=False):
    """R-MAT (a,b,c,d = .57,.19,.19,.05) on 2^n_log2 nodes plus hub_edges more out-edges of node 2^n_log2 - 1; CSR rows
    in (src, dst) order.  cyclic: every node also gets an edge to (v + 1) mod n, so every BFS runs around cycles"""
    rng = np.random.default_rng(seed)
    m = n_edges + hub_edges
    src = np.zeros(m, np.int64)
    dst = np.zeros(m, np.int64)
    for _ in range(n_log2):
        r = rng.random(m)
        src = (src << 1) | (r >= 0.76)
        dst = (dst << 1) | (((r >= 0.57) & (r < 0.76)) | (r >= 0.95))
    n = 1 << n_log2
    src[n_edges:] = n - 1
    if cyclic:
        src = np.concatenate([src, np.arange(n)])
        dst = np.concatenate([dst, (np.arange(n) + 1) % n])
    order = np.lexsort((dst, src))
    rp = np.zeros(n + 1, np.uint64)
    rp[1:] = np.cumsum(np.bincount(src, minlength=n))
    return rp, dst[order].astype(np.uint32)


def words(mask):
    from surrealdb_b200.graph import pack_bits
    return pack_bits(np.asarray(mask, bool))


def make_docs(rng, rp, n_docs):
    """empty, one-id, many-id and repeated documents, hubs and zero-degree sources among them"""
    n = rp.size - 1
    deg = np.diff(rp.astype(np.int64))
    hub, zero = int(np.argmax(deg)), np.nonzero(deg == 0)[0]
    docs = []
    for d in range(n_docs):
        k = d % 7
        if k == 0:
            docs.append(np.zeros(0, np.uint32))
        elif k in (1, 2):
            docs.append(rng.integers(0, n, 1).astype(np.uint32))
        elif k == 3:
            docs.append(rng.integers(0, n, rng.integers(2, 12)).astype(np.uint32))
        elif k == 4:
            docs.append(np.array([hub] + ([int(zero[d % zero.size])] if zero.size else []), np.uint32))
        elif k == 5 and docs:
            docs.append(docs[rng.integers(0, len(docs))].copy())
        else:
            docs.append(np.array([int(zero[d % zero.size]) if zero.size else 0], np.uint32))
    return docs


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


@pytest.fixture(scope="module")
def hubby(ctx):
    from surrealdb_b200.graph import CsrGraph
    rp, ci = rmat_with_hub(14, 200_000, 30_000, 11)
    return CsrGraph(ctx, rp, ci), rp, ci


@pytest.mark.parametrize("n_docs", [0, 1, 2, 1000, 20_000])
@pytest.mark.parametrize("limit", [0, 1, 3, 10**6])
def test_expand_batch_per_document_equals_oracle(hubby, n_docs, limit):
    from surrealdb_b200.graph import expand, expand_batch
    g, rp, ci = hubby
    rng = np.random.default_rng(n_docs * 7 + limit % 1000)
    docs = make_docs(rng, rp, n_docs)
    # the hub's 30k edges make a 3-hop unlimited chain explode; big batches keep to 1-2 hops there
    max_hops = 3 if (limit and limit <= 3) or n_docs <= 2 else (2 if n_docs <= 1000 else 1)
    for n_hops in range(1, max_hops + 1):
        got = expand_batch([g] * n_hops, docs, limit)
        assert len(got) == n_docs
        for d, doc in enumerate(docs):
            want = doc
            for _ in range(n_hops):
                want = O.graph_hop(rp, ci, want, limit)
            assert got[d].tobytes() == want.tobytes(), (n_hops, d, got[d].size, want.size)
        flat = np.concatenate(docs) if docs else np.zeros(0, np.uint32)
        cat = np.concatenate(got) if got else np.zeros(0, np.uint32)
        assert cat.tobytes() == expand([g] * n_hops, flat, limit).tobytes()


@pytest.mark.parametrize("density", [0.0, 0.01, 0.5, 1.0])
@pytest.mark.parametrize("limit", [0, 1, 3, 10**6])
def test_filtered_batch_mixed_chain_equals_reference(hubby, density, limit):
    from surrealdb_b200.graph import expand_batch, expand_filtered
    g, rp, ci = hubby
    n = rp.size - 1
    rng = np.random.default_rng(int(density * 100) + limit % 997)
    em, tm = rng.random(ci.size) < density, rng.random(n) < density
    docs = make_docs(rng, rp, 150)
    flat = np.concatenate(docs)
    for filters in ([(em, None)], [(None, tm)], [(em, tm)], [(em, None), None], [None, (em, tm)],
                    [(None, tm), None, (em, None)]):
        hops = [(rp, ci, None if f is None or f[0] is None else words(f[0]), None if f is None or f[1] is None else
                 words(f[1])) for f in filters]
        if len(filters) == 3 and limit not in (1, 3):
            continue  # three hops through the hub with a large limit leave the 2^32-id range
        got = expand_batch([g] * len(filters), docs, limit, filters)
        for d, doc in enumerate(docs):
            assert np.array_equal(got[d], R.chain(hops, doc, limit)), ([f is None for f in filters], d)
        assert np.concatenate(got).tobytes() == expand_filtered([g] * len(filters), filters, flat, limit).tobytes()


def test_device_batch_equals_host_batch(hubby):
    import torch
    from surrealdb_b200.graph import device_free, expand_batch, expand_batch_device
    g, rp, ci = hubby
    rng = np.random.default_rng(3)
    n = rp.size - 1
    docs = make_docs(rng, rp, 1000)
    flat = np.concatenate(docs)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([d.size for d in docs])
    em, tm = rng.random(ci.size) < 0.5, rng.random(n) < 0.5
    d_fr = torch.from_numpy(flat.view(np.int32)).cuda()
    d_off = torch.from_numpy(off.view(np.int64)).cuda()
    d_out_off = torch.zeros(off.size, dtype=torch.int64, device="cuda")
    d_e, d_t = (torch.from_numpy(words(m).view(np.int32)).cuda() for m in (em, tm))
    torch.cuda.synchronize()
    for limit in (0, 3):
        for host_f, dev_f in ((None, None), ([(em, None), (None, tm)], [(d_e, None), (None, d_t)]),
                              ([None, (em, tm)], [None, (d_e, d_t)])):
            want = expand_batch([g, g], docs, limit, host_f)
            ptr, cnt = expand_batch_device(g.ctx, [g, g], d_fr.data_ptr(), flat.size, d_off.data_ptr(), len(docs),
                                           d_out_off.data_ptr(), limit, dev_f)
            got_off = d_out_off.cpu().numpy().view(np.uint64)
            want_off = np.concatenate([[0], np.cumsum([w.size for w in want])]).astype(np.uint64)
            assert np.array_equal(got_off, want_off)
            assert cnt == int(want_off[-1])
            if cnt:
                assert np.array_equal(_d2h(ptr, cnt), np.concatenate(want))
            device_free(g.ctx, ptr)


class _Dev:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def _d2h(ptr, n):
    import torch
    return torch.as_tensor(_Dev(ptr, n), device="cuda").cpu().numpy().view(np.uint32)


@pytest.fixture(scope="module")
def cyclic(ctx):
    from surrealdb_b200.graph import CsrGraph
    rp, ci = rmat_with_hub(11, 6000, 500, 12, cyclic=True)
    return CsrGraph(ctx, rp, ci), rp, ci


@pytest.mark.parametrize("inclusive", [False, True])
@pytest.mark.parametrize("n_docs", [0, 1, 2, 1000])
def test_collect_batch_per_document_equals_oracle(cyclic, inclusive, n_docs):
    from surrealdb_b200.graph import collect, collect_batch
    g, rp, ci = cyclic
    rng = np.random.default_rng(n_docs + 10 * inclusive)
    docs = make_docs(rng, rp, n_docs)
    for mn, mx in ((0, 0), (1, 0), (2, 4), (3, 3), (1, 1), (0, 2)):
        got = collect_batch(g, docs, mn, mx, inclusive)
        assert len(got) == n_docs
        for d, doc in enumerate(docs):
            want = O.graph_collect(rp, ci, doc, mn, mx, inclusive)
            assert np.array_equal(got[d], want), (mn, mx, d, got[d].size, want.size)
            if d < 5:
                assert np.array_equal(got[d], collect(g, doc, mn, mx, inclusive))


@pytest.mark.parametrize("density", [0.0, 0.01, 0.5, 1.0])
def test_collect_batch_filtered_equals_reference(cyclic, density):
    from surrealdb_b200.graph import collect_batch
    g, rp, ci = cyclic
    n = rp.size - 1
    rng = np.random.default_rng(int(density * 100) + 1)
    em, tm = rng.random(ci.size) < density, rng.random(n) < density
    docs = make_docs(rng, rp, 200)
    for filt in ((em, None), (None, tm), (em, tm)):
        eb, tb = (None if m is None else words(m) for m in filt)
        for mn, mx, inc in ((1, 0, False), (0, 3, True), (2, 0, True), (3, 5, False)):
            got = collect_batch(g, docs, mn, mx, inc, filt)
            for d, doc in enumerate(docs):
                assert np.array_equal(got[d], R.collect(rp, ci, doc, eb, tb, mn, mx, inc)), (mn, mx, inc, d)


def test_collect_batch_is_not_dense_and_grows_its_table(ctx):
    # 20k documents on a sparse 2^22-node graph: n_docs x n_rows x 4 bytes = 335 GB of dense per-document state
    from surrealdb_b200.graph import CsrGraph, collect_batch, last_collect_table
    n = 1 << 22
    rng = np.random.default_rng(14)
    deg = rng.integers(0, 4, n)
    rp = np.concatenate([[0], np.cumsum(deg)]).astype(np.uint64)
    ci = rng.integers(0, n, int(rp[-1])).astype(np.uint32)
    g = CsrGraph(ctx, rp, ci)
    docs = [rng.integers(0, n, 1 + d % 3).astype(np.uint32) for d in range(20_000)]
    got = collect_batch(g, docs, 1, 3, False)
    diag = last_collect_table(g)
    assert diag["grows"] >= 1  # the visited pairs outgrew the table it started with
    total = sum(x.size for x in got)
    assert total > 100_000 and diag["peak_bytes"] < 100 * total
    for d in range(0, 20_000, 97):
        assert np.array_equal(got[d], O.graph_collect(rp, ci, docs[d], 1, 3, False)), d


@pytest.mark.parametrize("inclusive", [False, True])
def test_collect_batch_levels_that_overflow_the_table_repeat_in_a_larger_one(cyclic, monkeypatch, inclusive):
    # capping the table's size before a level makes every large level overflow it mid-pass: the pass repeats in a
    # table twice the size (rehashed), and the result is still every document's own
    from surrealdb_b200.graph import collect, collect_batch, last_collect_table
    g, rp, ci = cyclic
    docs = make_docs(np.random.default_rng(40 + inclusive), rp, 1000)
    want = collect_batch(g, docs, 1, 0, inclusive)
    monkeypatch.setenv("SDB_DEBUG_PAIR_TABLE_SLOTS", "64")
    got = collect_batch(g, docs, 1, 0, inclusive)
    diag = last_collect_table(g)
    assert diag["repeated_passes"] >= 2 and diag["grows"] >= 2
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    for d in range(0, 1000, 37):
        assert np.array_equal(got[d], collect(g, docs[d], 1, 0, inclusive)), d


def test_collect_batch_splits_documents_whose_summed_level_exceeds_2_32(ctx, monkeypatch):
    # node 0 has 2^22 edges, all to node 1: one document [0] has a level of 2^22 ids, 1025 of them 2^32 + 2^22 --
    # more than one hop may hold, while every document alone and the whole result (1025 x 1 ids) fit
    from surrealdb_b200.graph import CsrGraph, collect, collect_batch, last_collect_table
    deg = 1 << 22
    rp = np.array([0, deg, deg, deg], np.uint64)
    ci = np.ones(deg, np.uint32)
    g = CsrGraph(ctx, rp, ci)
    monkeypatch.setenv("SDB_DEBUG_PAIR_TABLE_SLOTS", "4096")  # one distinct pair per document: keep the table small
    docs = [[0]] * 1025 + [[2]]
    got = collect_batch(g, docs, 1, 0, True)
    assert last_collect_table(g)["splits"] >= 1
    assert [x.tolist() for x in got] == [[0, 1]] * 1025 + [[2]]
    assert np.array_equal(got[0], collect(g, [0], 1, 0, True))


def fmt_names(names):
    return "[" + ", ".join(f"'{x}'" for x in names) + "]"


def test_language_tests_in_one_batch_call_each(ctx):
    st = store(ctx)
    name = lambda ids: [st.node_props[i]["name"] for i in ids]  # noqa: E731
    level5 = sorted((k for k, v in F["node_props"].items() if k.startswith("person:") and v.get("level") == 5),
                    key=lambda k: k.split(":")[1])
    # traversal_forward.surql 4: SELECT id, name, ->knows->person.name AS knows FROM person:alice, person:bob
    rows = ["person:alice", "person:bob"]
    knows = st.lookup_batch([[r] for r in rows], [("out", "knows")])
    got = "[" + ", ".join(f"{{ id: {r}, knows: {fmt_names(name(k))}, name: '{name([r])[0]}' }}"
                          for r, k in zip(rows, knows)) + "]"
    assert got == G["cases"]["traversal_forward.surql"]["results"][4]
    # traversal_forward.surql 5: SELECT name, @->reports_to->person.name AS manager FROM person WHERE level = 5
    mgr = st.lookup_batch([[r] for r in level5], [("out", "reports_to")])
    got = "[" + ", ".join(f"{{ manager: {fmt_names(name(m))}, name: '{name([r])[0]}' }}" for r, m in zip(level5, mgr)) + "]"
    assert got == G["cases"]["traversal_forward.surql"]["results"][5]
    # path_collect.surql 4: SELECT name, @.{..+collect}(->reports_to->person).name AS managers FROM person WHERE level = 5
    case = P["cases"]["path_collect.surql"]
    assert re.search(r"\{\.\.\+collect\}", case["statements"][4])
    col = st.collect_batch([[r] for r in level5], "out", "reports_to", None, None, 1, 256, False)
    got = "[" + ", ".join(f"{{ managers: {fmt_names(name(m))}, name: '{name([r])[0]}' }}" for r, m in zip(level5, col)) + "]"
    assert got == case["results"][4]
    # the single-record statements 0, 1 and 3 as a batch of three rows
    three = st.collect_batch([["person:alice"]] * 2, "out", "reports_to", None, None, 1, 256, False)
    three += st.collect_batch([["person:alice"]], "out", "reports_to", None, None, 1, 3, False)
    for i, res in zip((0, 1, 3), three):
        assert "[" + ", ".join(res) + "]" == case["results"][i]
    # with a filter: per row equals collect_filtered of that row
    strong = lambda p: p.get("strength") != "weak"  # noqa: E731
    rows = ["person:alice", "person:dana", "person:bob"]
    got = st.collect_batch([[r] for r in rows], "out", "knows", strong, None, 1, 0, True)
    assert got == [st.collect_filtered(r, "out", "knows", strong, None, 1, 0, True) for r in rows]
    got = st.lookup_batch([[r] for r in rows], [("out", "knows", strong, None), ("out", "knows")])
    assert got == [st.lookup_filtered([r], [("out", "knows", strong, None), ("out", "knows", None, None)]) for r in rows]


def test_shard_handles_on_one_rank(ctx):
    from surrealdb_b200.graph import CsrGraph, CsrGraphShard, collect, collect_batch, expand, expand_batch
    rp, ci = rmat_with_hub(12, 40_000, 0, 61)
    n = rp.size - 1
    whole, full = CsrGraph(ctx, rp, ci), CsrGraphShard(ctx, rp, ci, 0, n)
    sub = CsrGraphShard(ctx, rp, ci, n // 4, n // 2)
    rng = np.random.default_rng(62)
    docs = make_docs(rng, rp, 500)
    for limit in (0, 7):
        want = expand_batch([whole, whole], docs, limit)
        got = expand_batch([full, full], docs, limit)
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
        # a sub-range shard alone on its rank: sources outside its rows expand to nothing, per document as flat
        got = expand_batch([sub], docs, limit)
        assert all(np.array_equal(a, expand([sub], d, limit)) for a, d in zip(got, docs))
    got = collect_batch(full, docs[:200], 1, 3, True)
    assert all(np.array_equal(a, collect(whole, d, 1, 3, True)) for a, d in zip(got, docs[:200]))


def test_shard_handles_two_gpus_threads():
    import threading
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from surrealdb_b200 import Context
    from surrealdb_b200.graph import CsrGraphShard, collect_batch, expand_batch
    rp, ci = rmat_with_hub(13, 90_000, 0, 63)
    n = rp.size - 1
    rng = np.random.default_rng(64)
    docs = make_docs(rng, rp, 700)
    want = []
    for d in docs:
        w = d
        for _ in range(3):
            w = O.graph_hop(rp, ci, w, 5)
        want.append(w)
    want_col = [O.graph_collect(rp, ci, d, 1, 4, False) for d in docs[:100]]
    ctxs = Context.create_multi([0, 1])
    cut = n // 3
    out, errs = [None, None], []

    def run(r):
        try:
            lo, hi = (0, cut) if r == 0 else (cut, n)
            g = CsrGraphShard(ctxs[r], rp, ci, lo, hi)
            out[r] = (expand_batch([g, g, g], docs, 5), collect_batch(g, docs[:100], 1, 4, False))
        except Exception as e:  # pragma: no cover
            errs.append(e)

    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    [t.start() for t in th]
    [t.join(120) for t in th]
    assert not errs, errs
    for r in range(2):
        assert all(np.array_equal(a, b) for a, b in zip(out[r][0], want))
        assert all(np.array_equal(a, b) for a, b in zip(out[r][1], want_col))


def live():
    from surrealdb_b200 import _lib as L
    n, b = C.c_uint64(), C.c_uint64()
    L.lib().sdb_debug_live_allocations(C.byref(n), C.byref(b))
    return n.value, b.value


@contextlib.contextmanager
def no_leaks():
    gc.collect()
    before = live()
    yield
    gc.collect()
    assert live() == before


def _raw_expand(g, fr, off, n_docs=None):
    from surrealdb_b200 import _lib as L
    fr = np.ascontiguousarray(fr, np.uint32)
    off = np.ascontiguousarray(off, np.uint64)
    arr = (C.c_void_p * 1)(g.h)
    out, n = C.c_void_p(), C.c_uint64()
    out_off = np.zeros(max(off.size, 1) + 1, np.uint64)
    return L.lib().sdb_graph_expand_batch(arr, None, 1, C.c_void_p(fr.ctypes.data) if fr.size else None, fr.size,
                                          C.c_void_p(off.ctypes.data), off.size - 1 if n_docs is None else n_docs, 0,
                                          C.byref(out), C.c_void_p(out_off.ctypes.data), C.byref(n))


def test_refusals_cancellation_and_buffers_back_at_baseline():
    import torch
    from surrealdb_b200 import Context, SdbError
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.graph import (CsrGraph, CsrGraphShard, collect_batch, device_free, expand_batch,
                                      expand_batch_device)
    rp, ci = rmat_with_hub(12, 40_000, 3000, 4, cyclic=True)
    n = rp.size - 1
    em, tm = (np.arange(ci.size) % 2) == 0, (np.arange(n) % 3) != 0
    with no_leaks():
        ctx = Context(0)
        g = CsrGraph(ctx, rp, ci)
        docs = [np.arange(i, n, 97, dtype=np.uint32)[:5] for i in range(50)]
        assert sum(x.size for x in expand_batch([g, g], docs, 2, [(em, tm), None])) > 0
        assert sum(x.size for x in collect_batch(g, docs, 1, 0, True, (em, None))) > 0
        # malformed doc_off shapes
        fr = np.array([1, 2, 3, 4], np.uint32)
        for off in ([1, 2, 4], [0, 3, 2, 4], [0, 2, 3], [0, 2, 5], [1]):
            assert _raw_expand(g, fr if off != [1] else [], off) == L.SDB_EINVAL, off
        assert _raw_expand(g, fr, [0, 4], 1 << 32) == L.SDB_EINVAL
        assert _raw_expand(g, [], [0]) == L.SDB_OK
        with pytest.raises(SdbError) as e:
            collect_batch(g, ([1, 2], [0, 1]))
        assert e.value.status == L.SDB_EINVAL
        # the device check of d_doc_off
        d_fr = torch.from_numpy(fr.view(np.int32)).cuda()
        d_out_off = torch.zeros(4, dtype=torch.int64, device="cuda")
        for off in ([0, 3, 2, 4], [1, 2, 4], [0, 2, 3], [0, 2, 9]):
            d_off = torch.tensor(off, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            with pytest.raises(SdbError) as e:
                expand_batch_device(ctx, [g], d_fr.data_ptr(), 4, d_off.data_ptr(), len(off) - 1, d_out_off.data_ptr())
            assert e.value.status == L.SDB_EINVAL, off
        d_off = torch.tensor([0, 1, 1, 4], dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ptr, cnt = expand_batch_device(ctx, [g], d_fr.data_ptr(), 4, d_off.data_ptr(), 3, d_out_off.data_ptr(), 0,
                                       [(None, None)])
        assert cnt > 0
        device_free(ctx, ptr)
        # ids out of range
        for call in (lambda: expand_batch([g], [[0], [n]]), lambda: collect_batch(g, [[0], [n + 3]]),
                     lambda: expand_batch([g], [[0], [n]], 0, [(em, None)])):
            with pytest.raises(SdbError) as e:
                call()
            assert e.value.status == L.SDB_EINVAL
        # filters on shard handles are refused; unfiltered batches on them are served
        shard = CsrGraphShard(ctx, rp, ci, 0, n)
        for call in (lambda: expand_batch([shard], docs, 0, [(em, None)]),
                     lambda: expand_batch([g, shard], docs, 0, [None, None]),
                     lambda: collect_batch(shard, docs, 1, 0, False, (None, tm)),
                     lambda: expand_batch_device(ctx, [shard], d_fr.data_ptr(), 4, d_off.data_ptr(), 3,
                                                 d_out_off.data_ptr(), 0, [None])):
            with pytest.raises(SdbError) as e:
                call()
            assert e.value.status == L.SDB_EUNSUPPORTED and "shard" in str(e.value)
        assert sum(x.size for x in expand_batch([shard], docs)) > 0
        # a CSR whose targets leave its rows: no target condition, no collect
        other = CsrGraph(ctx, np.array([0, 2, 3], np.uint64), np.array([1, 5, 0], np.uint32))
        with pytest.raises(SdbError) as e:
            expand_batch([other], [[0]], 0, [(None, np.ones(2, bool))])
        assert e.value.status == L.SDB_EINVAL
        with pytest.raises(SdbError) as e:
            collect_batch(other, [[0], [1]])
        assert e.value.status == L.SDB_EINVAL
        assert [x.tolist() for x in expand_batch([other], [[0], [], [1]], 0, [(np.array([False, True, True]), None)])] \
            == [[5], [], [0]]
        # cancellation, then a working call after the reset
        ctx.cancel()
        for call in (lambda: expand_batch([g], docs), lambda: collect_batch(g, docs)):
            with pytest.raises(SdbError) as e:
                call()
            assert e.value.status == L.SDB_ECANCELLED
        ctx.cancel_reset()
        assert sum(x.size for x in collect_batch(g, docs, 1, 2)) > 0
        del d_fr, d_off, d_out_off
        torch.cuda.synchronize()
        for h in (g, shard, other):
            h.close()
        ctx.close()
