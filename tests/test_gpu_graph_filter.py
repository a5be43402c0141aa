"""WHERE-filtered graph hops on the GPU (sdb_graph_expand_filtered[_device], sdb_graph_collect_filtered) against the
CPU restatement (tests/graph_filter_ref.py), the unfiltered oracle over the pruned CSR and the reference's language
tests."""
import contextlib
import ctypes as C
import gc
import json
import os

import numpy as np
import pytest

import graph_filter_ref as R
from oracle import pyoracle as O
from test_graph_filter_ref import COND, pruned, statements, store

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "graph_relations.json")))


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


@pytest.fixture(scope="module")
def st(ctx):
    return store(ctx)


def fmt(names):
    return "[" + ", ".join(names) + "]"


def test_language_tests_through_lookup_filtered(st):
    cases = statements()
    for stmt, want, run in cases:
        assert run(st.lookup_filtered) == want, stmt
    assert len(cases) == 19


def test_dataset_collect_and_recursion_filtered(st):
    # a condition every record satisfies gives the unfiltered language-test results (cycles_collect, depth_fixed)
    every = lambda p: True  # noqa: E731
    c = G["cases"]["cycles_collect.surql"]["results"]
    assert fmt(st.collect_filtered("person:alice", "out", "knows", every, None, 1, 6, False)) == c[0]
    assert fmt(st.collect_filtered("person:alice", "out", "knows", None, every, 1, 6, True)) == c[1]
    c = G["cases"]["depth_fixed.surql"]["results"]
    for n in (1, 2, 3, 4):
        assert fmt(st.recurse_filtered("person:alice", "out", "reports_to", every, every, n, n)) == c[n - 1]
    # `.{..+collect}->(knows WHERE strength = "strong")->person` and friends, against the CPU restatement
    strong, moderate = COND['strength = "strong"'], lambda p: p.get("strength") != "weak"
    for d in ("out", "in", "both"):
        rp, ci = st.csr_arrays("knows", d)
        for ep, tp in ((strong, None), (moderate, None), (None, lambda p: p["id"] != "person:bob"), (moderate, lambda p: p["id"] != "person:dana")):
            em, tm = st.hop_masks("knows", d, ep, tp)
            for start in ("person:alice", "person:dana", "person:dir_platform"):
                for inc, mx in ((False, 0), (True, 0), (False, 2)):
                    want = R.collect(rp, ci, st.ids([start]), None if em is None else _words(em),
                                     None if tm is None else _words(tm), 1, mx, inc)
                    assert st.collect_filtered(start, d, "knows", ep, tp, 1, mx, inc) == st.to_names(want), (d, start, inc, mx)


def test_bidirectional_edge_record_masks(st):
    # `<->(knows WHERE strength = "strong")<->person`: the mask marks both positions of a record at each endpoint
    strong = COND['strength = "strong"']
    rp, ci = st.csr_arrays("knows", "both")
    em, _ = st.hop_masks("knows", "both", strong, None)
    recs = st.edge_records("knows", "both")
    assert all(em[p] == (st.edge_props[recs[p]]["strength"] == "strong") for p in range(len(recs)))
    for start in ("person:alice", "person:lead_infra", "person:dir_platform", "person:dana"):
        got = st.lookup_filtered([start], [("both", "knows", strong, None)])
        assert got == st.to_names(R.hop(rp, ci, st.ids([start]), _words(em))), start
        two = st.lookup_filtered([start], [("both", "knows", strong, None), ("out", "knows", None, None)])
        assert two == [x for n in got for x in st.lookup([n], [("out", "knows")])]


def _words(mask):
    from surrealdb_b200.graph import pack_bits
    return pack_bits(np.asarray(mask, bool))


def rmat_with_hub(n_log2, n_edges, hub_edges, seed):
    """R-MAT (a,b,c,d = .57,.19,.19,.05) on 2^n_log2 nodes plus node 2^n_log2 - 1 (almost never a target) with hub_edges more
    out-edges; CSR rows in
    (src, dst) order"""
    rng = np.random.default_rng(seed)
    m = n_edges + hub_edges
    src = np.zeros(m, np.int64)
    dst = np.zeros(m, np.int64)
    for _ in range(n_log2):
        r = rng.random(m)
        src = (src << 1) | (r >= 0.76)
        dst = (dst << 1) | (((r >= 0.57) & (r < 0.76)) | (r >= 0.95))
    src[n_edges:] = (1 << n_log2) - 1
    order = np.lexsort((dst, src))
    n = 1 << n_log2
    rp = np.zeros(n + 1, np.uint64)
    rp[1:] = np.cumsum(np.bincount(src, minlength=n))
    return rp, dst[order].astype(np.uint32)


@pytest.fixture(scope="module")
def big(ctx):
    from surrealdb_b200.graph import CsrGraph
    rp, ci = rmat_with_hub(16, 1_500_000, (1 << 20) + 77, 21)
    deg = np.diff(rp.astype(np.int64))
    assert deg.max() >= 1 << 20
    rng = np.random.default_rng(5)
    frontier = rng.choice(np.nonzero(deg > 0)[0], 300).astype(np.uint32)
    frontier[[7, 100, 101]] = rp.size - 2  # the hub, three times (twice in a row)
    frontier[50] = frontier[51]
    return CsrGraph(ctx, rp, ci), rp, ci, frontier


@pytest.mark.parametrize("density", [0.0, 0.01, 0.5, 1.0])
@pytest.mark.parametrize("limit", [0, 1, 3, 10**6])
def test_rmat_hub_edge_and_target_bitmaps(big, density, limit):
    from surrealdb_b200.graph import expand, expand_filtered
    g, rp, ci, frontier = big
    rng = np.random.default_rng(int(density * 1000) + limit % 1000)
    n = rp.size - 1
    em = rng.random(ci.size) < density
    tm = rng.random(n) < density
    for eb, tb in ((em, None), (None, tm), (em, tm)):
        got = expand_filtered([g], [(eb, tb)], frontier, limit)
        want = R.hop(rp, ci, frontier, None if eb is None else _words(eb), None if tb is None else _words(tb), limit)
        assert got.size == want.size and np.array_equal(got, want), (eb is None, tb is None, got.size, want.size)
    if density == 1.0:  # all ones: bit-identical to the unfiltered call
        assert np.array_equal(got, expand([g], frontier, limit))
    if density == 0.0:
        assert got.size == 0


@pytest.mark.parametrize("limit", [0, 3])
def test_null_and_all_ones_bitmaps_equal_the_unfiltered_expand(big, limit):
    from surrealdb_b200.graph import expand, expand_filtered
    g, rp, ci, frontier = big
    want = expand([g, g], frontier[:40], limit)
    ones_e, ones_t = np.ones(ci.size, bool), np.ones(rp.size - 1, bool)
    for filters in ([None, None], [(None, None), (None, None)], [(ones_e, None), (None, ones_t)], [(ones_e, ones_t)] * 2,
                    [(np.full((ci.size + 31) // 32, 0xFFFFFFFF, np.uint32), None), None]):
        got = expand_filtered([g, g], filters, frontier[:40], limit)
        assert got.tobytes() == want.tobytes()
    zeros = [(np.zeros(ci.size, bool), None), None]
    assert expand_filtered([g, g], zeros, frontier, limit).size == 0
    assert expand_filtered([g, g], [None, (None, np.zeros(rp.size - 1, bool))], frontier, limit).size == 0


@pytest.fixture(scope="module")
def mid(ctx):
    from surrealdb_b200.graph import CsrGraph
    rp, ci = rmat_with_hub(16, 300_000, 0, 21)
    rng = np.random.default_rng(5)
    frontier = rng.choice(np.nonzero(np.diff(rp.astype(np.int64)) > 0)[0], 30).astype(np.uint32)
    return CsrGraph(ctx, rp, ci), rp, ci, frontier


@pytest.mark.parametrize("limit", [0, 1, 3, 10**6])
def test_multi_hop_chains_mix_filtered_and_unfiltered_hops(mid, limit):
    import torch
    from surrealdb_b200.graph import device_free, expand_filtered, expand_filtered_device
    g, rp, ci, fr = mid
    rng = np.random.default_rng(limit % 97)
    n = rp.size - 1
    em, tm = rng.random(ci.size) < 0.3, rng.random(n) < 0.5
    pr_e = pruned(rp, ci, em, np.ones(n, bool))
    pr_t = pruned(rp, ci, np.ones(ci.size, bool), tm)
    pr_et = pruned(rp, ci, em, tm)
    for filters, csrs in (([(em, None), None, (None, tm)], [pr_e, (rp, ci), pr_t]),
                          ([None, (em, tm), None], [(rp, ci), pr_et, (rp, ci)]),
                          ([(em, tm), (None, tm)], [pr_et, pr_t])):
        want = fr
        for rp2, ci2 in csrs:
            want = O.graph_hop(rp2, ci2, want, limit)
        got = expand_filtered([g] * len(filters), filters, fr, limit)
        assert got.size == want.size and np.array_equal(got, want), ([f is None for f in filters], got.size, want.size)
        # the device variant: bitmaps, frontier and result in HBM
        d_bits = [None if f is None else tuple(None if m is None else torch.from_numpy(_words(m).view(np.int32)).cuda()
                                                for m in f) for f in filters]
        d_fr = torch.from_numpy(fr.view(np.int32)).cuda()
        torch.cuda.synchronize()
        ptr, cnt = expand_filtered_device(g.ctx, [g] * len(filters), d_bits, d_fr.data_ptr(), fr.size, limit)
        assert cnt == want.size
        if cnt:
            assert np.array_equal(_d2h(ptr, cnt), want)
        device_free(g.ctx, ptr)
    assert want.size > (1000 if limit == 0 else 10)


class _Dev:
    """n uint32 at a device pointer, as torch sees them (__cuda_array_interface__)"""
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def _d2h(ptr, n):
    import torch
    return torch.as_tensor(_Dev(ptr, n), device="cuda").cpu().numpy().view(np.uint32)


def test_zero_degree_sources_and_edge_cases(ctx):
    from surrealdb_b200 import SdbError
    from surrealdb_b200.graph import CsrGraph, expand_filtered
    # a tile spanning thousands of zero-degree sources (the kernel's global-search path)
    n = 20000
    deg = np.zeros(n, np.int64)
    deg[::5000] = 3000
    rp = np.concatenate([[0], np.cumsum(deg)]).astype(np.uint64)
    ci = (np.arange(rp[-1]) % n).astype(np.uint32)
    g = CsrGraph(ctx, rp, ci)
    fr = np.arange(n, dtype=np.uint32)
    em = (np.arange(ci.size) % 3) != 1
    tm = (np.arange(n) % 7) != 0
    for limit in (0, 5, 10**6):
        assert np.array_equal(expand_filtered([g], [(em, tm)], fr, limit), R.hop(rp, ci, fr, _words(em), _words(tm), limit))
    assert expand_filtered([g], [(em, tm)], np.zeros(0, np.uint32)).size == 0
    with pytest.raises(SdbError) as e:
        expand_filtered([g], [(em, None)], [0, n])
    assert "out of range" in str(e.value)
    with pytest.raises(ValueError):
        expand_filtered([g, g], [(em, None)], [0])


@pytest.mark.parametrize("inclusive", [False, True])
def test_rmat_collect_filtered_equals_oracle(ctx, inclusive):
    from surrealdb_b200.graph import CsrGraph, collect, collect_filtered
    rp, ci = rmat_with_hub(14, 100_000, 5000, 8)
    g = CsrGraph(ctx, rp, ci)
    n = rp.size - 1
    rng = np.random.default_rng(3 + inclusive)
    for de, dt in ((0.5, 1.0), (1.0, 0.6), (0.7, 0.7), (0.01, 1.0), (0.0, 1.0)):
        em, tm = rng.random(ci.size) < de, rng.random(n) < dt
        for start, mn, mx in ((1, 1, 0), (77, 2, 4), (123, 1, 3), (9000, 1, 0), (rp.size - 2, 1, 2)):
            want = O.graph_collect(*pruned(rp, ci, em, tm), [start], mn, mx, inclusive)
            got = collect_filtered(g, (em, tm), [start], mn, mx, inclusive)
            assert np.array_equal(got, want), (de, dt, start, mn, mx, got.size, want.size)
            if de == 1.0 and dt == 1.0:
                assert np.array_equal(got, collect(g, [start], mn, mx, inclusive))
    ones = np.ones(ci.size, bool)
    assert np.array_equal(collect_filtered(g, (ones, None), [1], 1, 0, inclusive), collect(g, [1], 1, 0, inclusive))
    assert np.array_equal(collect_filtered(g, None, [1], 1, 3, inclusive), collect(g, [1], 1, 3, inclusive))


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


def test_refusals_and_buffers_back_at_baseline():
    import torch
    from surrealdb_b200 import Context, SdbError
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.graph import (CsrGraph, CsrGraphShard, collect_filtered, device_free, expand_filtered,
                                      expand_filtered_device)
    rp, ci = rmat_with_hub(12, 40_000, 3000, 4)
    n = rp.size - 1
    em, tm = (np.arange(ci.size) % 2) == 0, (np.arange(n) % 3) != 0
    with no_leaks():
        ctx = Context(0)
        g = CsrGraph(ctx, rp, ci)
        fr = np.arange(0, n, 7, dtype=np.uint32)
        for limit in (0, 2):
            assert expand_filtered([g, g], [(em, tm), (None, tm)], fr, limit).size > 0
        assert collect_filtered(g, (em, tm), [1], 1, 0, True).size > 0
        d_fr = torch.from_numpy(fr.view(np.int32)).cuda()
        d_e = torch.from_numpy(_words(em).view(np.int32)).cuda()
        torch.cuda.synchronize()
        ptr, cnt = expand_filtered_device(ctx, [g], [(d_e, None)], d_fr.data_ptr(), fr.size, 3)
        assert cnt > 0 and ptr
        device_free(ctx, ptr)
        # refused calls leave nothing behind
        with pytest.raises(SdbError) as e:
            expand_filtered([g, g], [(em, tm), None], [0, n + 5])
        assert e.value.status == L.SDB_EINVAL
        with pytest.raises(SdbError) as e:
            collect_filtered(g, (em, None), [n])
        assert e.value.status == L.SDB_EINVAL
        shard = CsrGraphShard(ctx, rp, ci, 0, n)
        for call in (lambda: expand_filtered([shard], [(em, None)], [1]),
                     lambda: expand_filtered([g, shard], [None, None], [1]),
                     lambda: collect_filtered(shard, (None, tm), [1]),
                     lambda: expand_filtered_device(ctx, [shard], [None], d_fr.data_ptr(), 1)):
            with pytest.raises(SdbError) as e:
                call()
            assert e.value.status == L.SDB_EUNSUPPORTED and "shard" in str(e.value)
        # a target condition needs every target inside the rows
        other = CsrGraph(ctx, np.array([0, 2, 3], np.uint64), np.array([1, 5, 0], np.uint32))
        with pytest.raises(SdbError) as e:
            expand_filtered([other], [(None, np.ones(2, bool))], [0])
        assert e.value.status == L.SDB_EINVAL
        assert expand_filtered([other], [(np.array([False, True, True]), None)], [0, 1]).tolist() == [5, 0]
        del d_fr, d_e
        torch.cuda.synchronize()
        for h in (g, shard, other):
            h.close()
        ctx.close()
