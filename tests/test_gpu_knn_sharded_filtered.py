"""Filtered brute-force KNN on row-sharded columns (sdb_knn_sharded_*_filtered) and the asynchronous filtered submit
with device bitmaps (sdb_knn_submit_filtered_device).  The bitmaps cover the global rows; each shard slices its own
rows out of them.  Every shard's list is compared with the CPU oracle over its slice, and the shards' lists merged by
sdb_topk_merge_device with the unsharded sdb_knn_bruteforce_filtered and the oracle, bit for bit (rows, distances,
counts): oracle.knn_topk(corpus, q, metric, k, skip=skip | ~filter)."""
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


@pytest.fixture
def minkowski_order():
    def set_order(p):
        O.lib().orc_set_minkowski_order(C.c_double(float(p)))
    yield set_order
    set_order(3.0)


def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return np.ascontiguousarray(pack_row_filter(np.asarray(masks, bool)))


def make_col(ctx, rows, metric, base=None, screen=None, order=None):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if rows.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, rows.shape[1], metric, dt, capacity=max(1, rows.shape[0]))
    col.append(rows)
    col.finalize()
    if base is not None:
        col.set_row_base(base)
    if screen:
        col.set_screen(screen)
    if order is not None:
        col.set_minkowski_order(order)
    return col


def bounds(bases, n):
    return list(zip(bases, bases[1:] + [n]))


def shard_knn(col, queries, k, f, qf, n_total):
    """one rank: sdb_knn_sharded_submit_filtered + sdb_knn_sharded_wait (the merge of one block is a copy)"""
    q = np.ascontiguousarray(queries, np.float64)
    nq = q.shape[0]
    rows, dist, cnt = np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32)
    t = col.sharded_submit_filtered_host(q.ctypes.data, nq, k, f.ctypes.data, f.shape[0], qf, n_total,
                                         rows.ctypes.data, dist.ctypes.data, cnt.ctypes.data)
    col.sharded_wait(t)
    return rows, dist, cnt


def merge(ctx, parts, k):
    """the shards' lists merged by (distance, global row) with sdb_topk_merge_device, as after the exchange"""
    import torch
    from surrealdb_b200.engine import topk_merge_device
    dev = torch.device("cuda", ctx.device)
    nq = parts[0][2].size
    r = torch.from_numpy(np.stack([p[0] for p in parts]).view(np.int64)).to(dev)
    d = torch.from_numpy(np.stack([p[1] for p in parts])).to(dev)
    c = torch.from_numpy(np.stack([p[2] for p in parts]).view(np.int32)).to(dev)
    out = (torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
           torch.zeros(nq, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()  # torch's stream and the library's are not ordered with each other
    topk_merge_device(ctx, len(parts), nq, k, r.data_ptr(), d.data_ptr(), c.data_ptr(), out[0].data_ptr(),
                      out[1].data_ptr(), out[2].data_ptr())
    return (out[0].cpu().numpy().view(np.uint64), out[1].cpu().numpy(), out[2].cpu().numpy().view(np.uint32))


def same(a, b, qs=None):
    """equal results: counts, and rows / distances up to each count, bit for bit"""
    ra, da, ca = a
    rb, db, cb = b
    assert list(ca) == list(cb), (ca, cb)
    for q in range(len(ca)) if qs is None else qs:
        n = ca[q]
        assert ra[q, :n].tobytes() == rb[q, :n].tobytes(), (q, ra[q, :n], rb[q, :n])
        assert da[q, :n].tobytes() == db[q, :n].tobytes(), (q, da[q, :n], db[q, :n])


def oracle_check(corpus, queries, metric, k, masks, qf, res, base=0, qs=None):
    """res over corpus rows [base, base + len(corpus)) with global ids == the oracle over that slice"""
    rows, dist, cnt = res
    n = corpus.shape[0]
    for q in range(queries.shape[0]) if qs is None else qs:
        sk = (~masks[qf[q], base : base + n]).astype(np.uint8)
        r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=sk)
        assert cnt[q] == r.size, (q, int(cnt[q]), r.size)
        assert list(rows[q, : cnt[q]]) == list(r + np.uint64(base)), (q, rows[q, : cnt[q]], r + np.uint64(base))
        if metric == "MINKOWSKI":  # pow(): CUDA's libm and the host's differ by an ulp per term (tests/test_gpu_knn.py)
            np.testing.assert_allclose(dist[q, : cnt[q]], d, rtol=1e-12)
        else:
            assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, dist[q, : cnt[q]], d)


# ---- 1. one rank, several shards on one device: every family, F32 and F64, aligned and unaligned bases ----
FAMILIES = [("COSINE", "TC_INT8", None), ("COSINE", "TC_BF16", None), ("EUCLIDEAN", None, None),
            ("PEARSON", None, None), ("MANHATTAN", None, None), ("MINKOWSKI", None, 3.0), ("MINKOWSKI", None, 2.5),
            ("HAMMING", None, None), ("JACCARD", None, None)]


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric,screen,order", FAMILIES)
def test_shards_merge_to_the_unsharded_call(ctx, minkowski_order, dtype, metric, screen, order):
    from surrealdb_b200.sharding import shard_range
    rng = np.random.default_rng(zlib.crc32(f"{dtype}{metric}{screen}{order}".encode()))
    n, dim, nq, k = 9000 + 37, 24, 12, 10
    npdt = np.float32 if dtype == "F32" else np.float64
    if metric in ("HAMMING", "JACCARD"):  # repeated values: the counts see ties
        corpus = rng.integers(-3, 4, (n, dim)).astype(npdt)
        queries = rng.integers(-3, 4, (nq, dim)).astype(np.float64)
    else:
        corpus = rng.uniform(-1, 1, (n, dim)).astype(npdt)
        queries = rng.uniform(-1, 1, (nq, dim))
    if order is not None:
        minkowski_order(order)
    counts = [n, n // 2, n // 10, 90, 5000, 3]  # 5000 and 90: screened unsharded, direct on some shards
    masks = np.zeros((len(counts), n), bool)
    for i, c in enumerate(counts):
        masks[i, rng.choice(n, c, replace=False)] = True
    f = pack(masks)
    qf = (np.arange(nq) % len(counts)).astype(np.uint32)
    whole = make_col(ctx, corpus, metric, screen=screen, order=order)
    want = whole.knn(queries, k, filters=f, query_filter=qf)
    oracle_check(corpus, queries, metric, k, masks, qf, want)
    aligned = [shard_range(n, 3, r)[0] for r in range(3)]
    for bases in (aligned, [0, 31, 33, 5003]):
        parts = []
        for lo, hi in bounds(bases, n):
            col = make_col(ctx, corpus[lo:hi], metric, base=lo, screen=screen, order=order)
            part = shard_knn(col, queries, k, f, qf, n)
            oracle_check(corpus[lo:hi], queries, metric, k, masks, qf, part, base=lo)  # its own slice, global ids
            parts.append(part)
            col.close()
        same(merge(ctx, parts, k), want)


# ---- 2. the bits around a shard's slice ----
def test_adversarial_bits_around_the_slice(ctx):
    rng = np.random.default_rng(21)
    n, dim, nq, k = 18000, 32, 8, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    bases = [0, 5003, 12001]
    lo, hi = 5003, 12001  # the middle shard
    masks = np.ones((3, n), bool)  # every row of the neighbouring shards passes, 12001.. (past the end) included
    masks[:, lo:hi] = False
    masks[0, lo] = True  # only the shard's first row
    masks[1, hi - 1] = True  # only its last row
    f = pack(masks)
    whole = make_col(ctx, corpus, "COSINE")
    cols = [make_col(ctx, corpus[a:b], "COSINE", base=a) for a, b in bounds(bases, n)]
    for fi, expect in ((0, [lo]), (1, [hi - 1]), (2, [])):
        qf = np.full(nq, fi, np.uint32)
        mid = shard_knn(cols[1], queries, k, f, qf, n)
        for q in range(nq):  # no padding row and no row of the next shard
            assert list(mid[0][q, : mid[2][q]]) == expect, (fi, q, mid[0][q, : mid[2][q]])
        parts = [mid if i == 1 else shard_knn(c, queries, k, f, qf, n) for i, c in enumerate(cols)]
        want = whole.knn(queries, k, filters=f, query_filter=qf)
        same(merge(ctx, parts, k), want)
        oracle_check(corpus, queries, "COSINE", k, masks, qf, want)
    # 6000 rows pass: direct on each of three shards, screened unsharded -- the same answers
    spread = np.zeros((2, n), bool)
    spread[0, np.linspace(0, n - 1, 6000).astype(np.int64)] = True
    spread[1] = True  # screened everywhere
    f = pack(spread)
    qf = np.zeros(nq, np.uint32)
    want = whole.knn(queries, k, filters=f, query_filter=qf)
    st = whole.stats()
    assert st["n_passes"] > 0 and st["screen_used"] != 3, st
    parts = []
    for c in cols:
        parts.append(shard_knn(c, queries, k, f, qf, n))
        st = c.stats()
        assert st["n_passes"] == 0 and st["screen_used"] == 3, st  # SDB_SCREEN_NONE_EXACT: no screen ran
    same(merge(ctx, parts, k), want)
    oracle_check(corpus, queries, "COSINE", k, spread, qf, want)
    # direct and screened queries in one batch; a zero query in each part (exact fallback: the repair round runs)
    queries[1] = 0.0
    queries[2] = 0.0
    qf = np.array([0, 0, 1, 1, 0, 1, 1, 0], np.uint32)
    want = whole.knn(queries, k, filters=f, query_filter=qf)
    parts = [shard_knn(c, queries, k, f, qf, n) for c in cols]
    same(merge(ctx, parts, k), want)
    oracle_check(corpus, queries, "COSINE", k, spread, qf, want)
    for (a, b), part in zip(bounds(bases, n), parts):
        oracle_check(corpus[a:b], queries, "COSINE", k, spread, qf, part, base=a)


# ---- 3. the repair ladder and the exact fallback read the sliced bitmap ----
def test_repair_round_under_an_unaligned_slice(ctx):
    rng = np.random.default_rng(77)
    n, dim, nq, k = 80000, 128, 320, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    center = rng.uniform(-1, 1, dim)
    corpus[1000:7000] = (center[None, :] + rng.normal(0, 2e-3, (6000, dim))).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    crowd = [5, 77, 130, 200, 201, 254]  # few enough (<= 2 + nq / 64 with the zero query) to be repaired alone
    for q in crowd:
        queries[q] = center + rng.normal(0, 1e-3, dim)
    queries[9] = 0.0  # exact fallback
    # every crowd query loses a different sixth of the cluster (near-duplicates beyond the first rung's lists remain)
    masks = np.ones((len(crowd) + 1, n), bool)
    for i in range(len(crowd)):
        masks[i + 1, 1000 + i * 1000 : 1000 + (i + 1) * 1000] = False
    qf = np.zeros(nq, np.uint32)
    for i, q in enumerate(crowd):
        qf[q] = i + 1
    f = pack(masks)
    lo = 1013  # unaligned: the cluster straddles the two shards
    cols = [make_col(ctx, corpus[a:b], "COSINE", base=a, screen="TC_INT8") for a, b in bounds([0, lo], n)]
    parts = [shard_knn(c, queries, k, f, qf, n) for c in cols]
    st = cols[1].stats()
    assert st["n_repaired"] > 0 and st["n_fallback"] >= 1, st
    check = crowd + [0, 9, 33, 319]
    oracle_check(corpus[lo:], queries, "COSINE", k, masks, qf, parts[1], base=lo, qs=check)
    oracle_check(corpus, queries, "COSINE", k, masks, qf, merge(ctx, parts, k), qs=check)
    for i, q in enumerate(crowd):
        r = parts[1][0][q].astype(np.int64)
        assert ((r >= 1000) & (r < 7000)).all() and not ((r - 1000) // 1000 == i).any(), (q, r)


# ---- 4. asynchrony ----
def test_tickets_mix_sharded_filtered_and_unfiltered(ctx):
    import torch
    rng = np.random.default_rng(31)
    lo, n_local, dim, nq, k = 1001, 20000, 48, 64, 10
    n = lo + n_local + 77  # the shard sits inside the global rows, unaligned at both ends
    corpus = rng.uniform(-1, 1, (n_local, dim)).astype(np.float32)
    col = make_col(ctx, corpus, "COSINE", base=lo)
    masks = np.stack([rng.random(n) < p for p in (0.3, 0.05, 0.002)])
    f = pack(masks)
    f_local = pack(masks[:, lo : lo + n_local])
    dev = torch.device("cuda", 0)
    df = torch.from_numpy(f.view(np.int32)).to(dev)
    qs = [np.ascontiguousarray(rng.uniform(-1, 1, (nq, dim))) for _ in range(4)]
    dq = torch.from_numpy(qs[2]).to(dev)
    qfs = [rng.integers(0, 3, nq).astype(np.uint32) for _ in range(4)]
    outs = [(np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32)) for _ in range(4)]
    douts = (torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
             torch.zeros(nq, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    p = lambda a: a.ctypes.data  # noqa: E731
    tickets = [
        col.sharded_submit_filtered_host(p(qs[0]), nq, k, p(f), 3, qfs[0], n, p(outs[0][0]), p(outs[0][1]),
                                         p(outs[0][2])),
        col.sharded_submit_host(p(qs[1]), nq, k, p(outs[1][0]), p(outs[1][1]), p(outs[1][2])),
        col.sharded_submit_filtered_device(dq.data_ptr(), nq, k, df.data_ptr(), 3, qfs[2], n, douts[0].data_ptr(),
                                           douts[1].data_ptr(), douts[2].data_ptr()),
        col.sharded_submit_host(p(qs[3]), nq, k, p(outs[3][0]), p(outs[3][1]), p(outs[3][2])),
    ]
    for i in (2, 0, 3, 1):
        col.sharded_wait(tickets[i])
    outs[2] = (douts[0].cpu().numpy().view(np.uint64), douts[1].cpu().numpy(), douts[2].cpu().numpy().view(np.uint32))
    for i in range(4):  # the blocking calls: the column's own rows, row_base added
        want = col.knn(qs[i], k, filters=f_local, query_filter=qfs[i]) if i % 2 == 0 else col.knn(qs[i], k)
        same(outs[i], want)
    oracle_check(corpus, qs[2], "COSINE", k, masks, qfs[2], outs[2], base=lo, qs=range(0, nq, 5))


def test_filtered_device_tickets_in_flight(ctx):
    import torch
    rng = np.random.default_rng(32)
    n, dim, nq, k = 30000 + 5, 64, 100, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    col = make_col(ctx, corpus, "EUCLIDEAN")
    dev = torch.device("cuda", 0)
    masks = [np.stack([rng.random(n) < p for p in dens]) for dens in ((0.5, 0.01), (0.1,), (1.0, 0.0002, 0.3), (0.05,))]
    fs = [pack(m) for m in masks]
    qs = [rng.uniform(-1, 1, (nq, dim)) for _ in range(4)]
    qfs = [rng.integers(0, m.shape[0], nq).astype(np.uint32) for m in masks]
    dq = [torch.from_numpy(q).to(dev) for q in qs]
    df = [torch.from_numpy(f.view(np.int32)).to(dev) for f in fs]
    outs = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
             torch.zeros(nq, dtype=torch.int32, device=dev)) for _ in range(4)]
    torch.cuda.synchronize()
    tickets = [col.submit_device_filtered(dq[i].data_ptr(), nq, k, df[i].data_ptr(), fs[i].shape[0], qfs[i], 500,
                                          outs[i][0].data_ptr(), outs[i][1].data_ptr(), outs[i][2].data_ptr())
               for i in range(4)]
    for i in (1, 3, 0, 2):
        col.wait(tickets[i])
    for i in range(4):
        got = (outs[i][0].cpu().numpy().view(np.uint64) - np.uint64(500), outs[i][1].cpu().numpy(),
               outs[i][2].cpu().numpy().view(np.uint32))
        want = col.knn(qs[i], k, filters=fs[i], query_filter=qfs[i])  # the blocking call, host bitmaps
        same(got, want)
        oracle_check(corpus, qs[i], "EUCLIDEAN", k, masks[i], qfs[i], got, qs=range(0, nq, 11))


# ---- 5. refusals ----
def test_refusals_and_ownership():
    from surrealdb_b200 import Context, SdbError
    from surrealdb_b200 import _lib as L
    live0 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live0[0]), C.byref(live0[1]))
    c2 = Context(0)  # its own context: everything this test allocates is released by the closes below
    rng = np.random.default_rng(41)
    lo, n_local, dim, nq, k = 33, 5000, 16, 3, 5
    n = lo + n_local
    corpus = rng.uniform(-1, 1, (n_local, dim)).astype(np.float32)
    col = make_col(c2, corpus, "COSINE", base=lo)
    q = np.ascontiguousarray(rng.uniform(-1, 1, (nq, dim)))
    masks = np.stack([rng.random(n) < 0.5, rng.random(n) < 0.5])
    f = pack(masks)
    qf = np.array([0, 1, 0], np.uint32)
    want = shard_knn(col, q, k, f, qf, n)
    oracle_check(corpus, q, "COSINE", k, masks, qf, want, base=lo)
    out = (np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32))
    # n_rows_total too small, no filter, a filter index out of range
    for n_filters, qf_bad, n_total in ((2, qf, n - 1), (0, qf, n), (2, np.array([0, 2, 1], np.uint32), n)):
        with pytest.raises(SdbError) as e:
            col.sharded_submit_filtered_host(q.ctypes.data, nq, k, f.ctypes.data, n_filters, qf_bad, n_total,
                                             out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data)
        assert e.value.status == L.SDB_EINVAL
        same(shard_knn(col, q, k, f, qf, n), want)  # the column still answers
    col.close()
    c2.close()
    live1 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live1[0]), C.byref(live1[1]))
    assert (live1[0].value, live1[1].value) == (live0[0].value, live0[1].value)


# ---- 6. two GPUs in one process ----
def test_two_gpus_knn_sharded_multi_filtered():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from surrealdb_b200 import Context
    from surrealdb_b200.engine import knn_sharded_multi
    rng = np.random.default_rng(51)
    n, dim, nq, k = 40000, 64, 33, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    queries[5] = 0.0
    ctxs = Context.create_multi([0, 1])
    bases = [0, 20003]
    shards = [make_col(c, corpus[a:b], "COSINE", base=a) for c, (a, b) in zip(ctxs, bounds(bases, n))]
    counts = [n, n // 3, 6000, 500]
    masks = np.zeros((len(counts), n), bool)
    for i, c in enumerate(counts):
        masks[i, rng.choice(n, c, replace=False)] = True
    qf = (np.arange(nq) % len(counts)).astype(np.uint32)
    res = knn_sharded_multi(shards, queries, k, filters=pack(masks), query_filter=qf)
    oracle_check(corpus, queries, "COSINE", k, masks, qf, res)
