"""`ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k` on row-sharded columns (sdb_corpus_order_sharded_*): several
shards on one device, each searched through the one-rank sharded call, their lists merged by sdb_order_merge_device
as after the exchange.  Every shard's list equals sdb_corpus_order_topk on that shard (global ids), and the merged
lists equal sdb_corpus_order_topk on the whole column byte for byte (rows, values, counts); spot checks against the
SortTopK reference over the CPU oracle (tests/sort_topk_ref.py).  Also: ties across shard boundaries, both merge
kernels in both directions against a numpy merge, the repair round of a DESC ranking, tickets mixed with sharded KNN,
refusals and ownership, and one process driving the shards (sdb_corpus_order_sharded_multi)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from sort_topk_ref import FN_IDS, row_values, sort_keyed

pytestmark = pytest.mark.gpu

KS = [1, 10, 256, 257, 1000, 4096]


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return np.ascontiguousarray(pack_row_filter(np.asarray(masks, bool)))


def make_col(ctx, rows, metric, base=None, screen=None, p=None):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if rows.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, rows.shape[1], metric, dt, capacity=max(1, rows.shape[0]))
    col.append(rows)
    col.finalize()
    if base is not None:
        col.set_row_base(base)
    if screen:
        col.set_screen(screen)
    if p is not None:
        col.set_minkowski_order(p)
    return col


def bounds(bases, n):
    return list(zip(bases, bases[1:] + [n]))


def shard_order(col, queries, k, fn, order, f=None, qf=None, n_total=0):
    """one rank: sdb_corpus_order_sharded_submit + sdb_knn_sharded_wait (the merge of one block is a copy)"""
    q = None if queries is None else np.ascontiguousarray(queries, np.float64)
    nq = 1 if q is None else q.shape[0]
    rows, vals, cnt = np.zeros((nq, max(k, 1)), np.uint64), np.zeros((nq, max(k, 1)), np.float64), np.zeros(nq, np.uint32)
    t = col.order_sharded_submit_host(0 if q is None else q.ctypes.data, nq, k, fn, order, rows.ctypes.data,
                                      vals.ctypes.data, cnt.ctypes.data, h_filters=0 if f is None else f.ctypes.data,
                                      n_filters=0 if f is None else f.shape[0], query_filter=qf, n_rows_total=n_total)
    col.sharded_wait(t)
    return rows[:, :k], vals[:, :k], cnt


def merge(ctx, parts, k, order):
    """the shards' lists merged in the ranking's direction with sdb_order_merge_device, as after the exchange"""
    import torch
    from surrealdb_b200.engine import order_merge_device
    dev = torch.device("cuda", ctx.device)
    nq = parts[0][2].size
    r = torch.from_numpy(np.stack([p[0] for p in parts]).view(np.int64)).to(dev)
    d = torch.from_numpy(np.stack([p[1] for p in parts])).to(dev)
    c = torch.from_numpy(np.stack([p[2] for p in parts]).view(np.int32)).to(dev)
    out = (torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
           torch.zeros(nq, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()  # torch's stream and the library's are not ordered with each other
    order_merge_device(ctx, len(parts), nq, k, order, r.data_ptr(), d.data_ptr(), c.data_ptr(), out[0].data_ptr(),
                       out[1].data_ptr(), out[2].data_ptr())
    return (out[0].cpu().numpy().view(np.uint64), out[1].cpu().numpy(), out[2].cpu().numpy().view(np.uint32))


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def same(a, b, k, qs=None):
    """equal results: counts, values bit for bit, rows in order (k <= 1000); above, where the reference sorts
    unstably, the rows of each group of equal values as sets"""
    ra, va, ca = a
    rb, vb, cb = b
    assert list(ca) == list(cb), (ca, cb)
    for q in range(len(ca)) if qs is None else qs:
        n = int(ca[q])
        assert _bits(va[q, :n]).tobytes() == _bits(vb[q, :n]).tobytes(), (q, va[q, :n], vb[q, :n])
        if k <= 1000:
            assert ra[q, :n].tobytes() == rb[q, :n].tobytes(), (q, ra[q, :n], rb[q, :n])
            continue
        bits = _bits(va[q, :n])
        j = 0
        while j < n:
            e = j
            while e < n and bits[e] == bits[j]:
                e += 1
            assert set(ra[q, j:e].tolist()) == set(rb[q, j:e].tolist()), (q, j, e)
            j = e


def oracle_check(res, vals, k, desc, passes, q, close=False):
    """query q of res against the SortTopK reference over the oracle's values (global rows); close: values to 1e-12
    relative (MINKOWSKI's pow())"""
    rows, got, cnt = res
    er, ev = sort_keyed(vals, k, desc, passes)
    assert int(cnt[q]) == er.size, (q, int(cnt[q]), er.size)
    if close:
        assert np.allclose(got[q, : er.size], ev, rtol=1e-12, atol=0, equal_nan=True), q
    else:
        assert _bits(got[q, : er.size]).tobytes() == _bits(ev).tobytes(), (q, got[q, : er.size], ev)
    same((rows[q : q + 1, : er.size], ev[None, :], cnt[q : q + 1]), (er[None, :], ev[None, :], cnt[q : q + 1]), k)


# ---- 1. every route, merged equals unsharded ------------------------------------------------------------------------
# (column metric, fn, order, screen, Minkowski order)
ROUTES = [(m, m, "ASC", None, None) for m in ("CHEBYSHEV", "COSINE", "EUCLIDEAN", "HAMMING", "JACCARD", "MANHATTAN",
                                               "MINKOWSKI", "PEARSON")] + [
    ("COSINE", "SIMILARITY_COSINE", "DESC", "TC_INT8", None),
    ("COSINE", "SIMILARITY_COSINE", "DESC", "TC_BF16", None),
    ("PEARSON", "PEARSON", "DESC", None, None),
    ("COSINE", "DOT", "ASC", None, None),
    ("COSINE", "DOT", "DESC", None, None),
    ("EUCLIDEAN", "DOT", "ASC", None, None),
    ("EUCLIDEAN", "DOT", "DESC", None, None),
    ("COSINE", "COSINE", "DESC", None, None),
    ("EUCLIDEAN", "COSINE", "DESC", None, None),
    ("COSINE", "SIMILARITY_COSINE", "ASC", None, None),
    ("EUCLIDEAN", "SIMILARITY_COSINE", "ASC", None, None),
    ("COSINE", "EUCLIDEAN", "ASC", None, None),
    ("COSINE", "EUCLIDEAN", "DESC", None, None),
    ("EUCLIDEAN", "EUCLIDEAN", "DESC", None, None),
    ("HAMMING", "HAMMING", "DESC", None, None),
    ("JACCARD", "JACCARD", "DESC", None, None),
    ("MANHATTAN", "MANHATTAN", "DESC", None, None),
    ("MINKOWSKI", "MINKOWSKI", "ASC", None, 2.5),
    ("MINKOWSKI", "MINKOWSKI", "DESC", None, 2.5),
    ("COSINE", "MAGNITUDE", "ASC", None, None),
    ("COSINE", "MAGNITUDE", "DESC", None, None),
]


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric,fn,order,screen,p", ROUTES)
def test_every_route_merges_to_the_unsharded_call(ctx, dtype, metric, fn, order, screen, p):
    from surrealdb_b200.sharding import shard_range
    rng = np.random.default_rng(zlib.crc32(f"{dtype}{metric}{fn}{order}{screen}{p}".encode()))
    n, dim = 9000 + 37, 24
    nq = 1 if fn == "MAGNITUDE" else 12
    npdt = np.float32 if dtype == "F32" else np.float64
    if metric in ("HAMMING", "JACCARD"):  # repeated values: the counts see ties
        corpus = rng.integers(-3, 4, (n, dim)).astype(npdt)
        queries = rng.integers(-3, 4, (nq, dim)).astype(np.float64)
    else:
        corpus = rng.uniform(-1, 1, (n, dim)).astype(npdt)
        queries = rng.uniform(-1, 1, (nq, dim))
    if fn == "MAGNITUDE":
        queries = None
    counts = [n, n // 2, n // 10, 90, 5000, 3]  # 5000 and 90: screened unsharded, direct on some shards
    masks = np.zeros((len(counts), n), bool)
    for i, c in enumerate(counts):
        masks[i, rng.choice(n, c, replace=False)] = True
    f = pack(masks)
    qf = (np.arange(nq) % len(counts)).astype(np.uint32)
    whole = make_col(ctx, corpus, metric, screen=screen, p=p)
    want = {}
    for k in KS:
        want[k, False] = whole.order_topk(queries, k, fn, order)
        want[k, True] = whole.order_topk(queries, k, fn, order, filters=f, query_filter=qf)
    # spot checks against the SortTopK reference over the oracle's values
    code, pp = FN_IDS[fn], 3.0 if p is None else p
    for q in (0, nq - 1):
        vals = row_values(code, corpus, None if queries is None else queries[q], minkowski_p=pp)
        for k in KS:
            oracle_check(want[k, False], vals, k, order == "DESC", None, q, close=fn == "MINKOWSKI")
            oracle_check(want[k, True], vals, k, order == "DESC", masks[qf[q]], q, close=fn == "MINKOWSKI")
    aligned = [shard_range(n, 3, r)[0] for r in range(3)]
    for bases in (aligned, [0, 31, 33, 5003]):
        parts = {key: [] for key in want}
        for lo, hi in bounds(bases, n):
            col = make_col(ctx, corpus[lo:hi], metric, base=lo, screen=screen, p=p)
            f_local = pack(masks[:, lo:hi])
            for k in KS:
                part = shard_order(col, queries, k, fn, order)
                same(part, col.order_topk(queries, k, fn, order), k)  # the shard's own call, global ids
                parts[k, False].append(part)
                part = shard_order(col, queries, k, fn, order, f, qf, n)
                same(part, col.order_topk(queries, k, fn, order, filters=f_local, query_filter=qf), k)
                parts[k, True].append(part)
            col.close()
        for (k, filtered), ps in parts.items():
            same(merge(ctx, ps, k, order), want[k, filtered], k)


# ---- 2. ties across shard boundaries: duplicate rows in different shards, +-0.0, NaNs of both signs ---------------
TINY = float(np.float32(-1.4e-45))  # the smallest negative f32 subnormal: exact in F32 and F64 columns
C_TINY = 3.6e-279  # TINY * C_TINY is a negative f64 subnormal, which a norm of 16 divides to -0.0


def tie_corpus(rng, m, dtype):
    """m base rows repeated three times (row i, i + m and i + 2m are equal).  Against q = [C_TINY, 1, 0, 0]: rows
    orthogonal to q (similarity +0.0), rows whose similarity underflows to -0.0, zero rows (similarity NaN of the
    negative sign), rows with a NaN (the positive sign) and a few rows on either side of zero."""
    x = np.zeros((m, 4))
    x[:, 2:] = rng.integers(1, 3, (m, 2))  # similarity +0.0
    kind = rng.permutation(m)
    x[kind[:20]] = 0.0
    x[kind[20:30], 0] = np.nan
    x[kind[30:60], 1] = 1.0
    x[kind[60:90], 1] = -1.0
    x[kind[90:130]] = [TINY, 0.0, 16.0, 0.0]  # similarity -0.0
    return np.concatenate([x, x, x]).astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_ties_across_shard_boundaries(ctx, dtype):
    rng = np.random.default_rng(17)
    m = 700
    x = tie_corpus(rng, m, dtype)
    n = x.shape[0]
    bases = [0, m - 7, 2 * m + 5]  # every copy straddles a boundary
    queries = np.array([[C_TINY, 1.0, 0.0, 0.0], [-C_TINY, -1.0, 0.0, 0.0], [1.0, -1.0, 0.0, 2.0]])
    routes = [("COSINE", "SIMILARITY_COSINE", "ASC"), ("COSINE", "SIMILARITY_COSINE", "DESC"),
              ("EUCLIDEAN", "SIMILARITY_COSINE", "DESC"), ("COSINE", "DOT", "ASC"), ("COSINE", "DOT", "DESC"),
              ("EUCLIDEAN", "EUCLIDEAN", "DESC"), ("MANHATTAN", "MANHATTAN", "DESC"), ("COSINE", "COSINE", "DESC")]
    neg_zero, nan_signs = 0, set()
    for metric, fn, order in routes:
        whole = make_col(ctx, x, metric)
        cols = [make_col(ctx, x[a:b], metric, base=a) for a, b in bounds(bases, n)]
        vals = [row_values(FN_IDS[fn], x, q) for q in queries]
        for k in (1, 10, 37, 256, 1000):
            want = whole.order_topk(queries, k, fn, order)
            got = merge(ctx, [shard_order(c, queries, k, fn, order) for c in cols], k, order)
            same(got, want, k)
            for q in range(queries.shape[0]):
                oracle_check(got, vals[q], k, order == "DESC", None, q)
                b = _bits(got[1][q, : got[2][q]])
                neg_zero += int((b == np.uint64(1 << 63)).sum())
                nan_signs |= {int(v >> np.uint64(63)) for v, d in zip(b, got[1][q, : got[2][q]]) if d != d}
        for c in cols:
            c.close()
        whole.close()
    assert neg_zero > 0 and nan_signs == {0, 1}  # -0.0 and NaNs of both signs came through the merge


# ---- 3. both merge kernels in both directions against a numpy merge -----------------------------------------------
ALL_ONES_NAN = np.uint64(0xFFFFFFFFFFFFFFFF).view(np.float64)
POOL = np.array([ALL_ONES_NAN, np.uint64(0xFFF8000000000000).view(np.float64), -np.inf, -2.5, -1.0, -0.0, 0.0, 5e-324,
                 1.0, 2.5, np.inf, np.uint64(0x7FF8000000000000).view(np.float64)])


def cmp_key(v, desc):
    """Number::cmp's total order (-0.0 == 0.0) as uint64 keys, reversed as a whole for DESC"""
    from select_ref import num_key as keys
    kk = keys(v)
    return ~kk if desc else kk


def make_lists(rng, n_lists, nq, k, desc):
    dist = POOL[rng.integers(0, POOL.size, (n_lists, nq, k))]
    rows = np.empty((n_lists, nq, k), np.uint64)
    for q in range(nq):  # disjoint shards: a row appears in one list only
        rows[:, q, :] = rng.permutation(4 * n_lists * k)[: n_lists * k].reshape(n_lists, k)
    o = np.argsort(rows, axis=-1, kind="stable")  # each list in (key, row) order for its direction
    rows, dist = np.take_along_axis(rows, o, -1), np.take_along_axis(dist, o, -1)
    o = np.argsort(cmp_key(dist.ravel(), desc).reshape(dist.shape), axis=-1, kind="stable")
    rows, dist = np.take_along_axis(rows, o, -1), np.take_along_axis(dist, o, -1)
    kind = rng.integers(0, 4, (n_lists, nq))  # empty, short, exactly k, above k
    counts = np.where(kind == 0, 0, np.where(kind == 1, rng.integers(0, k + 1, (n_lists, nq)),
                                             np.where(kind == 2, k, k + rng.integers(1, 5, (n_lists, nq)))))
    counts[:, 0] = rng.integers(0, 2, n_lists)  # fewer than k entries in all, or none
    if nq > 1:
        counts[:, 1] = 0
    return rows, dist, counts.astype(np.uint32)


def numpy_merge(rows, dist, counts, k, desc):
    """per query: [(row, value)] of the first min(count, k) entries of every list, by (key, row), the first k"""
    n_lists, nq = counts.shape
    out = []
    for q in range(nq):
        take = np.arange(k)[None, :] < np.minimum(counts[:, q], k)[:, None]
        r, d = rows[:, q, :][take], dist[:, q, :][take]
        o = np.lexsort((r, cmp_key(d, desc)))[:k]
        out.append(list(zip(r[o].tolist(), d[o])))
    return out


def run_merge(ctx, rows, dist, counts, k, order):
    """order None: sdb_topk_merge_device; "ASC" / "DESC": sdb_order_merge_device"""
    import torch
    from surrealdb_b200.engine import order_merge_device, topk_merge_device
    n_lists, nq = counts.shape
    dev = torch.device("cuda", 0)
    tr = torch.from_numpy(rows.view(np.int64).copy()).to(dev)
    td = torch.from_numpy(dist.copy()).to(dev)
    tc = torch.from_numpy(counts.view(np.int32).copy()).to(dev)
    o = (torch.full((nq, k), -1, dtype=torch.int64, device=dev), torch.full((nq, k), -7.0, dtype=torch.float64, device=dev),
         torch.full((nq,), -1, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    args = (tr.data_ptr(), td.data_ptr(), tc.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr())
    if order is None:
        topk_merge_device(ctx, n_lists, nq, k, *args)
    else:
        order_merge_device(ctx, n_lists, nq, k, order, *args)
    return o[0].cpu().numpy().view(np.uint64), o[1].cpu().numpy(), o[2].cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("k", [1, 7, 100, 256])
@pytest.mark.parametrize("n_lists", [2, 5, 31, 32, 33, 64])
@pytest.mark.parametrize("order", ["ASC", "DESC"])
def test_merge_kernels_both_directions(ctx, order, n_lists, k):
    from surrealdb_b200._lib import SDB_EUNSUPPORTED, SdbError
    desc = order == "DESC"
    rng = np.random.default_rng(zlib.crc32(f"{order}{n_lists}{k}".encode()))
    for nq in (1, 5, 37):
        rows, dist, counts = make_lists(rng, n_lists, nq, k, desc)
        if n_lists > 32 and n_lists * k > 8192:  # the sorter's 200 KB of shared memory
            with pytest.raises(SdbError) as e:
                run_merge(ctx, rows, dist, counts, k, order)
            assert e.value.status == SDB_EUNSUPPORTED
            continue
        want = numpy_merge(rows, dist, counts, k, desc)
        got_rows, got_dist, got_cnt = run_merge(ctx, rows, dist, counts, k, order)
        assert got_cnt.tolist() == [len(w) for w in want]
        for q in range(nq):
            c = len(want[q])
            assert got_rows[q, :c].tolist() == [e[0] for e in want[q]], (q, got_rows[q, :c])
            assert _bits(got_dist[q, :c]).tolist() == _bits([e[1] for e in want[q]]).tolist(), q
        if not desc:  # ASC is the KNN merge: sdb_topk_merge_device returns the same, byte for byte
            old = run_merge(ctx, rows, dist, counts, k, None)
            for a, b in zip(old, (got_rows, got_dist, got_cnt)):
                assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("order", ["ASC", "DESC"])
def test_warp_merge_at_k_4096(ctx, order):
    rng = np.random.default_rng(4096 + (order == "DESC"))
    k, nq = 4096, 3
    rows, dist, counts = make_lists(rng, 2, nq, k, order == "DESC")
    want = numpy_merge(rows, dist, counts, k, order == "DESC")
    got_rows, got_dist, got_cnt = run_merge(ctx, rows, dist, counts, k, order)
    for q in range(nq):
        c = len(want[q])
        assert int(got_cnt[q]) == c
        assert got_rows[q, :c].tolist() == [e[0] for e in want[q]]
        assert _bits(got_dist[q, :c]).tolist() == _bits([e[1] for e in want[q]]).tolist()


# ---- 4. the repair round of a DESC ranking ----------------------------------------------------------------------
def test_repair_round_in_a_desc_ranking(ctx):
    rng = np.random.default_rng(77)
    n, dim, nq, k = 80000, 128, 320, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    center = rng.uniform(-1, 1, dim)
    corpus[1000:7000] = (center[None, :] + rng.normal(0, 2e-3, (6000, dim))).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    crowd = [5, 77, 130, 200, 201, 254]
    for q in crowd:
        queries[q] = center + rng.normal(0, 1e-3, dim)
    queries[9] = 0.0  # exact fallback
    masks = np.ones((len(crowd) + 1, n), bool)  # every crowd query loses a different sixth of the cluster
    for i in range(len(crowd)):
        masks[i + 1, 1000 + i * 1000 : 1000 + (i + 1) * 1000] = False
    qf = np.zeros(nq, np.uint32)
    for i, q in enumerate(crowd):
        qf[q] = i + 1
    f = pack(masks)
    lo = 1013  # unaligned: the cluster straddles the two shards
    cols = [make_col(ctx, corpus[a:b], "COSINE", base=a, screen="TC_INT8") for a, b in bounds([0, lo], n)]
    parts = [shard_order(c, queries, k, "SIMILARITY_COSINE", "DESC", f, qf, n) for c in cols]
    st = cols[1].stats()
    assert st["n_repaired"] > 0 and st["n_fallback"] >= 1, st
    whole = make_col(ctx, corpus, "COSINE", screen="TC_INT8")
    want = whole.order_topk(queries, k, "SIMILARITY_COSINE", "DESC", filters=f, query_filter=qf)
    same(merge(ctx, parts, k, "DESC"), want, k)
    for q in crowd:
        vals = row_values(16, corpus[:8000], queries[q])
        passes = masks[qf[q], :8000]
        er, ev = sort_keyed(vals, k, True, passes)
        assert want[0][q].tolist() == er.tolist() and _bits(want[1][q]).tolist() == _bits(ev).tolist(), q


# ---- 5. tickets: sharded order and KNN tickets in flight together -------------------------------------------------
def test_tickets_mix_sharded_order_and_knn(ctx):
    import torch
    from surrealdb_b200 import SdbError
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
    p = lambda a: a.ctypes.data  # noqa: E731
    kinds = [("SIMILARITY_COSINE", "DESC", True, False), None, ("DOT", "ASC", False, True),
             ("EUCLIDEAN", "DESC", True, True), ("COSINE", "DESC", False, False), "filtered",
             ("SIMILARITY_COSINE", "DESC", False, True), ("MANHATTAN", "ASC", True, False)]
    for rnd in range(2):
        ks = kinds[4 * rnd : 4 * rnd + 4]
        qs = [np.ascontiguousarray(rng.uniform(-1, 1, (nq, dim))) for _ in range(4)]
        qfs = [rng.integers(0, 3, nq).astype(np.uint32) for _ in range(4)]
        outs = [(np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32)) for _ in range(4)]
        douts = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64,
                  device=dev), torch.zeros(nq, dtype=torch.int32, device=dev)) for _ in range(4)]
        dqs = [torch.from_numpy(q).to(dev) for q in qs]
        torch.cuda.synchronize()
        tickets = []
        for i, kind in enumerate(ks):
            if kind is None:
                t = col.sharded_submit_host(p(qs[i]), nq, k, p(outs[i][0]), p(outs[i][1]), p(outs[i][2]))
            elif kind == "filtered":
                t = col.sharded_submit_filtered_host(p(qs[i]), nq, k, p(f), 3, qfs[i], n, p(outs[i][0]),
                                                     p(outs[i][1]), p(outs[i][2]))
            else:
                fn, order, host, filtered = kind
                if host:
                    t = col.order_sharded_submit_host(p(qs[i]), nq, k, fn, order, p(outs[i][0]), p(outs[i][1]),
                                                      p(outs[i][2]), h_filters=p(f) if filtered else 0,
                                                      n_filters=3 if filtered else 0,
                                                      query_filter=qfs[i] if filtered else None,
                                                      n_rows_total=n if filtered else 0)
                else:
                    t = col.order_sharded_submit_device(dqs[i].data_ptr(), nq, k, fn, order, douts[i][0].data_ptr(),
                                                        douts[i][1].data_ptr(), douts[i][2].data_ptr(),
                                                        d_filters=df.data_ptr() if filtered else 0,
                                                        n_filters=3 if filtered else 0,
                                                        query_filter=qfs[i] if filtered else None,
                                                        n_rows_total=n if filtered else 0)
            tickets.append(t)
        with pytest.raises(SdbError):  # a fifth batch finds no free slot
            col.order_sharded_submit_host(p(qs[0]), nq, k, "DOT", "DESC", p(outs[0][0]), p(outs[0][1]), p(outs[0][2]))
        for i in rng.permutation(4):
            col.sharded_wait(tickets[int(i)])
        for i, kind in enumerate(ks):
            if kind is None:
                want, got = col.knn(qs[i], k), outs[i]
            elif kind == "filtered":
                want, got = col.knn(qs[i], k, filters=f_local, query_filter=qfs[i]), outs[i]
            else:
                fn, order, host, filtered = kind
                want = col.order_topk(qs[i], k, fn, order, filters=f_local if filtered else None,
                                      query_filter=qfs[i] if filtered else None)
                got = outs[i] if host else (douts[i][0].cpu().numpy().view(np.uint64), douts[i][1].cpu().numpy(),
                                            douts[i][2].cpu().numpy().view(np.uint32))
            for a, b in zip(got, want):
                assert a.tobytes() == b.tobytes(), (rnd, i, kind)


# ---- 6. refusals and ownership ------------------------------------------------------------------------------------
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
    want = shard_order(col, q, k, "SIMILARITY_COSINE", "DESC", f, qf, n)
    same(want, col.order_topk(q, k, "SIMILARITY_COSINE", "DESC", filters=pack(masks[:, lo:]), query_filter=qf), k)
    out = (np.zeros((nq, 4097), np.uint64), np.zeros((nq, 4097), np.float64), np.zeros(nq, np.uint32))
    o = (out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data)
    # unknown fn, unknown order, k = 4097, NULL queries for a function that takes one, n_rows_total too small
    for qp, fn, order, kk, n_total, status in ((q.ctypes.data, 99, "DESC", k, n, L.SDB_EINVAL),
                                               (q.ctypes.data, "DOT", 2, k, n, L.SDB_EINVAL),
                                               (q.ctypes.data, "DOT", "DESC", 4097, n, L.SDB_EUNSUPPORTED),
                                               (0, "DOT", "DESC", k, n, L.SDB_EINVAL),
                                               (q.ctypes.data, "DOT", "DESC", k, n - 1, L.SDB_EINVAL)):
        with pytest.raises(SdbError) as e:
            col.order_sharded_submit_host(qp, nq, kk, fn, order, *o, h_filters=f.ctypes.data, n_filters=2,
                                          query_filter=qf, n_rows_total=n_total)
        assert e.value.status == status
        same(shard_order(col, q, k, "SIMILARITY_COSINE", "DESC", f, qf, n), want, k)  # the column still answers
    # no ticket stayed claimed: four tickets fit
    outs = [(np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32)) for _ in range(4)]
    ts = [col.order_sharded_submit_host(q.ctypes.data, nq, k, "SIMILARITY_COSINE", "DESC", *(a.ctypes.data for a in b),
                                        h_filters=f.ctypes.data, n_filters=2, query_filter=qf, n_rows_total=n)
          for b in outs]
    for t in ts:
        col.sharded_wait(t)
    for b in outs:
        same(b, want, k)
    # the merge entry point refuses what the order calls refuse
    with pytest.raises(SdbError) as e:
        from surrealdb_b200.engine import order_merge_device
        order_merge_device(c2, 2, 1, 4097, "DESC", 8, 8, 8, 8, 8, 8)
    assert e.value.status == L.SDB_EUNSUPPORTED
    assert L.lib().sdb_order_merge_device(c2.h, 2, 1, 5, 7, 8, 8, 8, 0, 0, 0, 8, 8, 8) == L.SDB_EINVAL
    col.close()
    c2.close()
    live1 = (C.c_uint64(), C.c_uint64())
    L.lib().sdb_debug_live_allocations(C.byref(live1[0]), C.byref(live1[1]))
    assert (live1[0].value, live1[1].value) == (live0[0].value, live0[1].value)


# ---- 7. one process driving the shards ----------------------------------------------------------------------------
def test_order_sharded_multi_one_shard(ctx):
    """sdb_corpus_order_sharded_multi over a single shard: the driver of one process, on one GPU"""
    from surrealdb_b200.engine import order_sharded_multi
    rng = np.random.default_rng(61)
    n, dim, nq = 7000, 32, 9
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    col = make_col(ctx, corpus, "EUCLIDEAN")
    masks = np.stack([rng.random(n) < 0.4, rng.random(n) < 0.01])
    qf = (np.arange(nq) % 2).astype(np.uint32)
    for fn, order, k in (("EUCLIDEAN", "DESC", 10), ("DOT", "DESC", 256), ("SIMILARITY_COSINE", "ASC", 1000)):
        same(order_sharded_multi([col], queries, k, fn, order), col.order_topk(queries, k, fn, order), k)
        same(order_sharded_multi([col], queries, k, fn, order, filters=pack(masks), query_filter=qf),
             col.order_topk(queries, k, fn, order, filters=pack(masks), query_filter=qf), k)
    same(order_sharded_multi([col], None, 20, "MAGNITUDE", "DESC"), col.order_topk(None, 20, "MAGNITUDE", "DESC"), 20)


def test_two_gpus_order_sharded_multi():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from surrealdb_b200 import Context
    from surrealdb_b200.engine import order_sharded_multi
    rng = np.random.default_rng(51)
    n, dim, nq = 40000, 64, 33
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = rng.uniform(-1, 1, (nq, dim))
    queries[5] = 0.0
    ctxs = Context.create_multi([0, 1])
    bases = [0, 20003]
    shards = [make_col(c, corpus[a:b], "COSINE", base=a) for c, (a, b) in zip(ctxs, bounds(bases, n))]
    whole = make_col(ctxs[0], corpus, "COSINE")
    masks = np.stack([rng.random(n) < 0.5, rng.random(n) < 0.01])
    qf = (np.arange(nq) % 2).astype(np.uint32)
    for fn, order, k in (("SIMILARITY_COSINE", "DESC", 10), ("DOT", "ASC", 256), ("EUCLIDEAN", "DESC", 1000)):
        same(order_sharded_multi(shards, queries, k, fn, order), whole.order_topk(queries, k, fn, order), k)
        same(order_sharded_multi(shards, queries, k, fn, order, filters=pack(masks), query_filter=qf),
             whole.order_topk(queries, k, fn, order, filters=pack(masks), query_filter=qf), k)
