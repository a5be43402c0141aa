"""Brute-force KNN of HAMMING and JACCARD columns through the count path (count_pass in count.cu, then cand_final):
exact counts of every row, ranked per row range.  Every answer is compared bit for bit (rows, their order, f64
distances, counts) with the CPU oracle and with the same column under NONE_EXACT, the exact kernel."""
import zlib

import numpy as np
import pytest

import count_rank_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SIMT_F32, NONE_EXACT = 1, 3


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_col(ctx, corpus, skip=None, screen=None, metric="HAMMING"):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if corpus.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, corpus.shape[1], metric, dt, capacity=max(1, corpus.shape[0]))
    col.append(corpus)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if screen:
        col.set_screen(screen)
    return col


def sample(nq):
    return sorted(set(list(range(0, nq, max(1, nq // 16))) + [nq - 1]))


def check_oracle(corpus, queries, k, rows, dist, cnt, qs=None, skip=None, metric="HAMMING"):
    for q in range(queries.shape[0]) if qs is None else qs:
        r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=skip)
        assert cnt[q] == r.size, (q, int(cnt[q]), r.size)
        assert rows[q, : cnt[q]].tolist() == r.tolist(), (q, rows[q, : cnt[q]], r)
        assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, dist[q, : cnt[q]], d)


def counted_and_exact(col, queries, k, **kw):
    """The count path's answer (an explicit SIMT_F32 request: AUTO ranks a single query with the exact kernel),
    checked against the exact kernel's on the same column; returns it and its stats."""
    col.set_screen("SIMT_F32")
    rows, dist, cnt = col.knn(queries, k, **kw)
    st = col.stats()
    col.set_screen("NONE_EXACT")
    r2, d2, c2 = col.knn(queries, k, **kw)
    col.set_screen("AUTO")
    assert cnt.tolist() == c2.tolist()
    for q in range(queries.shape[0]):
        assert rows[q, : cnt[q]].tolist() == r2[q, : cnt[q]].tolist(), q
        assert dist[q, : cnt[q]].tobytes() == d2[q, : cnt[q]].tobytes(), q
    return rows, dist, cnt, st


def assert_counted(st, nq):
    assert st["screen_used"] == SIMT_F32 and st["n_passes"] == 1, st
    assert st["n_fallback"] == 0 and st["n_special_rows"] == 0, st


def gen(rng, kind, n, dim, fdt):
    if kind == "alphabet":
        return rng.integers(-3, 4, (n, dim)).astype(fdt), rng.integers(-3, 4, (64, dim)).astype(np.float64)
    if kind == "binary":
        return rng.integers(0, 2, (n, dim)).astype(fdt), rng.integers(0, 2, (64, dim)).astype(np.float64)
    return rng.uniform(-1, 1, (n, dim)).astype(fdt), rng.uniform(-1, 1, (64, dim))  # every distance is dim: all tied


# ---- 1. parity matrix ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 5, 33, 127, 768, 1100, 4097])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("kind", ["alphabet", "binary", "uniform"])
def test_parity_matrix(ctx, kind, dtype, dim):
    rng = np.random.default_rng(zlib.crc32(f"{kind}{dtype}{dim}".encode()))
    n = 3000 + 77 if dim <= 1100 else 700 + 3  # not a multiple of the 128-row step
    fdt = np.float32 if dtype == "F32" else np.float64
    corpus, queries = gen(rng, kind, n, dim, fdt)
    corpus[500:520] = corpus[10]  # duplicates on both sides of range boundaries
    corpus[n // 2 - 3: n // 2 + 3] = corpus[11]
    col = make_col(ctx, corpus)
    for nq in (1, 3, 64):
        for k in (1, 10, 100, 256):
            rows, dist, cnt, st = counted_and_exact(col, queries[:nq], k)
            assert_counted(st, nq)
            check_oracle(corpus, queries[:nq], k, rows, dist, cnt, qs=sample(nq))
    col.knn(queries[:1], 10)  # one query under AUTO: the exact kernel
    assert col.stats()["screen_used"] == NONE_EXACT and col.stats()["n_fallback"] == 1
    rows, dist, cnt = col.knn(queries[:3], 300)  # k > 256: the exact kernel
    assert col.stats()["n_fallback"] == 3
    check_oracle(corpus, queries[:3], 300, rows, dist, cnt)


def test_many_queries_and_small_corpora(ctx):
    rng = np.random.default_rng(1025)
    corpus, _ = gen(rng, "binary", 20000 + 5, 64, np.float32)
    queries = rng.integers(0, 2, (1025, 64)).astype(np.float64)
    col = make_col(ctx, corpus)
    for k in (10, 256):
        rows, dist, cnt, st = counted_and_exact(col, queries, k)
        assert_counted(st, 1025)
        check_oracle(corpus, queries, k, rows, dist, cnt, qs=sample(1025))
    for n in (1, 5, 130):  # fewer rows than ranges, fewer rows than k
        small = corpus[:n].copy()
        col = make_col(ctx, small)
        for k in (0, 1, 10, 256):
            rows, dist, cnt = col.knn(queries[:3], k)
            assert cnt.tolist() == [min(k, n)] * 3
            if k:
                assert_counted(col.stats(), 3)
                check_oracle(small, queries[:3], k, rows, dist, cnt)


@pytest.mark.parametrize("dim", [1, 5, 33, 127, 768])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("kind", ["alphabet", "binary", "uniform"])
def test_jaccard_parity(ctx, kind, dtype, dim):
    rng = np.random.default_rng(zlib.crc32(f"jac{kind}{dtype}{dim}".encode()))
    n = 2000 + 77
    fdt = np.float32 if dtype == "F32" else np.float64
    corpus, queries = gen(rng, kind, n, dim, fdt)
    corpus[500:520] = corpus[10]
    corpus[n // 2 - 3: n // 2 + 3] = corpus[11]
    if dim >= 5:
        corpus[7, :3] = [np.nan, -0.0, np.inf]
        queries[1, :3] = [np.nan, 0.0, -np.inf]
    col = make_col(ctx, corpus, metric="JACCARD")
    for nq in (1, 3, 64):
        for k in (1, 10, 100, 256):
            if nq == 64 and dim == 768 and k != 10:
                continue
            rows, dist, cnt, st = counted_and_exact(col, queries[:nq], k)
            assert_counted(st, nq)
            check_oracle(corpus, queries[:nq], k, rows, dist, cnt, qs=sample(nq), metric="JACCARD")
    col.knn(queries[:1], 10)  # one query under AUTO: counted too (the exact kernel is O(D^2) per row)
    assert_counted(col.stats(), 1)
    rows, dist, cnt = col.knn(queries[:2], 300)  # k > 256: the exact kernel
    assert col.stats()["n_fallback"] == 2
    check_oracle(corpus, queries[:2], 300, rows, dist, cnt, metric="JACCARD")


@pytest.mark.parametrize("metric", ["HAMMING", "JACCARD"])
def test_multi_step_ranges(ctx, metric):
    # many 128-row steps per range at small k: lists stay full across steps, and ranges meet inside the corpus
    rng = np.random.default_rng(zlib.crc32(f"steps{metric}".encode()))
    n, dim = 300_000 + 17, 16
    corpus = rng.integers(0, 4, (n, dim)).astype(np.float32)
    corpus[n // 3 - 2: n // 3 + 2] = corpus[5]  # duplicates across a likely range boundary
    queries = rng.integers(0, 4, (1025, dim)).astype(np.float64)
    col = make_col(ctx, corpus, metric=metric)
    for nq in (64, 1025):
        rows, dist, cnt, st = counted_and_exact(col, queries[:nq], 10) if nq == 64 else \
            (*col.knn(queries[:nq], 10), col.stats())
        assert_counted(st, nq)
        check_oracle(corpus, queries[:nq], 10, rows, dist, cnt, qs=sample(nq)[:8], metric=metric)


# ---- 2. values: signed zeros, infinities, subnormals, NaN payloads ---------------------------------------------------------
@pytest.mark.parametrize("metric", ["HAMMING", "JACCARD"])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_special_values(ctx, dtype, metric):
    rng = np.random.default_rng(zlib.crc32(f"values{dtype}".encode()))
    fdt = np.float32 if dtype == "F32" else np.float64
    n, dim = 4000 + 9, 24
    sub = np.finfo(fdt).smallest_subnormal
    alphabet = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, sub, -sub, 3 * sub, np.nan], fdt)
    corpus = alphabet[rng.integers(0, alphabet.size, (n, dim))]
    queries = alphabet[rng.integers(0, alphabet.size, (8, dim))].astype(np.float64)
    queries[0] = 0.0                # all zero
    queries[1] = np.nan             # all NaN
    queries[2, :3] = [np.inf, -np.inf, -0.0]
    queries[3, 0] = 0.1             # (F32 rows) an f64 element no f32 widens to: it matches nothing
    queries[3, 1] = 1e300
    queries[3, 2] = 1e-320
    col = make_col(ctx, corpus, metric=metric)
    for k in (1, 10, 256):
        rows, dist, cnt, st = counted_and_exact(col, queries, k)
        assert_counted(st, 8)
        check_oracle(corpus, queries, k, rows, dist, cnt, metric=metric)


@pytest.mark.parametrize("metric", ["HAMMING", "JACCARD"])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_nan_payloads_against_the_exact_kernel(ctx, dtype, metric):
    # non-canonical and negative NaN payloads: a row NaN matches a query NaN exactly when the device widens it to the
    # same bits (R.nan_patterns), which the exact kernel defines
    rng = np.random.default_rng(zlib.crc32(f"nan{dtype}".encode()))
    fdt = np.float32 if dtype == "F32" else np.float64
    pats = R.nan_patterns(fdt)
    n, dim = 3000, 16
    corpus = pats[rng.integers(0, pats.size, (n, dim))]
    corpus[::7, 0] = 1.0
    q32 = pats[rng.integers(0, pats.size, (6, dim))]
    queries = q32.astype(np.float64)  # the host's widening: payload kept, quiet bit set
    queries[5] = R.f64_nans()[rng.integers(0, 4, dim)]  # f64 payloads, some with no f32 preimage
    col = make_col(ctx, corpus, metric=metric)
    for k in (1, 10, 100):
        _, _, _, st = counted_and_exact(col, queries, k)
        assert_counted(st, 6)


# ---- 3. skip masks and removed rows -------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["HAMMING", "JACCARD"])
def test_skip_and_remove(ctx, metric):
    rng = np.random.default_rng(5)
    n, dim = 9000, 40
    corpus = rng.integers(0, 3, (n, dim)).astype(np.float32)
    queries = rng.integers(0, 3, (8, dim)).astype(np.float64)
    skip = (rng.random(n) < 0.2).astype(np.uint8)
    dead = np.unique(rng.integers(0, n, 200)).astype(np.uint64)
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, dim, metric, "F32", capacity=n)
    col.append(corpus)
    col.set_skip(skip)
    col.remove(dead[:100])
    col.finalize()
    col.remove(dead[100:])
    eff = skip.copy()
    eff[dead.astype(np.int64)] = 1
    rows, dist, cnt, st = counted_and_exact(col, queries, 10)
    assert_counted(st, 8)
    check_oracle(corpus, queries, 10, rows, dist, cnt, skip=eff, metric=metric)
    col.set_skip(np.ones(n, np.uint8))  # everything skipped
    col.finalize()
    rows, dist, cnt = col.knn(queries, 10)
    assert cnt.tolist() == [0] * 8


# ---- 4. filters ----------------------------------------------------------------------------------------------------------
def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return pack_row_filter(np.asarray(masks, bool))


@pytest.mark.parametrize("metric", ["HAMMING", "JACCARD"])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_filters(ctx, dtype, metric):
    rng = np.random.default_rng(zlib.crc32(f"filt{dtype}{metric}".encode()))
    n, dim = 40000 + 11, 48
    corpus = rng.integers(0, 4, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    col = make_col(ctx, corpus, metric=metric)
    masks = np.stack([np.ones(n, bool), rng.random(n) < 0.1, rng.random(n) < 0.01, np.zeros(n, bool),
                      rng.random(n) < 3000 / n])

    def run(queries, qf, k=10):
        kw = dict(filters=pack(masks), query_filter=qf)
        rows, dist, cnt, st = counted_and_exact(col, queries, k, **kw)
        for q in sample(queries.shape[0]):
            sk = (~masks[qf[q]]).astype(np.uint8)
            r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=sk)
            assert cnt[q] == r.size and rows[q, : cnt[q]].tolist() == r.tolist(), (q, qf[q])
            assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, qf[q])
        assert st["n_fallback"] == 0, st
        return st

    qs = rng.integers(0, 4, (6, dim)).astype(np.float64)
    st = run(qs, np.array([0, 1, 2, 3, 0, 1], np.uint32))   # 100 %, 10 %, 1 %, empty
    assert st["screen_used"] == SIMT_F32 and st["n_passes"] == 1
    st = run(qs, np.full(6, 4, np.uint32))                   # <= 4096 rows: the direct regime
    assert st["n_passes"] == 0, st
    run(qs, np.array([4, 0, 4, 2, 4, 1], np.uint32), k=256)  # mixed direct / counted batch
    qb = rng.integers(0, 4, (1100, dim)).astype(np.float64)
    run(qb, rng.integers(0, 5, 1100).astype(np.uint32))


# ---- 5. tickets, cancellation, shards, ownership -----------------------------------------------------------------------------
def test_async_tickets_in_flight(ctx):
    # four tickets in flight on two scratch sets: unfiltered, filtered (counted), unfiltered, filtered (direct regime)
    rng = np.random.default_rng(4)
    n, dim, nq, k = 20000, 64, 70, 10
    corpus = rng.integers(0, 2, (n, dim)).astype(np.float32)
    col = make_col(ctx, corpus)
    batches = [np.ascontiguousarray(rng.integers(0, 2, (nq, dim)).astype(np.float64)) for _ in range(4)]
    masks = np.zeros((2, n), bool)
    masks[0] = rng.random(n) < 0.3
    masks[1, rng.choice(n, 2000, replace=False)] = True
    filt = np.ascontiguousarray(pack(masks))
    qf = [None, np.zeros(nq, np.uint32), None, np.ones(nq, np.uint32)]
    outs = [(np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32)) for _ in range(4)]
    tickets = []
    for i in range(4):
        o = outs[i]
        if qf[i] is None:
            tickets.append(col.submit_host(batches[i].ctypes.data, nq, k, o[0].ctypes.data, o[1].ctypes.data,
                                           o[2].ctypes.data))
        else:
            tickets.append(col.submit_host_filtered(batches[i].ctypes.data, nq, k, filt.ctypes.data, 2, qf[i],
                                                    o[0].ctypes.data, o[1].ctypes.data, o[2].ctypes.data))
    for t in tickets:
        col.wait(t)
    for i in range(4):
        rows, dist, cnt = outs[i]
        skip = None if qf[i] is None else (~masks[int(qf[i][0])]).astype(np.uint8)
        check_oracle(corpus, batches[i], k, rows, dist, cnt, qs=sample(nq), skip=skip)


def test_cancellation_then_answers(ctx):
    from surrealdb_b200 import SdbError
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(9)
    corpus = rng.integers(0, 3, (30000, 32)).astype(np.float32)
    queries = rng.integers(0, 3, (4, 32)).astype(np.float64)
    col = make_col(ctx, corpus)
    flag = np.ones(1, np.int32)
    with pytest.raises(SdbError) as e:
        col.knn(queries, 10, cancel_flag=flag)
    assert e.value.status == L.SDB_ECANCELLED
    ctx.cancel()
    try:
        with pytest.raises(SdbError) as e:
            col.knn(queries, 10)
        assert e.value.status == L.SDB_ECANCELLED
    finally:
        ctx.cancel_reset()
    rows, dist, cnt = col.knn(queries, 10)
    check_oracle(corpus, queries, 10, rows, dist, cnt)


def test_two_shards_merged(ctx):
    import torch
    from surrealdb_b200 import VectorColumn
    from surrealdb_b200.engine import shard_block_layout, topk_merge_device
    rng = np.random.default_rng(2)
    rows_n, dim, nq, k, world = 20000, 32, 40, 10, 2
    corpus = rng.integers(0, 2, (rows_n, dim)).astype(np.float32)
    corpus[15000:15004] = corpus[100:104]  # exact ties across the shards resolve by global row
    queries = rng.integers(0, 2, (nq, dim)).astype(np.float64)
    queries[0] = corpus[100]
    dev = torch.device("cuda", 0)
    qd = torch.from_numpy(queries).to(dev)
    torch.cuda.synchronize()
    off_rows, off_dist, off_cnt, blk = shard_block_layout(nq, k)
    gathered = torch.zeros(world * blk, dtype=torch.uint8, device=dev)
    for r in range(world):
        base, n_local = r * rows_n // world, rows_n // world
        col = VectorColumn(ctx, dim, "HAMMING", "F32", capacity=n_local)
        col.append(corpus[base:base + n_local])
        col.finalize()
        p = gathered.data_ptr() + r * blk
        col.knn_device(qd.data_ptr(), nq, k, base, p + off_rows, p + off_dist, p + off_cnt)
        assert col.stats()["screen_used"] == SIMT_F32
    f_rows = torch.zeros((nq, k), dtype=torch.int64, device=dev)
    f_dist = torch.zeros((nq, k), dtype=torch.float64, device=dev)
    f_cnt = torch.zeros((nq,), dtype=torch.int32, device=dev)
    gp = gathered.data_ptr()
    topk_merge_device(ctx, world, nq, k, gp + off_rows, gp + off_dist, gp + off_cnt, f_rows.data_ptr(),
                      f_dist.data_ptr(), f_cnt.data_ptr(), stride_rows=blk // 8, stride_dist=blk // 8,
                      stride_counts=blk // 4)
    torch.cuda.synchronize()
    check_oracle(corpus, queries, k, f_rows.cpu().numpy().astype(np.uint64), f_dist.cpu().numpy(),
                 f_cnt.cpu().numpy().astype(np.uint32))


def test_allocations_return_to_baseline():
    import ctypes as C
    from surrealdb_b200 import Context
    from surrealdb_b200 import _lib as L

    def live():
        n, b = C.c_uint64(), C.c_uint64()
        L.lib().sdb_debug_live_allocations(C.byref(n), C.byref(b))
        return n.value, b.value

    rng = np.random.default_rng(3)
    before = live()
    own = Context(0)
    for metric in ("HAMMING", "JACCARD"):
        for dtype in (np.float32, np.float64):
            col = make_col(own, rng.integers(0, 3, (5000, 20)).astype(dtype), metric=metric)
            col.knn(rng.integers(0, 3, (70, 20)).astype(np.float64), 10)
            col.close()
    own.close()
    assert live() == before
