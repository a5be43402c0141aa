"""Brute-force KNN of MINKOWSKI columns of integer order 1 .. 8 through the f32 Lp screen (screen_lp.cu), the proof and
the exact re-rank.  Every answer equals the exact kernel's (SDB_SCREEN_NONE_EXACT) bit for bit -- rows, f64 distances,
counts -- and the CPU oracle's rows, with distances within 1e-12 of the oracle's (CUDA's pow() is not the host libm's).
The screen's premises (scores within beps of the reference, kept set = rows reaching tau, tau below the k-th score less
the margin, every excluded row beyond the proof's bound) are held through sdb_debug_screen_batch[_filtered]."""
import ctypes as C
import zlib

import numpy as np
import pytest

import minkowski_screen_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SIMT_F32, NONE_EXACT = 1, 3
ORDERS = [1, 2, 3, 4, 7, 8]


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


@pytest.fixture
def order_of_oracle():
    def set_order(p):
        O.lib().orc_set_minkowski_order(C.c_double(float(p)))
    yield set_order
    set_order(3.0)


def make_col(ctx, corpus, order, skip=None):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if corpus.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, corpus.shape[1], "MINKOWSKI", dt, capacity=max(1, corpus.shape[0]))
    col.append(corpus)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    col.set_minkowski_order(order)
    return col


def exact_of(col, queries, k, **kw):
    col.set_screen("NONE_EXACT")
    try:
        out = col.knn(queries, k, **kw)
        assert col.stats()["screen_used"] == NONE_EXACT
    finally:
        col.set_screen("AUTO")
    return out


def same(a, b):
    (ra, da, ca), (rb, db, cb) = a, b
    assert np.array_equal(ca, cb), "counts"
    for q in range(ca.shape[0]):
        n = int(ca[q])
        assert ra[q, :n].tolist() == rb[q, :n].tolist(), (q, ra[q, :n], rb[q, :n])
        assert da[q, :n].tobytes() == db[q, :n].tobytes(), (q, da[q, :n], db[q, :n])


def check_oracle(corpus, queries, k, res, qs, skip=None):
    """rows equal the oracle's (a swap is allowed only between distances equal to 1e-12, where the two libms' pow()
    may order a near-tie differently), distances within 1e-12 relative, counts exact."""
    rows, dist, cnt = res
    for q in qs:
        r, d = O.knn_topk(corpus, queries[q], "minkowski", k, skip=skip)
        n = int(cnt[q])
        assert n == r.size, (q, n, r.size)
        assert np.allclose(dist[q, :n], d, rtol=1e-12, atol=0.0), (q, dist[q, :n], d)
        for i in np.flatnonzero(rows[q, :n] != r):
            assert abs(dist[q, i] - d[i]) <= 1e-12 * abs(d[i]) and np.isin(rows[q, i], r), (q, i)


def sample(nq, m=3):
    return sorted(set(list(range(0, nq, max(1, nq // m))) + [nq - 1]))


# ---- 1. parity matrix ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 7, 100, 768, 1025, 4100])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("order", ORDERS)
def test_parity_matrix(ctx, order_of_oracle, order, dtype, dim):
    order_of_oracle(order)
    rng = np.random.default_rng(zlib.crc32(f"mink{order}{dtype}{dim}".encode()))
    n = 3000 if dim <= 1025 else 1200
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    col = make_col(ctx, corpus, order)
    nqs = (1, 3, 17, 32, 64, 2100) if dim <= 768 else (1, 32, 64, 1024)
    for nq in nqs:
        queries = rng.uniform(-1, 1, (nq, dim))
        for k in (1, 10, 100, 256, 257):
            if nq > 64 and k not in (10, 257):
                continue
            res = col.knn(queries, k)
            st = col.stats()
            if k <= 256:
                assert st["screen_used"] == SIMT_F32 and st["n_passes"] > 0, (nq, k, st)
                if dim > 1:  # (one dimension: ties everywhere, the proof may fail more often)
                    assert st["n_fallback"] <= 2 + nq // 64, (nq, k, st)
            else:
                assert st["screen_used"] == NONE_EXACT, (nq, k, st)
            same(res, exact_of(col, queries, k))
            if k in (10, 257):
                check_oracle(corpus, queries, k, res, sample(nq, 2))


@pytest.mark.parametrize("order", [1.5, 0.5, 9.0, 0.0, -1.0, np.inf])
def test_unscreened_orders_stay_exact(ctx, order_of_oracle, order):
    order_of_oracle(order)
    rng = np.random.default_rng(31)
    corpus = rng.uniform(-2, 2, (2000, 24)).astype(np.float32)
    queries = rng.uniform(-2, 2, (5, 24))
    col = make_col(ctx, corpus, order)
    for screen in ("AUTO", "SIMT_F32"):
        col.set_screen(screen)
        rows, dist, cnt = col.knn(queries, 10)
        assert col.stats()["screen_used"] == NONE_EXACT, (order, screen)
    col.set_screen("AUTO")
    if np.isfinite(order) and order > 0:
        check_oracle(corpus, queries, 10, (rows, dist, cnt), range(5))


def test_order_change_after_finalize(ctx, order_of_oracle):
    rng = np.random.default_rng(34)
    corpus = rng.uniform(-1, 1, (5000, 64)).astype(np.float32)
    queries = rng.uniform(-1, 1, (40, 64))
    col = make_col(ctx, corpus, 3)
    for p in (3, 4, 1.5, 8, 1):
        order_of_oracle(p)
        col.set_minkowski_order(p)
        res = col.knn(queries, 10)
        assert col.stats()["screen_used"] == (NONE_EXACT if p == 1.5 else SIMT_F32), p
        same(res, exact_of(col, queries, 10))
        check_oracle(corpus, queries, 10, res, sample(40))


def test_single_query_is_screened(ctx):
    rng = np.random.default_rng(35)
    corpus = rng.uniform(-1, 1, (4000, 96)).astype(np.float32)
    q = rng.uniform(-1, 1, (1, 96))
    col = make_col(ctx, corpus, 3)
    res = col.knn(q, 10)
    assert col.stats()["screen_used"] == SIMT_F32
    same(res, exact_of(col, q, 10))


# ---- 2. adversarial inputs -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("order", [2, 3, 8])
def test_adversarial_rows(ctx, order_of_oracle, order, dtype):
    order_of_oracle(order)
    rng = np.random.default_rng(zlib.crc32(f"advmink{order}{dtype}".encode()))
    n, dim = 5000, 64
    fdt = np.float32 if dtype == "F32" else np.float64
    corpus = rng.uniform(-1, 1, (n, dim)).astype(fdt)
    queries = rng.uniform(-1, 1, (12, dim))
    corpus[100:110] = corpus[50]                  # duplicates across the k cut
    corpus[200] = queries[1].astype(fdt)
    corpus[201] = corpus[200]
    corpus[202] = np.nextafter(corpus[200], fdt(np.inf))  # one-ulp near-ties
    corpus[300, 3] = np.nan                       # special rows
    corpus[301, 0] = np.inf
    corpus[302, 5] = -np.inf
    corpus[303] = 0.0
    corpus[304] = -0.0
    corpus[306] = rng.uniform(-1, 1, dim) * 1e-41  # f32-subnormal elements
    if dtype == "F64":
        corpus[305, 2] = 1e39                     # beyond f32 range: special
        corpus[307, :4] = 1e-300
    queries[2] = corpus[303]                      # the all-zero row's exact match
    queries[3, 7] = 1e300                         # beyond f32 range: the exact path
    queries[4] = corpus[300].astype(np.float64)   # near the NaN row
    queries[4, 3] = 0.5
    queries[5] = corpus[202].astype(np.float64)
    queries[6] = corpus[306].astype(np.float64)   # subnormal query next to the subnormal row
    col = make_col(ctx, corpus, order)
    for k in (1, 10, 100, 256):
        res = col.knn(queries, k)
        assert col.stats()["screen_used"] == SIMT_F32
        same(res, exact_of(col, queries, k))
        check_oracle(corpus, queries, k, res, range(12))
    assert col.stats()["n_special_rows"] == (3 if dtype == "F32" else 4)  # NaN, +-inf (f64: and 1e39) rows


@pytest.mark.parametrize("scale", [1e5, 1e-6])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_order_8_overflow_and_underflow_scales(ctx, order_of_oracle, scale, dtype):
    # (1e5)^8 = 1e40 overflows f32 and (1e-6)^8 = 1e-48 underflows it: the launch's power-of-two scale keeps both in
    # range, and the answers stay the exact kernel's
    order_of_oracle(8)
    rng = np.random.default_rng(int(scale * 1e6) % 1000 + 8)
    corpus = (rng.uniform(-1, 1, (6000, 128)) * scale).astype(np.float32 if dtype == "F32" else np.float64)
    queries = rng.uniform(-1, 1, (70, 128)) * scale
    col = make_col(ctx, corpus, 8)
    res = col.knn(queries, 10)
    st = col.stats()
    assert st["screen_used"] == SIMT_F32 and st["n_fallback"] <= 3, st
    same(res, exact_of(col, queries, 10))
    check_oracle(corpus, queries, 10, res, sample(70))


@pytest.mark.parametrize("rounded", ["query", "rows"])
def test_subnormal_rounding_of_queries_and_rows(ctx, order_of_oracle, rounded):
    # Elements 0.49 ulp off f32's subnormal grid: the f32 copy the screen reads moves every element by almost 2^-150,
    # an error the launch's scale does not shrink.  Row A is the true nearest (d = 0.51 D^(1/2) units of 2^-149) but
    # screens at 32 units; row B screens at 23 units but lies at 21.3.  A bound without the unscaled D^(1/p) 2^-149
    # term would cut A from the list (tau ~ -25) and still accept B through the proof: a wrong answer.
    order_of_oracle(2)
    unit, dim = 2.0 ** -149, 1024
    base = 1000 * unit
    rng = np.random.default_rng(2149)
    off = rng.integers(40, 60, (3000, dim)) * np.where(rng.random((3000, dim)) < 0.5, -1, 1)  # far rows
    off[7] = 1                                     # row A
    off[3] = 0                                     # row B: 429 elements at +1, 100 at -1, 495 at 0
    off[3, :429] = 1
    off[3, 429:529] = -1
    if rounded == "query":  # rows on the grid (F32), the f64 query 0.49 ulp above it
        corpus = (base + off * unit).astype(np.float32)
        queries = np.full((2, dim), base + 0.49 * unit)
    else:                   # the query on the grid, f64 rows that round onto the grid's +1 / -1 / 0
        true_off = np.where(off == 1, 0.51, np.where(off == -1, -1.49, np.where(off == 0, 0.49, off)))
        corpus = base + true_off * unit
        queries = np.full((2, dim), base)
    queries[1, ::2] += 3 * unit                   # a second query elsewhere
    col = make_col(ctx, corpus, 2)
    for k in (1, 10):
        res = col.knn(queries, k)
        assert col.stats()["screen_used"] == SIMT_F32
        assert res[0][0, 0] == 7, res[0][0, :k]
        same(res, exact_of(col, queries, k))
        check_oracle(corpus, queries, k, res, range(2))


def test_special_overflow_is_exact(ctx):
    rng = np.random.default_rng(1025)
    corpus = rng.uniform(-1, 1, (6000, 16)).astype(np.float32)
    corpus[rng.choice(6000, 1025, replace=False), 3] = np.nan  # 1025 special rows: more than the list
    queries = rng.uniform(-1, 1, (5, 16))
    col = make_col(ctx, corpus, 3)
    res = col.knn(queries, 10)
    assert col.stats()["screen_used"] == NONE_EXACT
    same(res, exact_of(col, queries, 10))


def test_near_duplicate_crowd_on_a_large_offset(ctx, order_of_oracle):
    # 20000 rows within 1e-2 of each other on an offset of 1e4: the bound (relative to the norms) is wider than the
    # spread, every row is a candidate and the lists of both rungs overflow -- the answers stay exact and the fallbacks
    # are counted
    order_of_oracle(3)
    rng = np.random.default_rng(77)
    dim = 32
    corpus = (1e4 + rng.uniform(0, 1e-2, (20000, dim))).astype(np.float32)
    queries = 1e4 + rng.uniform(0, 1e-2, (6, dim))
    col = make_col(ctx, corpus, 3)
    res = col.knn(queries, 10)
    st = col.stats()
    assert st["screen_used"] == SIMT_F32 and st["n_fallback"] == 6, st
    same(res, exact_of(col, queries, 10))
    check_oracle(corpus, queries, 10, res, range(6))


# ---- 3. skip masks and removed rows -----------------------------------------------------------------------------------
def test_skip_and_remove(ctx, order_of_oracle):
    order_of_oracle(4)
    rng = np.random.default_rng(5)
    n, dim = 8000, 40
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = corpus[rng.integers(0, n, 8)].astype(np.float64) + rng.normal(0, 1e-3, (8, dim))
    skip = (rng.random(n) < 0.2).astype(np.uint8)
    dead = np.unique(rng.integers(0, n, 200)).astype(np.uint64)
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, dim, "MINKOWSKI", "F32", capacity=n)
    col.set_minkowski_order(4)
    col.append(corpus)
    col.set_skip(skip)
    col.remove(dead[:100])                        # before finalize
    col.finalize()
    col.remove(dead[100:])                        # after
    eff = skip.copy()
    eff[dead.astype(np.int64)] = 1
    res = col.knn(queries, 10)
    assert col.stats()["screen_used"] == SIMT_F32
    same(res, exact_of(col, queries, 10))
    check_oracle(corpus, queries, 10, res, range(8), skip=eff)


# ---- 4. filters ------------------------------------------------------------------------------------------------------
def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return pack_row_filter(np.asarray(masks, bool))


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("order", [3, 8])
def test_filters(ctx, order_of_oracle, order, dtype):
    order_of_oracle(order)
    rng = np.random.default_rng(zlib.crc32(f"filtmink{order}{dtype}".encode()))
    n, dim = 40000 + 11, 48
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    col = make_col(ctx, corpus, order)
    masks = np.stack([np.ones(n, bool), rng.random(n) < 0.1, rng.random(n) < 0.01, rng.random(n) < 0.05,
                      rng.random(n) < 3000 / n])

    def run(queries, qf, k=10):
        kw = dict(filters=pack(masks), query_filter=qf)
        res = col.knn(queries, k, **kw)
        st = col.stats()
        same(res, exact_of(col, queries, k, **kw))
        for q in sample(queries.shape[0], 4):
            check_oracle(corpus, queries, k, res, [q], skip=(~masks[qf[q]]).astype(np.uint8))
        return st

    qs = rng.uniform(-1, 1, (6, dim))
    st = run(qs, np.array([0, 1, 2, 3, 0, 1], np.uint32))  # 100 %, 10 %, 1 %, 5 %
    assert st["screen_used"] == SIMT_F32 and st["n_passes"] > 0
    st = run(qs, np.full(6, 4, np.uint32))                  # <= 4096 rows: the direct regime, no screen
    assert st["n_passes"] == 0, st
    run(qs, np.array([4, 0, 4, 2, 4, 1], np.uint32))        # mixed direct / screened batch
    qb = rng.uniform(-1, 1, (2100, dim))                    # query-chunked batch
    run(qb, rng.integers(0, 5, 2100).astype(np.uint32))


# ---- 5. tickets, cancellation, shards ----------------------------------------------------------------------------------
def test_async_tickets_in_flight(ctx):
    import torch
    rng = np.random.default_rng(4)
    n, dim, nq, k = 20000, 64, 70, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    # four batches of different magnitudes: each ticket's launches use their own batch's scale
    batches = [rng.uniform(-1, 1, (nq, dim)) * s for s in (1.0, 30.0, 0.01, 1.0)]
    col = make_col(ctx, corpus, 5)
    dev = torch.device("cuda", 0)
    qd = [torch.from_numpy(b).to(dev) for b in batches]
    outs = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
             torch.zeros(nq, dtype=torch.int32, device=dev)) for _ in range(4)]
    torch.cuda.synchronize()
    tickets = [col.submit_device(qd[i].data_ptr(), nq, k, 0, outs[i][0].data_ptr(), outs[i][1].data_ptr(),
                                 outs[i][2].data_ptr()) for i in range(4)]
    for t in tickets:
        col.wait(t)
    torch.cuda.synchronize()
    for i in range(4):
        rows, dist, cnt = (o.cpu().numpy() for o in outs[i])
        same((rows.astype(np.uint64), dist, cnt.astype(np.uint32)), exact_of(col, batches[i], k))


def test_cancellation_then_answers(ctx):
    from surrealdb_b200 import SdbError
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(9)
    corpus = rng.uniform(-1, 1, (30000, 32)).astype(np.float32)
    queries = rng.uniform(-1, 1, (4, 32))
    col = make_col(ctx, corpus, 3)
    flag = np.ones(1, np.int32)
    with pytest.raises(SdbError) as e:
        col.knn(queries, 10, cancel_flag=flag)
    assert e.value.status == L.SDB_ECANCELLED
    res = col.knn(queries, 10)
    assert col.stats()["screen_used"] == SIMT_F32
    same(res, exact_of(col, queries, 10))


def test_two_shards_merged(ctx):
    import torch
    from surrealdb_b200 import VectorColumn
    from surrealdb_b200.engine import shard_block_layout, topk_merge_device
    rng = np.random.default_rng(2)
    rows_n, dim, nq, k, world = 20000, 64, 40, 10, 2
    corpus = rng.uniform(-1, 1, (rows_n, dim)).astype(np.float32)
    corpus[15000:15004] = corpus[100:104]  # exact ties across the shards resolve by global row
    queries = rng.uniform(-1, 1, (nq, dim))
    queries[0] = corpus[100]
    dev = torch.device("cuda", 0)
    qd = torch.from_numpy(queries).to(dev)
    torch.cuda.synchronize()
    off_rows, off_dist, off_cnt, blk = shard_block_layout(nq, k)
    gathered = torch.zeros(world * blk, dtype=torch.uint8, device=dev)
    for r in range(world):
        base, n_local = r * rows_n // world, rows_n // world
        col = VectorColumn(ctx, dim, "MINKOWSKI", "F32", capacity=n_local)
        col.append(corpus[base:base + n_local])
        col.finalize()
        col.set_minkowski_order(3)
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
    whole = make_col(ctx, corpus, 3)
    same((f_rows.cpu().numpy().astype(np.uint64), f_dist.cpu().numpy(), f_cnt.cpu().numpy().astype(np.uint32)),
         exact_of(whole, queries, k))


# ---- 6. the proof's premises -------------------------------------------------------------------------------------------
def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def debug_batch(col, Q, k, score_all, n_pad, cap=4096, filters=None, qf=None):
    from surrealdb_b200 import _lib as L
    nq = Q.shape[0]
    capq = max(cap, n_pad) if score_all else cap
    o = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
             a=np.zeros((nq, capq, 3), np.uint32))
    if not score_all:
        o["b"] = np.zeros((nq, capq, 2), np.uint32)
        o["rr"] = np.zeros((nq, capq + 1024), np.uint32)
    args = (col.h, _p(Q), nq, k, SIMT_F32, 0, cap, int(score_all), _p(o["qf"]), _p(o["qmag"]), _p(o["qu"]), None,
            None, _p(o["a"]), _p(o.get("b")), _p(o.get("rr")))
    if filters is None:
        L.check(L.lib().sdb_debug_screen_batch(*args))
    else:
        L.check(L.lib().sdb_debug_screen_batch_filtered(*args, _p(filters), filters.shape[0], _p(qf), -1))
    o["tau"], o["margin"], o["beps"] = o["qf"][:, 0], o["qf"][:, 1], o["qf"][:, 3]
    o["flags"], o["qflags"], o["n_a"], o["n_e"] = (o["qu"][:, j].astype(np.int64) for j in (0, 1, 3, 5))
    return o


PREMISE_CASES = {
    "uniform_d100": lambda rng: rng.uniform(-1, 1, (3000, 100)),
    "binades_d257": lambda rng: np.exp2(rng.uniform(-20, 20, (2000, 257))) * np.where(np.arange(257) % 2, -1.0, 1.0),
    "rounding_up_d1025": lambda rng: np.concatenate([R.rounding_up_rows(64, 1025), rng.uniform(0, 1e-3, (900, 1025))]),
    "special_d33": lambda rng: np.where(rng.random((2500, 33)) < 0.002, np.nan, rng.uniform(-1, 1, (2500, 33))),
}


def corpus_state(col, n):
    from surrealdb_b200 import _lib as L
    f, u = np.zeros(4, np.float32), np.zeros(5, np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, _p(f), _p(u), None, None, None, None))
    mnorm, n_special, n_pad = f[3], int(u[0]), int(u[4])
    snorm = np.zeros(n_pad, np.float32)
    special = np.zeros(max(n_special, 1), np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, None, None, None, None, _p(snorm), _p(special)))
    return mnorm, n_special, n_pad, snorm, special


def scores_of(o, nq, n):
    S = np.full((nq, n), np.nan, np.float32)
    for q in range(nq):
        rws = o["a"][q, : o["n_a"][q], 0]
        keep = rws < n
        S[q, rws[keep]] = o["a"][q, : o["n_a"][q], 1][keep].view(np.float32)
    return S


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("case", list(PREMISE_CASES))
@pytest.mark.parametrize("order", [2, 3, 8])
def test_proof_premises(ctx, order, case, dtype):
    rng = np.random.default_rng(zlib.crc32(f"mink{order}{case}{dtype}".encode()))
    X = PREMISE_CASES[case](rng).astype(np.float32 if dtype == "F32" else np.float64)
    n, dim = X.shape
    k = 10
    col = make_col(ctx, X, order)
    mnorm, n_special, n_pad, snorm, special = corpus_state(col, n)
    valid = ~np.isnan(snorm[:n])
    finite32 = np.isfinite(X.astype(np.float32)).all(axis=1)
    assert np.array_equal(valid, finite32) and np.isnan(snorm[n:]).all() and (snorm[:n][valid] == 0).all()
    assert set(special[:n_special].tolist()) == set(np.flatnonzero(~finite32).tolist())
    assert mnorm == R.max_abs(X[valid])  # max_norm: the largest |x^_i| of a screened row
    Q = X[rng.integers(0, n, 20)].astype(np.float64)
    Q = np.where(np.isfinite(Q), Q, 0.25) * rng.uniform(0.9, 1.1, (20, 1))
    Q[::4] = rng.uniform(-1, 1, Q[::4].shape) * np.nanmax(np.abs(X[valid]))
    Q = np.ascontiguousarray(Q)
    # (1) with score_all every valid pair is within beps of the reference distance
    o = debug_batch(col, Q, k, True, n_pad)
    S = scores_of(o, Q.shape[0], n)
    assert not np.isnan(S[:, valid]).any() and np.isnan(S[:, ~valid]).all()
    d = R.reference(Q, X[valid], order)
    ok_q = (o["qflags"] & 1) == 0
    want_beps = R.beps(order, dim, mnorm, Q.astype(np.float32), R.batch_exponent(mnorm, Q.astype(np.float32)))
    assert (o["beps"][ok_q] >= want_beps[ok_q] * (1 - 1e-9)).all()
    dev = np.abs(-S[:, valid].astype(np.float64) - d)[ok_q]
    slack = dev - o["beps"][ok_q, None].astype(np.float64)
    assert (slack <= 0).all(), f"screen error above beps: {slack.max():.3g}"
    # (2)-(4) the production sequence: kept set, tau, and an audit of the proof
    o = debug_batch(col, Q, k, False, n_pad)
    audit(o, S, d, valid, ok_q, k)


def audit(o, S, d, valid, ok_q, k, passing=None):
    """kept set = rows reaching tau, tau <= k-th (passing) score - margin, every excluded row at or beyond the proof's
    bound.  d: [nq][valid rows] reference distances; passing: [nq][n] the query's filter (None: every row)."""
    idx = np.flatnonzero(valid)
    for q in np.flatnonzero(ok_q):
        tau = np.float32(o["tau"][q])
        pas = np.ones(valid.size, bool) if passing is None else passing[q]
        sel = pas[idx]
        rows_a = o["a"][q, : o["n_a"][q], 0].astype(np.int64)
        sq = S[q, idx]
        if not (o["flags"][q] & 1):
            assert np.array_equal(np.sort(rows_a), idx[sel & (sq >= tau)]), (q, "kept set")
        if tau > -np.inf:
            s_k = np.sort(sq[sel])[::-1][k - 1]
            assert np.float64(tau) <= np.nextafter(np.float64(s_k) - np.float64(o["margin"][q]), np.inf), q
        if not (o["flags"][q] & 2) and tau > -np.inf:
            out = np.zeros(valid.size, bool)
            out[idx[sel]] = True
            out[o["rr"][q, : o["n_e"][q]].astype(np.int64)] = False
            bound = -np.float64(tau) - np.float64(o["beps"][q])
            dq = np.full(valid.size, np.inf)
            dq[idx] = d[q]
            bad = np.flatnonzero(out & (dq < bound))
            assert bad.size == 0, (q, bad[:5].tolist())


@pytest.mark.parametrize("order", [3, 8])
def test_filtered_proof_premises(ctx, order):
    # a filter that rejects each query's best rows: tau must stay below the k-th PASSING score
    rng = np.random.default_rng(zlib.crc32(f"filtprem{order}".encode()))
    n, dim, k, nq = 20000, 64, 10, 8
    X = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    col = make_col(ctx, X, order)
    mnorm, _, n_pad, snorm, _ = corpus_state(col, n)
    valid = ~np.isnan(snorm[:n])
    Q = rng.uniform(-1, 1, (nq, dim))
    d = R.reference(Q, X, order)  # (no special rows: every row is valid)
    masks = np.ones((nq, n), bool)
    for q in range(nq):
        masks[q, np.argsort(d[q])[:500]] = False      # the 500 nearest rows fail the filter
        masks[q] &= rng.random(n) < 0.5
    qf = np.arange(nq, dtype=np.uint32)
    filt = np.ascontiguousarray(pack(masks))
    S = scores_of(debug_batch(col, Q, k, True, n_pad), nq, n)  # every score, unfiltered
    o = debug_batch(col, Q, k, False, n_pad, filters=filt, qf=qf)
    audit(o, S, d, valid, np.ones(nq, bool), k, passing=masks)
