"""Brute-force KNN of MANHATTAN / CHEBYSHEV columns through the f32 L1 / L-infinity screen (screen_lp.cu), the proof
and the exact re-rank.  Every answer is compared bit for bit (rows, f64 distances, counts) with the CPU oracle; the
screen's premises (scores within beps of the reference, kept set = rows reaching tau, tau below the k-th score less
the margin, every excluded row beyond the proof's bound) are held through sdb_debug_screen_batch."""
import ctypes as C
import zlib

import numpy as np
import pytest

import lp_screen_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SIMT_F32, NONE_EXACT = 1, 3
METRICS = ["MANHATTAN", "CHEBYSHEV"]


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_col(ctx, corpus, metric, skip=None, screen=None):
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


def check(corpus, queries, metric, k, rows, dist, cnt, qs=None, skip=None):
    qs = range(queries.shape[0]) if qs is None else qs
    for q in qs:
        r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=skip)
        assert cnt[q] == r.size, (q, int(cnt[q]), r.size)
        assert rows[q, : cnt[q]].tolist() == r.tolist(), (q, rows[q, : cnt[q]], r)
        assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, dist[q, : cnt[q]], d)


def sample(nq):
    return sorted(set(list(range(0, nq, max(1, nq // 24))) + [nq - 1]))


# ---- 1. parity matrix ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 7, 100, 768, 1025, 4100])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric", METRICS)
def test_parity_matrix(ctx, metric, dtype, dim):
    rng = np.random.default_rng(zlib.crc32(f"{metric}{dtype}{dim}".encode()))
    n = 6000 if dim <= 1025 else 2500
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    col = make_col(ctx, corpus, metric)
    nqs = (1, 3, 17, 32, 64, 1024, 2100) if dim <= 768 else (1, 32, 64, 1024)
    for nq, screen in [(nq, "AUTO") for nq in nqs] + [(1, "SIMT_F32")]:
        col.set_screen(screen)
        queries = rng.uniform(-1, 1, (nq, dim))
        for k in (1, 10, 100, 256, 257):
            if nq > 64 and k not in (10, 257):
                continue
            rows, dist, cnt = col.knn(queries, k)
            st = col.stats()
            if nq == 1 and screen == "AUTO":  # one query: AUTO ranks it with the exact kernel (DESIGN.md section 5)
                assert st["screen_used"] == NONE_EXACT, (k, st)
            elif k <= 256:
                assert st["screen_used"] == SIMT_F32 and st["n_passes"] > 0, (nq, k, st)
                if dim > 1:  # (one dimension: ties everywhere, the proof may fail more often)
                    assert st["n_fallback"] <= 2 + nq // 64, (nq, k, st)
            else:
                assert st["screen_used"] == NONE_EXACT, (nq, k, st)
            check(corpus, queries, metric, k, rows, dist, cnt, qs=sample(nq))


# ---- 2. adversarial inputs -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric", METRICS)
def test_adversarial_rows(ctx, metric, dtype):
    rng = np.random.default_rng(zlib.crc32(f"adv{metric}{dtype}".encode()))
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
    if dtype == "F64":
        corpus[305, 2] = 1e39                     # beyond f32 range: special
        corpus[306] = rng.uniform(-1, 1, dim) * 1e-41  # f32-subnormal elements
        corpus[307, :4] = 1e-300
    queries[2] = corpus[303]                      # the all-zero row's exact match
    queries[3, 7] = 1e300                         # beyond f32 range: the exact path
    queries[4] = corpus[300].astype(np.float64)   # near the NaN row
    queries[4, 3] = 0.5
    queries[5] = corpus[202].astype(np.float64)
    col = make_col(ctx, corpus, metric)
    for k in (1, 10, 100, 256):
        rows, dist, cnt = col.knn(queries, k)
        assert col.stats()["screen_used"] == SIMT_F32
        check(corpus, queries, metric, k, rows, dist, cnt)
    assert col.stats()["n_special_rows"] == (3 if dtype == "F32" else 4)  # NaN, +-inf (f64: and 1e39) rows


@pytest.mark.parametrize("metric", METRICS)
def test_special_overflow_is_exact(ctx, metric):
    rng = np.random.default_rng(1025)
    corpus = rng.uniform(-1, 1, (6000, 16)).astype(np.float32)
    corpus[rng.choice(6000, 1025, replace=False), 3] = np.nan  # 1025 special rows: more than the list
    queries = rng.uniform(-1, 1, (5, 16))
    col = make_col(ctx, corpus, metric)
    rows, dist, cnt = col.knn(queries, 10)
    assert col.stats()["screen_used"] == NONE_EXACT
    check(corpus, queries, metric, 10, rows, dist, cnt)


@pytest.mark.parametrize("metric", METRICS)
def test_near_duplicate_crowd_on_a_large_offset(ctx, metric):
    # 20000 rows within 1e-2 of each other on an offset of 1e4: the bound (relative to the norms) is wider than the
    # spread, every row is a candidate and the lists of both rungs overflow -- the answers stay exact and the
    # fallbacks are counted
    rng = np.random.default_rng(77)
    dim = 32
    corpus = (1e4 + rng.uniform(0, 1e-2, (20000, dim))).astype(np.float32)
    queries = 1e4 + rng.uniform(0, 1e-2, (6, dim))
    col = make_col(ctx, corpus, metric)
    rows, dist, cnt = col.knn(queries, 10)
    st = col.stats()
    assert st["screen_used"] == SIMT_F32 and st["n_fallback"] == 6, st
    check(corpus, queries, metric, 10, rows, dist, cnt)


# ---- 3. skip masks and removed rows -----------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_skip_and_remove(ctx, metric):
    rng = np.random.default_rng(5)
    n, dim = 8000, 40
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = corpus[rng.integers(0, n, 8)].astype(np.float64) + rng.normal(0, 1e-3, (8, dim))
    skip = (rng.random(n) < 0.2).astype(np.uint8)
    dead = np.unique(rng.integers(0, n, 200)).astype(np.uint64)
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, dim, metric, "F32", capacity=n)
    col.append(corpus)
    col.set_skip(skip)
    col.remove(dead[:100])                        # before finalize
    col.finalize()
    col.remove(dead[100:])                        # after
    eff = skip.copy()
    eff[dead.astype(np.int64)] = 1
    rows, dist, cnt = col.knn(queries, 10)
    assert col.stats()["screen_used"] == SIMT_F32
    check(corpus, queries, metric, 10, rows, dist, cnt, skip=eff)


# ---- 4. filters ------------------------------------------------------------------------------------------------------
def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return pack_row_filter(np.asarray(masks, bool))


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("metric", METRICS)
def test_filters(ctx, metric, dtype):
    rng = np.random.default_rng(zlib.crc32(f"filt{metric}{dtype}".encode()))
    n, dim = 40000 + 11, 48
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    col = make_col(ctx, corpus, metric)
    masks = np.stack([np.ones(n, bool), rng.random(n) < 0.1, rng.random(n) < 0.01, rng.random(n) < 0.05,
                      rng.random(n) < 3000 / n])

    def run(queries, qf, k=10):
        rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
        for q in sample(queries.shape[0]):
            sk = (~masks[qf[q]]).astype(np.uint8)
            r, d = O.knn_topk(corpus, queries[q], metric.lower(), k, skip=sk)
            assert cnt[q] == r.size and rows[q, : cnt[q]].tolist() == r.tolist(), (q, qf[q])
            assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, qf[q])
        return col.stats()

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
    col = make_col(ctx, corpus, "MANHATTAN")
    dev = torch.device("cuda", 0)
    batches = [rng.uniform(-1, 1, (nq, dim)) for _ in range(4)]
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
        check(corpus, batches[i], "MANHATTAN", k, rows.astype(np.uint64), dist, cnt.astype(np.uint32),
              qs=sample(nq))


def test_cancellation_then_answers(ctx):
    from surrealdb_b200 import SdbError
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(9)
    corpus = rng.uniform(-1, 1, (30000, 32)).astype(np.float32)
    queries = rng.uniform(-1, 1, (4, 32))
    col = make_col(ctx, corpus, "CHEBYSHEV")
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
    check(corpus, queries, "CHEBYSHEV", 10, rows, dist, cnt)


@pytest.mark.parametrize("metric", METRICS)
def test_two_shards_merged(ctx, metric):
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
        col = VectorColumn(ctx, dim, metric, "F32", capacity=n_local)
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
    check(corpus, queries, metric, k, f_rows.cpu().numpy().astype(np.uint64), f_dist.cpu().numpy(),
          f_cnt.cpu().numpy().astype(np.uint32))


# ---- 6. the proof's premises -------------------------------------------------------------------------------------------
def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def debug_batch(col, Q, k, score_all, n_pad, cap=4096):
    from surrealdb_b200 import _lib as L
    nq = Q.shape[0]
    capq = max(cap, n_pad) if score_all else cap
    o = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
             a=np.zeros((nq, capq, 3), np.uint32))
    if not score_all:
        o["b"] = np.zeros((nq, capq, 2), np.uint32)
        o["rr"] = np.zeros((nq, capq + 1024), np.uint32)
    L.check(L.lib().sdb_debug_screen_batch(col.h, _p(Q), nq, k, SIMT_F32, 0, cap, int(score_all), _p(o["qf"]),
                                           _p(o["qmag"]), _p(o["qu"]), None, None, _p(o["a"]), _p(o.get("b")),
                                           _p(o.get("rr"))))
    o["tau"], o["margin"], o["beps"] = o["qf"][:, 0], o["qf"][:, 1], o["qf"][:, 3]
    o["flags"], o["qflags"], o["n_a"], o["n_e"] = (o["qu"][:, j].astype(np.int64) for j in (0, 1, 3, 5))
    return o


def _rounding_up_rows(n, dim):
    x = np.full((n, dim), 2.0 ** -24 * (1 + 2.0 ** -10), np.float32)
    x[:, 0] = 1.0
    return x


PREMISE_CASES = {
    "uniform_d100": lambda rng: rng.uniform(-1, 1, (3000, 100)),
    "binades_d257": lambda rng: np.exp2(rng.uniform(-20, 20, (2000, 257))) * np.where(np.arange(257) % 2, -1.0, 1.0),
    "rounding_up_d1025": lambda rng: np.concatenate([_rounding_up_rows(64, 1025), rng.uniform(0, 1e-3, (900, 1025))]),
    "special_d33": lambda rng: np.where(rng.random((2500, 33)) < 0.002, np.nan, rng.uniform(-1, 1, (2500, 33))),
}


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("case", list(PREMISE_CASES))
@pytest.mark.parametrize("metric", METRICS)
def test_proof_premises(ctx, metric, case, dtype):
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(zlib.crc32(f"{metric}{case}{dtype}".encode()))
    X = PREMISE_CASES[case](rng).astype(np.float32 if dtype == "F32" else np.float64)
    n, dim = X.shape
    k = 10
    col = make_col(ctx, X, metric)
    f, u = np.zeros(4, np.float32), np.zeros(5, np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, _p(f), _p(u), None, None, None, None))
    mnorm, n_special, n_pad = f[3], int(u[0]), int(u[4])
    snorm = np.zeros(n_pad, np.float32)
    special = np.zeros(max(n_special, 1), np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, None, None, None, None, _p(snorm), _p(special)))
    valid = ~np.isnan(snorm[:n])
    finite32 = np.isfinite(X.astype(np.float32)).all(axis=1)
    assert np.array_equal(valid, finite32) and np.isnan(snorm[n:]).all() and (snorm[:n][valid] == 0).all()
    assert set(special[:n_special].tolist()) == set(np.flatnonzero(~finite32).tolist())
    assert mnorm >= R.f32_norm(X[valid], metric).max()
    Q = X[rng.integers(0, n, 20)].astype(np.float64)
    Q = np.where(np.isfinite(Q), Q, 0.25) * rng.uniform(0.9, 1.1, (20, 1))
    Q[::4] = rng.uniform(-1, 1, Q[::4].shape) * np.nanmax(np.abs(X[valid]))
    Q = np.ascontiguousarray(Q)
    # (1) with score_all every valid pair is within beps of the reference distance
    o = debug_batch(col, Q, k, True, n_pad)
    S = np.full((Q.shape[0], n), np.nan, np.float32)
    for q in range(Q.shape[0]):
        rws = o["a"][q, : o["n_a"][q], 0]
        keep = rws < n
        S[q, rws[keep]] = o["a"][q, : o["n_a"][q], 1][keep].view(np.float32)
    assert not np.isnan(S[:, valid]).any() and np.isnan(S[:, ~valid]).all()
    d = R.reference(Q, X, metric)
    ok_q = (o["qflags"] & 1) == 0
    want_beps = R.beps(metric, dim, mnorm, Q.astype(np.float32))
    assert (o["beps"][ok_q] >= want_beps[ok_q] * (1 - 1e-9)).all()
    dev = np.abs(-S[:, valid].astype(np.float64) - d[:, valid])[ok_q]
    slack = dev - o["beps"][ok_q, None].astype(np.float64)
    assert (slack <= 0).all(), f"screen error above beps: {slack.max():.3g}"
    # (2)-(4) the production sequence: kept set, tau, and an audit of the proof
    o = debug_batch(col, Q, k, False, n_pad)
    for q in np.flatnonzero(ok_q):
        tau = np.float32(o["tau"][q])
        rows_a = o["a"][q, : o["n_a"][q], 0].astype(np.int64)
        sq = S[q, valid]
        if not (o["flags"][q] & 1):
            assert np.array_equal(np.sort(rows_a), np.flatnonzero(valid)[sq >= tau]), (q, "kept set")
        if tau > -np.inf:
            s_k = np.sort(sq)[::-1][k - 1]
            assert np.float64(tau) <= np.nextafter(np.float64(s_k) - np.float64(o["margin"][q]), np.inf), q
        if not (o["flags"][q] & 2) and tau > -np.inf:
            out = valid.copy()
            out[o["rr"][q, : o["n_e"][q]].astype(np.int64)] = False
            bound = -np.float64(tau) - np.float64(o["beps"][q])
            bad = np.flatnonzero(out & (d[q] < bound))
            assert bad.size == 0, (q, bad[:5].tolist())
